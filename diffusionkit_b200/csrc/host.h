// Host-side internals shared by the translation units of libdkb200.so.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <unordered_map>

#include "../../include/dkb200.h"

typedef CUresult (*dk_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                       const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                       CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct dk_ctx {
  int device;
  int sm_count;
  dk_encode_tiled_fn encode_tiled;
  long long launches;
  void* nccl_comm;  // ncclComm_t, lazily created by dk_comm_init
  void* nccl_lib;   // dlopen handle
  // Kernel set-up belongs to the kernel as loaded in this device's context, so it is cached here, not per process:
  std::unordered_map<const void*, int> smem_limit;    // kernel -> dynamic shared-memory limit set (dk_kernel_smem)
  std::unordered_map<const void*, int> max_clusters;  // GEMM kernel -> resident 2-CTA clusters
};

void dk_set_error(const char* fmt, ...);

// Every entry point runs on ITS context's device whatever the calling thread's current device is (two pipelines on
// two GPUs in one process), and leaves the thread's device as it found it.
struct DkDeviceGuard {
  int prev = -1;
  bool switched = false;
  explicit DkDeviceGuard(const dk_ctx* c) {
    if (c != nullptr && cudaGetDevice(&prev) == cudaSuccess && prev != c->device)
      switched = cudaSetDevice(c->device) == cudaSuccess;
  }
  ~DkDeviceGuard() {
    if (switched) cudaSetDevice(prev);
  }
  DkDeviceGuard(const DkDeviceGuard&) = delete;
  DkDeviceGuard& operator=(const DkDeviceGuard&) = delete;
};

#define DK_CHECK_CUDA(expr)                                                                        \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      dk_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));          \
      return -2;                                                                                   \
    }                                                                                              \
  } while (0)

#define DK_REQUIRE(cond, ...)        \
  do {                               \
    if (!(cond)) {                   \
      dk_set_error(__VA_ARGS__);     \
      return -1;                     \
    }                                \
  } while (0)

#define DK_LAUNCH_CHECK(ctx)                                                                       \
  do {                                                                                             \
    cudaError_t _e = cudaGetLastError();                                                           \
    if (_e != cudaSuccess) {                                                                       \
      dk_set_error("%s:%d: kernel launch failed -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return -3;                                                                                   \
    }                                                                                              \
    (ctx)->launches++;                                                                             \
  } while (0)

// Opens every entry point that takes a ctx: a null ctx is refused with a message that names the entry point, and the
// rest of the call runs on the ctx's device.
#define DK_ENTRY(ctx)                                       \
  DK_REQUIRE((ctx) != nullptr, "%s: null ctx", __func__); \
  DkDeviceGuard dk_guard_(ctx)

#define DK_DTYPE_OK(dt) DK_REQUIRE((dt) == DK_BF16 || (dt) == DK_FP16, "%s: bad dtype %d", __func__, (dt))

// Runs the statement with T bound to the 16-bit type of a dtype that DK_DTYPE_OK has accepted.
#define DK_DISPATCH(dt, ...)   \
  do {                         \
    if ((dt) == DK_BF16) {     \
      using T = __nv_bfloat16; \
      __VA_ARGS__;             \
    } else {                   \
      using T = __half;        \
      __VA_ARGS__;             \
    }                          \
  } while (0)

// Raises func's dynamic shared-memory limit to `bytes` the first time it is launched through ctx.
int dk_kernel_smem(dk_ctx* ctx, const void* func, int bytes);

// Tiled tensor map over a tensor of 16-bit (elem_bytes 2) or 8-bit (elem_bytes 1) elements, 128B swizzle, zero OOB
// fill (a zero byte is e4m3 +0).
//   rank 2..4; dims[0] is the contiguous dimension; strides_bytes has rank-1 entries (dims 1..), multiples of 16.
//   elem_strides (optional, rank entries): traversal stride per dimension; to load N elements with stride s the box
//   entry must be N * s (cuTensorMapEncodeTiled semantics).
int dk_make_tmap(dk_ctx* ctx, CUtensorMap* map, int elem_bytes, const void* base, int rank, const uint64_t* dims,
                 const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides = nullptr);
static inline int dk_make_tmap_16b(dk_ctx* ctx, CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                                   const uint64_t* strides_bytes, const uint32_t* box,
                                   const uint32_t* elem_strides = nullptr) {
  return dk_make_tmap(ctx, map, 2, base, rank, dims, strides_bytes, box, elem_strides);
}

static inline int dk_ceil_div(int a, int b) { return (a + b - 1) / b; }

static inline bool dk_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Blocks for a grid-stride kernel: one work item per thread, at most 16 blocks per SM.
static inline int dk_grid_for(long long work_items, int threads, int sm_count) {
  long long blocks = (work_items + threads - 1) / threads;
  const long long cap = static_cast<long long>(sm_count) * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}
