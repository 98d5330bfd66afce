// Context, error reporting, tensor-map encoding and the NCCL weight-broadcast wrappers of libdkb200.so.
#include <dlfcn.h>

#include "host.h"

static thread_local char g_err[1024] = "";

void dk_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" const char* dk_last_error(void) { return g_err; }
extern "C" const char* dk_version(void) { return "dkb200 0.1.0 (sm_90a)"; }

extern "C" int dk_ctx_create(int device, dk_ctx** out) {
  DK_REQUIRE(out != nullptr, "dk_ctx_create: null out");
  *out = nullptr;
  int ndev = 0;
  DK_CHECK_CUDA(cudaGetDeviceCount(&ndev));
  DK_REQUIRE(device >= 0 && device < ndev, "dk_ctx_create: device %d out of range (%d devices)", device, ndev);
  int prev_device = 0;
  DK_CHECK_CUDA(cudaGetDevice(&prev_device));
  struct Restore {   // the caller's current device is not ours to change
    int d;
    ~Restore() { cudaSetDevice(d); }
  } restore{prev_device};
  DK_CHECK_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  DK_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
  DK_REQUIRE(prop.major == 9 && prop.minor == 0, "dk_ctx_create: device %d is sm_%d%d; this library is built for sm_90a only", device,
             prop.major, prop.minor);
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  DK_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  DK_REQUIRE(fn != nullptr && qres == cudaDriverEntryPointSuccess, "dk_ctx_create: cuTensorMapEncodeTiled not found");
  dk_ctx* c = new dk_ctx();
  c->device = device;
  c->sm_count = prop.multiProcessorCount;
  c->encode_tiled = reinterpret_cast<dk_encode_tiled_fn>(fn);
  c->launches = 0;
  c->nccl_comm = nullptr;
  c->nccl_lib = nullptr;
  *out = c;
  return 0;
}

extern "C" void dk_ctx_destroy(dk_ctx* ctx) {
  if (ctx == nullptr) return;
  dk_comm_destroy(ctx);
  delete ctx;
}

extern "C" long long dk_ctx_launch_count(dk_ctx* ctx) { return ctx ? ctx->launches : 0; }

int dk_make_tmap_16b(dk_ctx* ctx, CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides) {
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = elem_strides ? elem_strides[i] : 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  // the data type only matters for OOB-fill / element size; bf16 and fp16 are both 2-byte tiles
  CUresult r = ctx->encode_tiled(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank),
                                 const_cast<void*>(base), gdim, gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                 CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    dk_set_error("cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu,%llu,..] box [%u,%u,..] base %p", (int)r, rank,
                 (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0],
                 rank > 1 ? box[1] : 0, base);
    return -4;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------
// NCCL (loaded lazily with dlopen so the library has no hard link-time dependency)
// ------------------------------------------------------------------------------------------------
typedef struct {
  char internal[128];
} dk_nccl_uid;
typedef int (*nccl_get_uid_fn)(dk_nccl_uid*);
typedef int (*nccl_init_rank_fn)(void**, int, dk_nccl_uid, int);
typedef int (*nccl_bcast_fn)(const void*, void*, size_t, int, int, void*, cudaStream_t);
typedef int (*nccl_destroy_fn)(void*);

static void* dk_open_nccl() {
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    void* h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (h) return h;
  }
  return nullptr;
}

extern "C" int dk_comm_unique_id(uint8_t id_host[128]) {
  void* lib = dk_open_nccl();
  DK_REQUIRE(lib != nullptr, "dk_comm_unique_id: libnccl not found");
  auto get = reinterpret_cast<nccl_get_uid_fn>(dlsym(lib, "ncclGetUniqueId"));
  DK_REQUIRE(get != nullptr, "dk_comm_unique_id: ncclGetUniqueId missing");
  dk_nccl_uid uid;
  const int rc = get(&uid);
  DK_REQUIRE(rc == 0, "ncclGetUniqueId failed (%d)", rc);
  memcpy(id_host, uid.internal, 128);
  return 0;
}

extern "C" int dk_comm_init(dk_ctx* ctx, int rank, int world, const uint8_t id_host[128]) {
  DK_REQUIRE(ctx != nullptr, "dk_comm_init: null ctx");
  DkDeviceGuard dk_guard_(ctx);
  DK_REQUIRE(ctx->nccl_comm == nullptr, "dk_comm_init: communicator already initialised");
  void* lib = dk_open_nccl();
  DK_REQUIRE(lib != nullptr, "dk_comm_init: libnccl not found");
  auto init = reinterpret_cast<nccl_init_rank_fn>(dlsym(lib, "ncclCommInitRank"));
  DK_REQUIRE(init != nullptr, "dk_comm_init: ncclCommInitRank missing");
  dk_nccl_uid uid;
  memcpy(uid.internal, id_host, 128);
  DK_CHECK_CUDA(cudaSetDevice(ctx->device));
  void* comm = nullptr;
  const int rc = init(&comm, world, uid, rank);
  DK_REQUIRE(rc == 0, "ncclCommInitRank failed (%d)", rc);
  ctx->nccl_comm = comm;
  ctx->nccl_lib = lib;
  return 0;
}

extern "C" int dk_comm_broadcast(dk_ctx* ctx, void* ptr, size_t bytes, int root, void* stream) {
  DK_REQUIRE(ctx != nullptr && ctx->nccl_comm != nullptr, "dk_comm_broadcast: communicator not initialised");
  DkDeviceGuard dk_guard_(ctx);
  auto bcast = reinterpret_cast<nccl_bcast_fn>(dlsym(ctx->nccl_lib, "ncclBroadcast"));
  DK_REQUIRE(bcast != nullptr, "dk_comm_broadcast: ncclBroadcast missing");
  const int rc = bcast(ptr, ptr, bytes, /*ncclInt8*/ 0, root, ctx->nccl_comm, static_cast<cudaStream_t>(stream));
  DK_REQUIRE(rc == 0, "ncclBroadcast failed (%d)", rc);
  return 0;
}

extern "C" int dk_comm_destroy(dk_ctx* ctx) {
  if (ctx == nullptr || ctx->nccl_comm == nullptr) return 0;
  auto destroy = reinterpret_cast<nccl_destroy_fn>(dlsym(ctx->nccl_lib, "ncclCommDestroy"));
  if (destroy) destroy(ctx->nccl_comm);
  ctx->nccl_comm = nullptr;
  return 0;
}
