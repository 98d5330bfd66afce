// diffusionkit_b200 — sm_90a device-side primitives (hand-written PTX wrappers).
//
// Everything here is the Hopper programming model spelled out directly:
// mbarrier producer/consumer pipelines, TMA tiled loads (cp.async.bulk.tensor),
// wgmma warpgroup MMAs with register accumulators.  No CUTLASS.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "wgmma.cuh"

namespace dk {

// --------------------------------------------------------------------------------------------
// generic helpers
// --------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}


// --------------------------------------------------------------------------------------------
// mbarrier
// --------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"   // (a suspend-time hint was measured 35 % slower)
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok;
}
// Wait until the phase with the given parity has completed.  try_wait suspends the thread in hardware for ~100 clocks
// per attempt; the retry loop is kept minimal (ncu: with a clock64() watchdog in it the polling loops of the waiting
// warps were a quarter of all instructions the attention kernel issued).  The watchdog counts attempts instead:
// 2^26 of them is a few seconds, then the kernel traps, so a dead-locked pipeline fails its launch with an error
// instead of hanging the GPU.  The trap is inline and the wait calls nothing: a function call anywhere in a kernel
// makes ptxas serialise all of its wgmma instructions (warning C7510, which the build refuses), so the watchdog does
// not report which block or barrier tripped it.
#ifndef DK_WATCHDOG_SPINS
#define DK_WATCHDOG_SPINS (1u << 26)
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins == DK_WATCHDOG_SPINS) asm volatile("trap;");
  }
}

// Whole-warp wait with a single polling lane: lane 0 spins (hardware-suspended try_wait), the other 31 lanes park at
// the warp barrier instead of burning issue slots and power on their own polls.
__device__ __forceinline__ void mbar_wait_warp(uint64_t* bar, uint32_t parity) {
  if ((threadIdx.x & 31) == 0) mbar_wait(bar, parity);
  __syncwarp();
}

// 32-bit store to shared memory through its shared-window address: unlike a store through a generic pointer, it does
// not keep the compiler from moving global loads above it
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v));
}

// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// --------------------------------------------------------------------------------------------
// thread-block clusters
// --------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// every thread of every CTA of the cluster; orders barrier initialisation / remote shared-memory traffic
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `cta` of the cluster (which may be this CTA).  Plain
// arrive: a .release.cluster arrive after every k-block made the GEMM mainloop markedly slower (measured on H100).
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}" ::"r"(smem_u32(bar)),
      "r"(cta)
      : "memory");
}

// --------------------------------------------------------------------------------------------
// TMA (tiled tensor maps, 128B swizzle) — completion signalled on an mbarrier as transaction bytes
// --------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::
          "r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// The same box written to the same shared-memory offset of every CTA in cta_mask; each destination CTA's mbarrier at
// bar's offset receives the transaction bytes.
__device__ __forceinline__ void tma_load_2d_multicast(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                                      uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster "
      "[%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// --------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA): A and B read from shared memory through matrix descriptors (A optionally from registers),
// D accumulated in registers of the 128 threads of a warpgroup.
// --------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keep the accumulator registers live across the asynchronous MMAs (the compiler must not move reads or writes of them
// across a wgmma_wait)
template <int N>
__device__ __forceinline__ void reg_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Shared-memory matrix descriptor (sm_90 wgmma format) for a 128B-swizzled tile whose rows are 128-byte lines as
// written by a TMA box with a 64 x 16-bit inner extent.
//   K-major  operand: rows = M/N index, the 128B line holds 64 consecutive K.  SBO = 1024 B (8-row group stride).
//                     Stepping K by 16 inside the line is a 32-byte start-address step.
//   MN-major operand: rows = K index, the 128B line holds 64 consecutive M/N.  SBO = 1024 B (8 K-rows),
//                     LBO = byte stride between successive 64-wide M/N atoms.
// The swizzle is a function of the shared-memory address bits (chunk ^= line & 7) for the TMA write and the operand
// read alike, so a start address shifted by whole 128-byte lines addresses the shifted tile (base offset field 0).
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);           // [0,14)  start address >> 4
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;      // [16,30) leading byte offset >> 4
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;      // [32,46) stride byte offset >> 4
  d |= static_cast<uint64_t>(1) << 62;                               // [62,64) layout: SWIZZLE_128B
  return d;
}

// One lane of a converged warp (the TMA issue idiom: the whole warp runs the loop so addresses stay in uniform
// registers; only the issue itself is predicated on the elected lane).
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// Accumulator fragment of one m64nN wgmma (this thread's N/2 floats) -> fp32 rows of a shared-memory staging tile.
// Fragment layout: warp w of the warpgroup owns rows 16w..16w+15; d[4j + 2i + e] is row 16w + lane/4 + 8i,
// column 8j + 2*(lane%4) + e.
template <int N>
__device__ __forceinline__ void stage_acc_rows(float* stage, int ld, int row0, const float (&d)[N / 2]) {
  const int t = threadIdx.x & 127;
  const int r = row0 + (t >> 5) * 16 + ((t & 31) >> 2);
  const int c = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i)
      *reinterpret_cast<float2*>(stage + (r + 8 * i) * ld + 8 * j + c) = make_float2(d[4 * j + 2 * i], d[4 * j + 2 * i + 1]);
}

// --------------------------------------------------------------------------------------------
// 16-bit type traits (bf16 for FLUX, fp16 for SD3 — reference: mlx/__init__.py:76,610)
// --------------------------------------------------------------------------------------------
template <typename T>
struct Half16;
template <>
struct Half16<__nv_bfloat16> {
  using T2 = __nv_bfloat162;
  static constexpr bool is_bf16 = true;
  __device__ static __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  __device__ static __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
  __device__ static __forceinline__ uint32_t pack(float lo, float hi) {
    __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&t);
  }
  __device__ static __forceinline__ float2 unpack(uint32_t u) {
    __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&u);
    return __bfloat1622float2(t);
  }
};
template <>
struct Half16<__half> {
  using T2 = __half2;
  static constexpr bool is_bf16 = false;
  __device__ static __forceinline__ float to_f(__half v) { return __half2float(v); }
  __device__ static __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
  __device__ static __forceinline__ uint32_t pack(float lo, float hi) {
    __half2 t = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&t);
  }
  __device__ static __forceinline__ float2 unpack(uint32_t u) {
    __half2 t = *reinterpret_cast<__half2*>(&u);
    return __half22float2(t);
  }
};

// 8 consecutive 16-bit values (one 16-byte aligned vector) <-> fp32
template <typename T>
__device__ __forceinline__ void load8(const T* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = Half16<T>::unpack(w[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
template <typename T>
__device__ __forceinline__ void store8(T* p, const float (&v)[8]) {
  uint4 o;
  o.x = Half16<T>::pack(v[0], v[1]);
  o.y = Half16<T>::pack(v[2], v[3]);
  o.z = Half16<T>::pack(v[4], v[5]);
  o.w = Half16<T>::pack(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = o;
}
template <typename T>
__device__ __forceinline__ float round16(float v) {
  return Half16<T>::to_f(Half16<T>::from_f(v));
}

__device__ __forceinline__ float gelu_erf(float v) { return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f)); }
// x * sigmoid(x) with ex2.approx + rcp.approx (the IEEE divide made the GroupNorm-apply kernel issue-bound)
__device__ __forceinline__ float silu_f(float v) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * v));
  return __fdividef(v, 1.0f + e);
}

// x * sigmoid(1.702 x): mlx nn.gelu_fast_approx, CLIP's "quick_gelu" (reference mlx/clip.py:11)
__device__ __forceinline__ float quick_gelu_f(float v) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.702f * 1.4426950408889634f * v));
  return __fdividef(v, 1.0f + e);
}

// 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3))): torch's gelu(approximate="tanh"), SigLIP's "gelu_pytorch_tanh".
// The accurate tanhf, not tanh.approx.f32 (relative error about 2^-11), like torch's fp32 tanh.
__device__ __forceinline__ float gelu_tanh_f(float v) {
  const float inner = 0.7978845608028654f * (v + 0.044715f * v * v * v);
  return 0.5f * v * (1.0f + tanhf(inner));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace dk
