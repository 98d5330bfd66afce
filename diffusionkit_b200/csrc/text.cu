// Kernels of the text-encoder path (SURVEY.md §8 row f2): CLIP-L/G and the T5-XXL encoder.  The projections and MLPs
// run on the wgmma GEMM (gemm.cu); this file holds what sits between them: embedding lookup, T5's
// RMSNorm over the fp32 residual stream, the gated-GELU product, and attention for short sequences
// (S <= 512, head dim 64) with CLIP's causal mask or T5's relative-position bias.  All are small next to the denoise
// path (T5-XXL at 512 tokens: 4.3 GFLOP of attention per layer against 0.6 TFLOP of GEMM).
#include "common.cuh"
#include "host.h"

namespace dk {

// ------------------------------------------------------------------------------------------------
// token (+ position) embedding: out[i] = table[ids[i]] (+ pos[i % L])      reference mlx/clip.py:97-98, t5.py:322
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void embedding_kernel(const T* __restrict__ table, const int* __restrict__ ids, const T* __restrict__ pos,
                                 T* __restrict__ out, long long n, int d, int L) {
  const int vpr = d / 8;
  const long long nvec = n * vpr;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / vpr;
    const int c = static_cast<int>(i - r * vpr) * 8;
    float a[8];
    load8(table + static_cast<long long>(ids[r]) * d + c, a);
    if (pos != nullptr) {
      float p[8];
      load8(pos + static_cast<long long>(r % L) * d + c, p);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += p[j];
    }
    store8(out + r * d + c, a);
  }
}

// ------------------------------------------------------------------------------------------------
// T5 RMSNorm over the fp32 residual stream: y = T(w * x * rsqrt(mean(x^2) + eps))     reference mlx/t5.py:150-170
// One 256-thread block per row, row in registers (d <= 4096).
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
rmsnorm_f32_kernel(const float* __restrict__ x, const T* __restrict__ w, T* __restrict__ y, int d, float eps) {
  __shared__ float red[8];
  const long long row = blockIdx.x;
  const float4* xr = reinterpret_cast<const float4*>(x + row * d);
  const int nvec = d / 4;
  float4 v[4];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int vec = threadIdx.x + i * 256;
    if (vec < nvec) {
      v[i] = xr[vec];
      ss += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w;
    }
  }
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = (threadIdx.x & 31) < 8 ? red[threadIdx.x & 31] : 0.f;
  tot = warp_sum(tot);
  const float rstd = rsqrtf(tot / d + eps);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int vec = threadIdx.x + i * 256;
    if (vec < nvec) {
      const uint2 wu = *reinterpret_cast<const uint2*>(w + vec * 4);
      const float2 w01 = Half16<T>::unpack(wu.x), w23 = Half16<T>::unpack(wu.y);
      uint2 o;
      o.x = Half16<T>::pack(w01.x * (v[i].x * rstd), w01.y * (v[i].y * rstd));
      o.y = Half16<T>::pack(w23.x * (v[i].z * rstd), w23.y * (v[i].w * rstd));
      *reinterpret_cast<uint2*>(y + row * d + vec * 4) = o;
    }
  }
}

// x32 += float(y16): the T5 residual stream stays fp32 (reference t5.py:214-221)
template <typename T>
__global__ void add_f32_16_kernel(float* __restrict__ x, const T* __restrict__ y, long long n) {
  const long long nvec = n / 8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float a[8];
    load8(y + i * 8, a);
    float4* xp = reinterpret_cast<float4*>(x + i * 8);
    float4 lo = xp[0], hi = xp[1];
    lo.x += a[0]; lo.y += a[1]; lo.z += a[2]; lo.w += a[3];
    hi.x += a[4]; hi.y += a[5]; hi.z += a[6]; hi.w += a[7];
    xp[0] = lo;
    xp[1] = hi;
  }
}

// gated activation of T5's DenseActivation: out[r, f] = gelu(h[r, f]) * h[r, F + f]   (h = x @ [wi_0 | wi_1]^T)
// reference mlx/t5.py:195-199 with act = nn.gelu (exact erf)
template <typename T>
__global__ void glu_gelu_kernel(const T* __restrict__ h, T* __restrict__ out, long long rows, int F) {
  const int vpr = F / 8;
  const long long nvec = rows * vpr;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / vpr;
    const int c = static_cast<int>(i - r * vpr) * 8;
    float a[8], b[8];
    load8(h + r * 2 * F + c, a);
    load8(h + r * 2 * F + F + c, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = gelu_erf(a[j]) * b[j];
    store8(out + r * F + c, a);
  }
}

// ------------------------------------------------------------------------------------------------
// Attention for short sequences, head dim 64: out = softmax(scale * q k^T + bias) v, scores and probabilities fp32.
//   bias: CLIP's causal mask (-6e4 above the diagonal, mlx/clip.py:84-90) and/or T5's relative-position bias, passed as
//   rel_bias[head][j - i + S - 1] (the bucket of t5.py:21-64 depends on key - query only).
// Grid (ceil(S / 64), heads, B), 8 warps; K^T and V of one (batch, head) staged in shared memory as bf16/fp16 pairs;
// one warp per query row: lanes own keys j = lane + 32 i for q k^T, and the channel pair 2*lane for P V.
// ------------------------------------------------------------------------------------------------
constexpr int AS_MAX_S = 512;
constexpr int AS_NK = AS_MAX_S / 32;
constexpr int AS_QB = 64;

template <typename T>
__global__ void __launch_bounds__(256)
attention_small_kernel(const T* __restrict__ qkv, const T* __restrict__ rel_bias, T* __restrict__ out, int S, int heads,
                       float scale, int causal) {
  extern __shared__ uint32_t as_smem[];
  const int Spad = (S + 31) & ~31;
  const int SP = Spad + 1;                     // row stride of K^T: keeps the transposing stores conflict-free
  uint32_t* kt = as_smem;                      // [32][SP]   word (c2, j) = K[j][2*c2 .. 2*c2+1]
  uint32_t* v2 = as_smem + 32 * SP;            // [Spad][32] word (j, c2) = V[j][2*c2 .. 2*c2+1]
  uint32_t* qs = v2 + Spad * 32;               // [8 warps][32]
  const int h = blockIdx.y, b = blockIdx.z;
  const int ld = 3 * heads * 64;
  const T* base = qkv + static_cast<long long>(b) * S * ld + h * 64;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  for (int idx = tid; idx < Spad * 8; idx += 256) {
    const int j = idx >> 3, part = idx & 7;
    uint4 kw = make_uint4(0u, 0u, 0u, 0u), vw = kw;
    if (j < S) {
      kw = *reinterpret_cast<const uint4*>(base + static_cast<long long>(j) * ld + heads * 64 + part * 8);
      vw = *reinterpret_cast<const uint4*>(base + static_cast<long long>(j) * ld + 2 * heads * 64 + part * 8);
    }
    kt[(part * 4 + 0) * SP + j] = kw.x;
    kt[(part * 4 + 1) * SP + j] = kw.y;
    kt[(part * 4 + 2) * SP + j] = kw.z;
    kt[(part * 4 + 3) * SP + j] = kw.w;
    *reinterpret_cast<uint4*>(v2 + j * 32 + part * 4) = vw;
  }
  __syncthreads();

  const int nk = Spad >> 5;
  for (int rr = warp; rr < AS_QB; rr += 8) {
    const int r = blockIdx.x * AS_QB + rr;
    if (r >= S) break;
    qs[warp * 32 + lane] = *reinterpret_cast<const uint32_t*>(base + static_cast<long long>(r) * ld + 2 * lane);
    __syncwarp();
    float acc[AS_NK];
#pragma unroll
    for (int i = 0; i < AS_NK; ++i) acc[i] = 0.f;
#pragma unroll 4
    for (int c2 = 0; c2 < 32; ++c2) {
      const float2 q = Half16<T>::unpack(qs[warp * 32 + c2]);
      const uint32_t* krow = kt + c2 * SP + lane;
#pragma unroll
      for (int i = 0; i < AS_NK; ++i) {
        if (i < nk) {
          const float2 k = Half16<T>::unpack(krow[32 * i]);
          acc[i] = fmaf(q.x, k.x, fmaf(q.y, k.y, acc[i]));
        }
      }
    }
    float m = -INFINITY;
#pragma unroll
    for (int i = 0; i < AS_NK; ++i) {
      if (i < nk) {
        const int j = lane + 32 * i;
        float s = acc[i] * scale;
        if (rel_bias != nullptr && j < S)
          s += Half16<T>::to_f(rel_bias[static_cast<long long>(h) * (2 * S - 1) + (j - r + S - 1)]);
        if (causal && j > r) s += -6e4f;
        if (j >= S) s = -INFINITY;
        acc[i] = s;
        m = fmaxf(m, s);
      }
    }
    m = warp_max(m);
    float l = 0.f;
#pragma unroll
    for (int i = 0; i < AS_NK; ++i) {
      if (i < nk) {
        acc[i] = __expf(acc[i] - m);
        l += acc[i];
      }
    }
    l = warp_sum(l);
    float o0 = 0.f, o1 = 0.f;
#pragma unroll
    for (int i = 0; i < AS_NK; ++i) {
      if (i < nk) {
        const int jn = min(32, S - 32 * i);
        for (int t = 0; t < jn; ++t) {
          const float p = __shfl_sync(0xffffffffu, acc[i], t);
          const float2 v = Half16<T>::unpack(v2[(32 * i + t) * 32 + lane]);
          o0 = fmaf(p, v.x, o0);
          o1 = fmaf(p, v.y, o1);
        }
      }
    }
    const float inv = 1.f / l;
    *reinterpret_cast<uint32_t*>(out + (static_cast<long long>(b) * S + r) * heads * 64 + h * 64 + 2 * lane) =
        Half16<T>::pack(o0 * inv, o1 * inv);
    __syncwarp();
  }
}

// K^T [32][Spad + 1], V [Spad][32] and the query rows of the 8 warps, in 32-bit words
static inline int as_smem_bytes(int S) {
  const int Spad = (S + 31) & ~31;
  return (32 * (Spad + 1) + Spad * 32 + 8 * 32) * 4;
}

}  // namespace dk

using namespace dk;

extern "C" int dk_embedding(dk_ctx* ctx, int dtype, const void* table, const int* ids, const void* pos, void* out,
                            long long n, int d, int vocab, int pos_len, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(n > 0 && d > 0 && d % 8 == 0, "dk_embedding: d (%d) must be a positive multiple of 8", d);
  DK_REQUIRE(vocab > 0, "dk_embedding: empty table");
  DK_REQUIRE(pos == nullptr || pos_len > 0, "dk_embedding: position table without a length");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (embedding_kernel<T><<<dk_grid_for(n * (d / 8), 256, ctx->sm_count), 256, 0, stream>>>(
                         static_cast<const T*>(table), ids, static_cast<const T*>(pos), static_cast<T*>(out), n, d,
                         pos_len > 0 ? pos_len : 1)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_rmsnorm_f32(dk_ctx* ctx, int dtype, const float* x, const void* weight, void* y, int rows, int d,
                              float eps, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(rows > 0 && d > 0 && d % 4 == 0 && d <= 4096, "dk_rmsnorm_f32: d (%d) must be a multiple of 4, <= 4096", d);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (rmsnorm_f32_kernel<T><<<rows, 256, 0, stream>>>(x, static_cast<const T*>(weight),
                                                                       static_cast<T*>(y), d, eps)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_add_f32_16(dk_ctx* ctx, int dtype, float* x, const void* y, long long n, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(n % 8 == 0, "dk_add_f32_16: n must be a multiple of 8");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (add_f32_16_kernel<T><<<dk_grid_for(n / 8, 256, ctx->sm_count), 256, 0, stream>>>(
                         x, static_cast<const T*>(y), n)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_glu_gelu(dk_ctx* ctx, int dtype, const void* h, void* out, long long rows, int F, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(rows > 0 && F > 0 && F % 8 == 0, "dk_glu_gelu: F (%d) must be a positive multiple of 8", F);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (glu_gelu_kernel<T><<<dk_grid_for(rows * (F / 8), 256, ctx->sm_count), 256, 0, stream>>>(
                         static_cast<const T*>(h), static_cast<T*>(out), rows, F)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_attention_small(dk_ctx* ctx, int dtype, const void* qkv, const void* rel_bias, void* out, int B, int S,
                                  int heads, int head_dim, float scale, int causal, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(head_dim == 64, "dk_attention_small: head dim %d unsupported (64)", head_dim);
  DK_REQUIRE(B > 0 && heads > 0 && S > 0 && S <= AS_MAX_S, "dk_attention_small: S (%d) must be in [1, %d]", S, AS_MAX_S);
  DK_REQUIRE(dk_aligned16(qkv), "dk_attention_small: qkv must be 16-byte aligned");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const dim3 grid(dk_ceil_div(S, AS_QB), heads, B);
  DK_DISPATCH(dtype, {
    auto kern = attention_small_kernel<T>;
    if (int rc = dk_kernel_smem(ctx, reinterpret_cast<const void*>(kern), as_smem_bytes(AS_MAX_S))) return rc;
    kern<<<grid, 256, as_smem_bytes(S), stream>>>(static_cast<const T*>(qkv), static_cast<const T*>(rel_bias),
                                                  static_cast<T*>(out), S, heads, scale, causal);
  });
  DK_LAUNCH_CHECK(ctx);
  return 0;
}
