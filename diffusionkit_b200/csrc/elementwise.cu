// HBM-bound kernels of the denoise + decode path: normalisations, modulation, RoPE, layout shuffles, sampler update.
// All of them move 128-bit vectors per thread, reduce with warp shuffles, and do their arithmetic in fp32.
#include <cuda_fp8.h>

#include "common.cuh"
#include "host.h"

namespace dk {

// block-wide sum for blockDim.x = NT (multiple of 32); every thread gets the result
template <int NT>
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (lane < NT / 32) ? red[lane] : 0.f;
  t = warp_sum(t);
  return t;
}
template <int NT>
__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (lane < NT / 32) ? red[lane] : -INFINITY;
  t = warp_max(t);
  return t;
}

// ------------------------------------------------------------------------------------------------
// K2: LayerNorm, mlx.fast.layer_norm semantics: biased variance, fp32 accumulation, (x-mu)*rsqrt(var+eps)*w + b.
//   MODULATE: no affine of its own, adaLN modulate w = 1 + scale, b = shift of the row's batch
//             (reference mlx/mmdit.py:958-972);
//   otherwise the learned affine w = scale, b = shift of nn.LayerNorm, the same for every row (mlx/clip.py:32-33,78).
// ------------------------------------------------------------------------------------------------
constexpr int LN_WARPS = 4;     // rows per block
constexpr int LN_MAXV = 16;     // h <= 32 lanes * 8 * 16 = 4096

// Row quantisation to e4m3: scale = amax(|row|) / 448 (1 for an all-zero row), q = cvt.rn.satfinite.e4m3(v / scale), all
// in fp32 with IEEE division, so the result is a function of the row alone.
__device__ __forceinline__ float e4m3_row_scale(float amax) { return amax > 0.f ? __fdiv_rn(amax, 448.0f) : 1.0f; }
// 8 consecutive values -> 8 e4m3 bytes, one 64-bit store
__device__ __forceinline__ void store8_e4m3(uint8_t* p, const float (&v)[8], float scale) {
  uint32_t w[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    uint32_t b[2];
#pragma unroll
    for (int j = 0; j < 2; ++j)
      b[j] = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(v[4 * k + 2 * j], scale), __fdiv_rn(v[4 * k + 2 * j + 1], scale)),
                                      __NV_SATFINITE, __NV_E4M3);
    w[k] = b[0] | (b[1] << 16);
  }
  *reinterpret_cast<uint2*>(p) = make_uint2(w[0], w[1]);
}
// A row held by one warp in registers (vector lane + 32 i of nvec) whose lanes know their own maximum -> e4m3 + scale
template <int NV>
__device__ __forceinline__ void store_row_e4m3(const float (&v)[NV][8], float lane_amax, int nvec, int lane,
                                               uint8_t* qr, float* scale_out) {
  const float sc = e4m3_row_scale(warp_max(lane_amax));
  if (lane == 0) *scale_out = sc;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vec = lane + i * 32;
    if (vec < nvec) store8_e4m3(qr + vec * 8, v[i], sc);
  }
}

// One warp per row: the row lives in registers (<= 16 x 128-bit loads in flight per lane), statistics via warp
// shuffles only — no shared memory, no block barriers.  Q8: the fp32 result row is not rounded to 16 bits but
// quantised to e4m3 (q, qscale[row]) while it is still in registers.
template <typename T, int NV, bool MODULATE, bool Q8>
__global__ void __launch_bounds__(LN_WARPS * 32)
layernorm_kernel(const T* __restrict__ x, T* __restrict__ y, const T* __restrict__ shift, const T* __restrict__ scale,
                 long long mod_ld, int rows, int rows_per_batch, int h, float eps, uint8_t* __restrict__ q8,
                 float* __restrict__ qscale) {
  const int row = blockIdx.x * LN_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const T* xr = x + static_cast<long long>(row) * h;
  T* yr = y + static_cast<long long>(row) * h;
  const int nvec = h / 8;
  float v[NV][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vec = lane + i * 32;
    if (vec < nvec) {
      load8(xr + vec * 8, v[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[i][j];
    }
  }
  const float mean = warp_sum(s) / h;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vec = lane + i * 32;
    if (vec < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[i][j] - mean;
        q += d * d;
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / h + eps);
  const T* sh = shift;
  const T* sc = scale;
  if (MODULATE) {
    const int b = row / rows_per_batch;
    sh += static_cast<long long>(b) * mod_ld;
    sc += static_cast<long long>(b) * mod_ld;
  }
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vec = lane + i * 32;
    if (vec < nvec) {
      float a[8], c[8], o[8];
      load8(sc + vec * 8, a);
      load8(sh + vec * 8, c);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        o[j] = MODULATE ? (v[i][j] - mean) * rstd * (1.0f + a[j]) + c[j] : (v[i][j] - mean) * rstd * a[j] + c[j];
      if (Q8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          v[i][j] = o[j];
          amax = fmaxf(amax, fabsf(o[j]));
        }
      } else {
        store8(yr + vec * 8, o);
      }
    }
  }
  if (Q8) store_row_e4m3<NV>(v, amax, nvec, lane, q8 + static_cast<long long>(row) * h, qscale + row);
}

// y: 16-bit output, or with Q8 the e4m3 output whose row scales go to qscale
template <typename T, bool MODULATE, bool Q8 = false>
static void launch_layernorm(const void* x, void* y, const void* shift, const void* scale, long long mod_ld, int rows,
                             int rows_per_batch, int h, float eps, cudaStream_t stream, float* qscale = nullptr) {
  const int blocks = dk_ceil_div(rows, LN_WARPS);
  const int nv = dk_ceil_div(h / 8, 32);   // vectors per lane
  auto kern = nv <= 4 ? layernorm_kernel<T, 4, MODULATE, Q8>
              : nv <= 8 ? layernorm_kernel<T, 8, MODULATE, Q8>
              : nv <= 12 ? layernorm_kernel<T, 12, MODULATE, Q8>
              : layernorm_kernel<T, 16, MODULATE, Q8>;
  kern<<<blocks, LN_WARPS * 32, 0, stream>>>(static_cast<const T*>(x), Q8 ? nullptr : static_cast<T*>(y),
                                             static_cast<const T*>(shift), static_cast<const T*>(scale), mod_ld, rows,
                                             rows_per_batch, h, eps, Q8 ? static_cast<uint8_t*>(y) : nullptr, qscale);
}

// ------------------------------------------------------------------------------------------------
// Row quantiser to e4m3 (weights by output feature, activations by token).  One warp per row: rows of up to
// 32 * 8 * LN_MAXV columns are read once and held in registers, wider rows (the [attn | GELU(fc1)] buffer) are read a
// second time for the conversion.
// ------------------------------------------------------------------------------------------------
template <typename T, int NV>
__global__ void __launch_bounds__(LN_WARPS * 32)
quantize_rows_e4m3_kernel(const T* __restrict__ x, long long ldx, uint8_t* __restrict__ q, float* __restrict__ scale,
                          int rows, int cols) {
  const int row = blockIdx.x * LN_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const T* xr = x + static_cast<long long>(row) * ldx;
  uint8_t* qr = q + static_cast<long long>(row) * cols;
  const int nvec = cols / 8;
  float amax = 0.f;
  if (NV > 0) {
    float v[NV > 0 ? NV : 1][8];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vec = lane + i * 32;
      if (vec < nvec) {
        load8(xr + vec * 8, v[i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(v[i][j]));
      }
    }
    store_row_e4m3<(NV > 0 ? NV : 1)>(v, amax, nvec, lane, qr, scale + row);
  } else {
    float v[8];
    for (int vec = lane; vec < nvec; vec += 32) {
      load8(xr + vec * 8, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(v[j]));
    }
    const float sc = e4m3_row_scale(warp_max(amax));
    if (lane == 0) scale[row] = sc;
    for (int vec = lane; vec < nvec; vec += 32) {
      load8(xr + vec * 8, v);
      store8_e4m3(qr + vec * 8, v, sc);
    }
  }
}

template <typename T>
static void launch_quantize_rows(const void* x, long long ldx, void* q, float* scale, int rows, int cols,
                                 cudaStream_t stream) {
  const int nv = dk_ceil_div(cols / 8, 32);   // vectors per lane
  auto kern = nv <= 4 ? quantize_rows_e4m3_kernel<T, 4>
              : nv <= 8 ? quantize_rows_e4m3_kernel<T, 8>
              : nv <= 12 ? quantize_rows_e4m3_kernel<T, 12>
              : nv <= LN_MAXV ? quantize_rows_e4m3_kernel<T, 16>
              : quantize_rows_e4m3_kernel<T, 0>;
  kern<<<dk_ceil_div(rows, LN_WARPS), LN_WARPS * 32, 0, stream>>>(static_cast<const T*>(x), ldx, static_cast<uint8_t*>(q),
                                                                  scale, rows, cols);
}

// ------------------------------------------------------------------------------------------------
// QK-RMSNorm + RoPE, in place on the q and k thirds of the packed QKV buffer.  One warp per (row, head, q|k).
// ------------------------------------------------------------------------------------------------
template <typename T, int D>
__global__ void __launch_bounds__(256)
qk_norm_rope_kernel(T* __restrict__ qkv, int rows, int S, int heads, int split, const T* __restrict__ q_w,
                    const T* __restrict__ k_w, const T* __restrict__ q_w2, const T* __restrict__ k_w2,
                    const float* __restrict__ rope, float eps) {
  constexpr int EPL = D / 32;  // elements per lane: 2 (d=64) or 4 (d=128)
  const long long gw = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long total = static_cast<long long>(rows) * heads * 2;
  if (gw >= total) return;
  const int which = static_cast<int>(gw % 2);  // 0 = q, 1 = k
  const int head = static_cast<int>((gw / 2) % heads);
  const long long row = gw / (2LL * heads);
  const int pos = static_cast<int>(row % S);
  const int h = heads * D;
  T* p = qkv + row * (3LL * h) + static_cast<long long>(which) * h + head * D + lane * EPL;

  float v[EPL];
  if (EPL == 4) {
    const uint2 u = *reinterpret_cast<const uint2*>(p);
    const float2 a = Half16<T>::unpack(u.x), b = Half16<T>::unpack(u.y);
    v[0] = a.x;
    v[1] = a.y;
    v[EPL - 2] = b.x;
    v[EPL - 1] = b.y;
  } else {
    const uint32_t u = *reinterpret_cast<const uint32_t*>(p);
    const float2 a = Half16<T>::unpack(u);
    v[0] = a.x;
    v[1] = a.y;
  }
  const T* w = (pos < split) ? (which == 0 ? q_w : k_w) : (which == 0 ? q_w2 : k_w2);
  if (w != nullptr) {
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < EPL; ++i) ss += v[i] * v[i];
    ss = warp_sum(ss);
    const float rstd = rsqrtf(ss / D + eps);
#pragma unroll
    for (int i = 0; i < EPL; ++i)
      v[i] = round16<T>(v[i] * rstd * Half16<T>::to_f(w[lane * EPL + i]));  // nn.RMSNorm output in the activation dtype
  }
  if (rope != nullptr) {
    // rope[pos][pair] = (cos, sin); out = (x0 cos - x1 sin, x0 sin + x1 cos)  — mlx/mmdit.py:934-942
    const float* rp = rope + (static_cast<long long>(pos) * (D / 2) + lane * (EPL / 2)) * 2;
#pragma unroll
    for (int i = 0; i < EPL / 2; ++i) {
      const float c = rp[2 * i], sn = rp[2 * i + 1];
      const float x0 = v[2 * i], x1 = v[2 * i + 1];
      v[2 * i] = x0 * c - x1 * sn;
      v[2 * i + 1] = x0 * sn + x1 * c;
    }
  }
  if (EPL == 4) {
    uint2 o;
    o.x = Half16<T>::pack(v[0], v[1]);
    o.y = Half16<T>::pack(v[EPL - 2], v[EPL - 1]);
    *reinterpret_cast<uint2*>(p) = o;
  } else {
    *reinterpret_cast<uint32_t*>(p) = Half16<T>::pack(v[0], v[1]);
  }
}

// ------------------------------------------------------------------------------------------------
// small elementwise kernels (grid-stride over 8-element vectors)
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void silu_add_kernel(const T* __restrict__ y, const T* __restrict__ temb, T* __restrict__ c, int n_t, int B,
                                int h) {
  const long long nvec = static_cast<long long>(n_t) * B * h / 8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long e = i * 8;
    const int col = static_cast<int>(e % h);
    const long long row = e / h;
    const int b = static_cast<int>(row % B);
    const int t = static_cast<int>(row / B);
    float a[8], d[8], o[8];
    load8(y + static_cast<long long>(b) * h + col, a);
    load8(temb + static_cast<long long>(t) * h + col, d);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = silu_f(round16<T>(a[j] + d[j]));
    store8(c + e, o);
  }
}

template <typename T>
__global__ void act_kernel(const T* __restrict__ x, T* __restrict__ y, long long n, int act) {
  const long long nvec = n / 8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float a[8];
    load8(x + i * 8, a);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      a[j] = act == DK_ACT_SILU ? silu_f(a[j])
             : act == DK_ACT_GELU_ERF ? gelu_erf(a[j])
             : act == DK_ACT_QUICK_GELU ? quick_gelu_f(a[j])
             : act == DK_ACT_GELU_TANH ? gelu_tanh_f(a[j])
             : a[j];
    store8(y + i * 8, a);
  }
}

// patchify / unpatchify: one thread per (token, output feature)
template <typename T>
__global__ void patchify_kernel(const T* __restrict__ latent, T* __restrict__ rows, int B, int H, int W, int C,
                                int order) {
  const int F = 4 * C;
  const long long total = static_cast<long long>(B) * (H / 2) * (W / 2) * F;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int f = static_cast<int>(i % F);
    const long long tok = i / F;
    const int wp = static_cast<int>(tok % (W / 2));
    const int hp = static_cast<int>((tok / (W / 2)) % (H / 2));
    const int b = static_cast<int>(tok / (static_cast<long long>(W / 2) * (H / 2)));
    int c, ph, pw;
    if (order == 0) {  // (c, ph, pw)
      c = f / 4;
      ph = (f / 2) % 2;
      pw = f % 2;
    } else {  // (ph, pw, c)
      ph = f / (2 * C);
      pw = (f / C) % 2;
      c = f % C;
    }
    rows[i] = latent[((static_cast<long long>(b) * H + 2 * hp + ph) * W + 2 * wp + pw) * C + c];
  }
}
template <typename T>
__global__ void unpatchify_kernel(const T* __restrict__ rows, T* __restrict__ latent, int B, int H, int W, int C,
                                  int order) {
  const int F = 4 * C;
  const long long total = static_cast<long long>(B) * H * W * C;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    const int x = static_cast<int>((i / C) % W);
    const int y = static_cast<int>((i / (static_cast<long long>(C) * W)) % H);
    const int b = static_cast<int>(i / (static_cast<long long>(C) * W * H));
    const int ph = y & 1, pw = x & 1;
    const long long tok = (static_cast<long long>(b) * (H / 2) + y / 2) * (W / 2) + x / 2;
    const int f = order == 0 ? (c * 4 + ph * 2 + pw) : ((ph * 2 + pw) * C + c);
    latent[i] = rows[tok * F + f];
  }
}

template <typename T>
__global__ void pos_embed_crop_kernel(const T* __restrict__ table, T* __restrict__ out, int max_hw, int hp, int wp,
                                      int h) {
  const int y0 = (max_hw - hp) / 2, x0 = (max_hw - wp) / 2;
  const long long nvec = static_cast<long long>(hp) * wp * h / 8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long e = i * 8;
    const int col = static_cast<int>(e % h);
    const long long tok = e / h;
    const int xx = static_cast<int>(tok % wp), yy = static_cast<int>(tok / wp);
    *reinterpret_cast<uint4*>(out + e) =
        *reinterpret_cast<const uint4*>(table + (static_cast<long long>(y0 + yy) * max_hw + x0 + xx) * h + col);
  }
}

template <typename T>
__global__ void copy_rows_kernel(const T* __restrict__ src, T* __restrict__ dst, int B, int rows, int h, int dst_rows,
                                 int dst_off, int src_rows, int src_off) {
  const long long nvec = static_cast<long long>(B) * rows * h / 8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long e = i * 8;
    const int col = static_cast<int>(e % h);
    const long long rr = e / h;
    const int r = static_cast<int>(rr % rows);
    const int b = static_cast<int>(rr / rows);
    *reinterpret_cast<uint4*>(dst + (static_cast<long long>(b) * dst_rows + dst_off + r) * h + col) =
        *reinterpret_cast<const uint4*>(src + (static_cast<long long>(b) * src_rows + src_off + r) * h + col);
  }
}

// ------------------------------------------------------------------------------------------------
// sampler (fp32 state) — reference mlx/__init__.py:691-719, 775-782; mlx/sampler.py:37-39
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void sampler_prepare_kernel(const float* __restrict__ x, T* __restrict__ xin, long long n, int reps) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const T v = Half16<T>::from_f(x[i]);
    for (int k = 0; k < reps; ++k) xin[k * n + i] = v;
  }
}
// The CFG-mixed denoised estimate D of element i, shared by every sampler update.  The negative rows sit n elements
// after the positive ones ([positive x B | negative x B], reference :718).  SLG (skip-layer guidance, DESIGN.md §13):
// a third block of rows at 2n holds the positive rows' forward with joint blocks skipped, and
// D = D_neg + w (D_pos - D_neg) + slg (D_pos - D_skip).  The entry points refuse SLG without CFG.
template <bool SLG, typename T>
__device__ __forceinline__ float cfg_denoised(const T* __restrict__ xin, const T* __restrict__ out, long long n,
                                              long long i, float sigma, float cfg, float slg) {
  // calculate_denoised: model_input - model_output * sigma (fp32 sigma promotes to fp32)
  float den = Half16<T>::to_f(xin[i]) - Half16<T>::to_f(out[i]) * sigma;
  if (cfg > 0.f) {
    const float den_pos = den;
    const float den_neg = Half16<T>::to_f(xin[n + i]) - Half16<T>::to_f(out[n + i]) * sigma;
    den = den_neg + cfg * (den_pos - den_neg);
    if constexpr (SLG) {
      const float den_skip = Half16<T>::to_f(xin[2 * n + i]) - Half16<T>::to_f(out[2 * n + i]) * sigma;
      den += slg * (den_pos - den_skip);
    }
  }
  return den;
}
template <typename T, bool SLG>
__global__ void sampler_step_kernel(float* __restrict__ x, const T* __restrict__ xin, const T* __restrict__ out,
                                    long long n, float sigma, float sigma_next, float cfg, float slg) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float den = cfg_denoised<SLG>(xin, out, n, i, sigma, cfg, slg);
    const float xv = x[i];
    const float d = (xv - den) / sigma;          // to_d
    x[i] = xv + d * (sigma_next - sigma);        // Euler
  }
}
// Heun predictor (Karras et al. 2022, Alg. 2): the Euler step to x2, keeping its slope d for the corrector; x is
// left as it is.
template <typename T, bool SLG>
__global__ void sampler_heun_predict_kernel(const float* __restrict__ x, const T* __restrict__ xin,
                                            const T* __restrict__ out, float* __restrict__ d, float* __restrict__ x2,
                                            long long n, float sigma, float sigma_next, float cfg, float slg) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float xv = x[i];
    const float dv = (xv - cfg_denoised<SLG>(xin, out, n, i, sigma, cfg, slg)) / sigma;
    d[i] = dv;
    x2[i] = xv + dv * (sigma_next - sigma);
  }
}
// Heun corrector: xin / out are the forward at (x2, sigma_next); x moves by the mean of the two slopes.
template <typename T, bool SLG>
__global__ void sampler_heun_correct_kernel(float* __restrict__ x, const float* __restrict__ d,
                                            const float* __restrict__ x2, const T* __restrict__ xin,
                                            const T* __restrict__ out, long long n, float sigma, float sigma_next,
                                            float cfg, float slg) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float d2 = (x2[i] - cfg_denoised<SLG>(xin, out, n, i, sigma_next, cfg, slg)) / sigma_next;
    x[i] += (d[i] + d2) * 0.5f * (sigma_next - sigma);
  }
}
// DPM-Solver++(2M): x <- a x + b D + c D_prev, then D_prev <- D.  d_prev is not read when c == 0: on the first step
// it holds whatever the allocation held, and 0 * NaN is NaN.
template <typename T, bool SLG>
__global__ void sampler_dpmpp_2m_kernel(float* __restrict__ x, float* __restrict__ d_prev, const T* __restrict__ xin,
                                        const T* __restrict__ out, long long n, float sigma, float a, float b, float c,
                                        float cfg, float slg) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float den = cfg_denoised<SLG>(xin, out, n, i, sigma, cfg, slg);
    float v = a * x[i] + b * den;
    if (c != 0.f) v += c * d_prev[i];
    x[i] = v;
    d_prev[i] = den;
  }
}
// Philox4x32-10 (Salmon et al. 2011, "Parallel random numbers: as easy as 1, 2, 3"): ten rounds of two 32 x 32 -> 64-bit
// multiplies, the key bumped by the Weyl constants between rounds.
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t lo0 = 0xD2511F53u * ctr.x, hi0 = __umulhi(0xD2511F53u, ctr.x);
    const uint32_t lo1 = 0xCD9E8D57u * ctr.z, hi1 = __umulhi(0xCD9E8D57u, ctr.z);
    ctr = make_uint4(hi1 ^ ctr.y ^ k0, lo1, hi0 ^ ctr.w ^ k1, lo0);
  }
  return ctr;
}
// The top 23 bits of a Philox word as ((v >> 9) + 0.5) 2^-23: exact in fp32 and strictly inside (0, 1), so logf is
// finite.  (Taking 24 bits, (k + 0.5) 2^-24 needs 25 significant bits for k >= 2^23 and rounds, up to 1.0 at the top.)
__device__ __forceinline__ float philox_uniform(uint32_t v) {
  return (static_cast<float>(v >> 9) + 0.5f) * 0x1p-23f;
}
// Box-Muller with the accurate logf / sqrtf / sincospif: (r cos 2 pi u_t, r sin 2 pi u_t), r = sqrt(-2 log u_r)
__device__ __forceinline__ float2 box_muller(float u_r, float u_t) {
  const float r = sqrtf(-2.f * logf(u_r));
  float s, c;
  sincospif(2.f * u_t, &s, &c);
  return make_float2(r * c, r * s);
}
// Stochastic samplers (DESIGN.md §16): x <- a x + b D + c D_prev + noise z, then D_prev <- D when d_prev is given.
// Each thread owns 4 consecutive elements e = 4q .. 4q + 3 of image blockIdx.y (n_img elements per image; the rows of
// xin / out sit n = B n_img apart per replica, as cfg_denoised expects).  z comes from one Philox call with counter
// (q, step, 0, 0) and key (lo32(seed), hi32(seed)) of that image's seed: Box-Muller on (u0, u1) gives elements 0 and 1,
// on (u2, u3) elements 2 and 3, so an image's noise depends only on its seed, the step and the element.  With
// noise == 0 nothing is drawn and each element's arithmetic is sampler_dpmpp_2m_kernel's, in the same order.
template <typename T, bool SLG>
__global__ void __launch_bounds__(256) sampler_sde_step_kernel(float* __restrict__ x, float* __restrict__ d_prev,
                                                               const T* __restrict__ xin, const T* __restrict__ out,
                                                               long long n_img, long long n, float sigma, float a,
                                                               float b, float c, float noise, float cfg, float slg,
                                                               const uint64_t* __restrict__ seeds, uint32_t step) {
  const long long img = blockIdx.y;
  uint32_t k0 = 0, k1 = 0;
  if (noise != 0.f) {
    const uint64_t s = seeds[img];
    k0 = static_cast<uint32_t>(s);
    k1 = static_cast<uint32_t>(s >> 32);
  }
  const long long n4 = n_img >> 2;
  for (long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; q < n4;
       q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long i0 = img * n_img + 4 * q;
    float z[4] = {0.f, 0.f, 0.f, 0.f};
    if (noise != 0.f) {
      const uint4 v = philox4x32_10(make_uint4(static_cast<uint32_t>(q), step, 0u, 0u), k0, k1);
      const float2 z01 = box_muller(philox_uniform(v.x), philox_uniform(v.y));
      const float2 z23 = box_muller(philox_uniform(v.z), philox_uniform(v.w));
      z[0] = z01.x, z[1] = z01.y, z[2] = z23.x, z[3] = z23.y;
    }
    const float4 x4 = *reinterpret_cast<const float4*>(x + i0);
    const float xs[4] = {x4.x, x4.y, x4.z, x4.w};
    float ps[4] = {0.f, 0.f, 0.f, 0.f};
    if (c != 0.f) {
      const float4 p4 = *reinterpret_cast<const float4*>(d_prev + i0);
      ps[0] = p4.x, ps[1] = p4.y, ps[2] = p4.z, ps[3] = p4.w;
    }
    float res[4], den[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      den[k] = cfg_denoised<SLG>(xin, out, n, i0 + k, sigma, cfg, slg);
      float v = a * xs[k] + b * den[k];
      if (c != 0.f) v += c * ps[k];
      if (noise != 0.f) v += noise * z[k];
      res[k] = v;
    }
    *reinterpret_cast<float4*>(x + i0) = make_float4(res[0], res[1], res[2], res[3]);
    if (d_prev != nullptr) *reinterpret_cast<float4*>(d_prev + i0) = make_float4(den[0], den[1], den[2], den[3]);
  }
}
// Masked inpainting (DESIGN.md §17), after a solver step to sigma: every latent position the mask keeps (mask byte 0)
// is reset to the re-noised source a eps + b x0 (a = sigma, b = 1 - sigma), rounded as axpby_kernel rounds it,
// fma(a, eps, b x0); a repainted position (mask byte != 0) is neither read nor written.  x, eps, x0 are (B, HW, C)
// fp32 and mask is (HW) uint8; one thread per 4-channel vector of image blockIdx.y, which lies within one position
// since C % 4 == 0 (c4 = C / 4 vectors per position).
__global__ void __launch_bounds__(256) inpaint_blend_kernel(float* __restrict__ x, const float* __restrict__ eps,
                                                            const float* __restrict__ x0,
                                                            const uint8_t* __restrict__ mask, unsigned n4_img,
                                                            unsigned c4, float a, float b) {
  const long long base = static_cast<long long>(blockIdx.y) * n4_img;
  for (unsigned q = blockIdx.x * blockDim.x + threadIdx.x; q < n4_img; q += gridDim.x * blockDim.x) {
    if (mask[q / c4] != 0) continue;
    const float4 e = reinterpret_cast<const float4*>(eps)[base + q];
    const float4 z = reinterpret_cast<const float4*>(x0)[base + q];
    reinterpret_cast<float4*>(x)[base + q] =
        make_float4(__fmaf_rn(a, e.x, __fmul_rn(b, z.x)), __fmaf_rn(a, e.y, __fmul_rn(b, z.y)),
                    __fmaf_rn(a, e.z, __fmul_rn(b, z.z)), __fmaf_rn(a, e.w, __fmul_rn(b, z.w)));
  }
}
// Inpainting paste-back: every pixel of the uint8 (B, P, 3) image whose mask byte is 0 becomes the source's (P, 3)
// pixel.  One thread per 4 pixels = 12 bytes = 3 words of image blockIdx.y; four repainted pixels are left untouched,
// four kept ones are stored without reading the image.
__global__ void __launch_bounds__(256) inpaint_paste_kernel(uint8_t* __restrict__ img, const uint8_t* __restrict__ src,
                                                            const uint8_t* __restrict__ mask, unsigned n4_img) {
  uint32_t* dst = reinterpret_cast<uint32_t*>(img) + 3ll * blockIdx.y * n4_img;
  const uint32_t* from = reinterpret_cast<const uint32_t*>(src);
  for (unsigned q = blockIdx.x * blockDim.x + threadIdx.x; q < n4_img; q += gridDim.x * blockDim.x) {
    const uint32_t m = reinterpret_cast<const uint32_t*>(mask)[q];
    uint32_t keep[3] = {0u, 0u, 0u};  // byte k of the 12 belongs to pixel k / 3
#pragma unroll
    for (int k = 0; k < 12; ++k)
      if (((m >> (8 * (k / 3))) & 0xFFu) == 0u) keep[k / 4] |= 0xFFu << (8 * (k % 4));
    if ((keep[0] | keep[1] | keep[2]) == 0u) continue;
    const bool all = (keep[0] & keep[1] & keep[2]) == 0xFFFFFFFFu;
#pragma unroll
    for (int w = 0; w < 3; ++w) {
      const uint32_t s = from[3ll * q + w];
      dst[3ll * q + w] = all ? s : (dst[3ll * q + w] & ~keep[w]) | (s & keep[w]);
    }
  }
}
__global__ void axpb_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float a, float b) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    y[i] = x[i] * a + b;
}
// MLX affine 4-bit weights (mx.quantize, group_size 64, bits 4; reference nn.quantize call sites mlx/model_io.py:728-734,
// 772-775) -> dense 16-bit: w[n, k] = scales[n, k / group] * q[n, k] + biases[n, k / group], q = nibble (k % 8) of
// word wq[n, k / 8] (element 0 in the low bits).  One thread = one word = 8 outputs = one 16-byte store.
template <typename T>
__global__ void dequant_q4_kernel(const uint32_t* __restrict__ wq, const T* __restrict__ scales,
                                  const T* __restrict__ biases, T* __restrict__ out, long long N, int K, int group) {
  const int wpr = K / 8;  // words per row
  const int gpr = K / group;
  const long long nwords = N * wpr;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nwords;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long n = i / wpr;
    const int k0 = static_cast<int>(i - n * wpr) * 8;
    const uint32_t w = wq[i];
    const float sc = Half16<T>::to_f(scales[n * gpr + k0 / group]);
    const float bi = Half16<T>::to_f(biases[n * gpr + k0 / group]);
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a = __fmaf_rn(sc, static_cast<float>((w >> (8 * j)) & 0xFu), bi);
      const float b = __fmaf_rn(sc, static_cast<float>((w >> (8 * j + 4)) & 0xFu), bi);
      o[j] = Half16<T>::pack(a, b);
    }
    *reinterpret_cast<uint4*>(out + n * K + k0) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// u8 / 255 * 2 - 1 as three separately rounded fp32 ops like the reference's (x / 255) * 2 - 1 (no FMA contraction);
// it is also SigLIP's (x / 255 - 0.5) / 0.5.  dk_image_pre and dk_image_patches both normalise through it.
__device__ __forceinline__ float u8_to_unit(uint8_t u) {
  return __fsub_rn(__fmul_rn(__fdiv_rn(static_cast<float>(u), 255.f), 2.f), 1.f);
}

// read_image (reference mlx/__init__.py:536-551): uint8 [pixels, src_c >= 3] -> 16-bit [pixels, cpad], channels 0..2 =
// u8_to_unit (fp32 arithmetic, then rounded to T), channels 3.. = 0 (the tensor-core conv wants Cin % 64 == 0)
template <typename T>
__global__ void image_pre_kernel(const uint8_t* __restrict__ img, T* __restrict__ out, long long pixels, int src_c,
                                 int cpad) {
  const int vpp = cpad / 8;
  const long long nvec = pixels * vpp;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i / vpp;
    const int v = static_cast<int>(i - p * vpp);
    uint4 w = make_uint4(0u, 0u, 0u, 0u);
    if (v == 0) {
      const uint8_t* px = img + p * src_c;
      w.x = Half16<T>::pack(u8_to_unit(px[0]), u8_to_unit(px[1]));
      w.y = Half16<T>::pack(u8_to_unit(px[2]), 0.f);
    }
    *reinterpret_cast<uint4*>(out + p * cpad + v * 8) = w;
  }
}

// FLUX.1 Fill's masked image (DESIGN.md §18): image_pre_kernel for one (H, W) image whose pixels with a nonzero mask
// byte are written as 0 in every channel, BFL's (x / 255 * 2 - 1) * (1 - mask) with +0 for the masked pixels.  Kept
// pixels round through the same u8_to_unit.  One thread per 8-channel vector of the [pixels, cpad] output.
template <typename T>
__global__ void image_pre_masked_kernel(const uint8_t* __restrict__ img, const uint8_t* __restrict__ mask,
                                        T* __restrict__ out, long long pixels, int src_c, int cpad) {
  const int vpp = cpad / 8;
  const long long nvec = pixels * vpp;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i / vpp;
    const int v = static_cast<int>(i - p * vpp);
    uint4 w = make_uint4(0u, 0u, 0u, 0u);
    if (v == 0 && mask[p] == 0) {
      const uint8_t* px = img + p * src_c;
      w.x = Half16<T>::pack(u8_to_unit(px[0]), u8_to_unit(px[1]));
      w.y = Half16<T>::pack(u8_to_unit(px[2]), 0.f);
    }
    *reinterpret_cast<uint4*>(out + p * cpad + v * 8) = w;
  }
}

// FLUX.1 Fill's conditioning rows (DESIGN.md §18): row n = (h, w) of the (H/16, W/16) token grid gets
// [lat[n, 0:64] | 256 mask channels], 320 columns.  Mask channel j = c * 4 + ph * 2 + pw with c = ph1 * 8 + pw1 holds
// mask[(2h + ph) * 8 + ph1, (2w + pw) * 8 + pw1] != 0 as 1 or 0: BFL's "b (h ph1) (w pw1) -> b (ph1 pw1) h w" then
// "b c (h ph) (w pw) -> b (h w) (c ph pw)".  One thread per 8-column output vector (40 per row): vectors 0-7 copy the
// latent, vector 8 + q holds channels c = 2q and 2q + 1.
template <typename T>
__global__ void fill_cond_rows_kernel(const T* __restrict__ lat, const uint8_t* __restrict__ mask, T* __restrict__ out,
                                      int H, int W) {
  const int wt = W / 16;
  const long long nvec = static_cast<long long>(H / 16) * wt * 40;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / 40;
    const int v = static_cast<int>(i - row * 40);
    uint4 o;
    if (v < 8) {
      o = *reinterpret_cast<const uint4*>(lat + row * 64 + v * 8);
    } else {
      const int h = static_cast<int>(row / wt), w = static_cast<int>(row - static_cast<long long>(h) * wt);
      float m[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int c = 2 * (v - 8) + k / 4, ph = (k >> 1) & 1, pw = k & 1;
        const long long y = (2 * h + ph) * 8 + (c >> 3), x = (2 * w + pw) * 8 + (c & 7);
        m[k] = mask[y * W + x] != 0 ? 1.f : 0.f;
      }
      o.x = Half16<T>::pack(m[0], m[1]);
      o.y = Half16<T>::pack(m[2], m[3]);
      o.z = Half16<T>::pack(m[4], m[5]);
      o.w = Half16<T>::pack(m[6], m[7]);
    }
    *reinterpret_cast<uint4*>(out + row * 320 + v * 8) = o;
  }
}

// Patch rows of a stride-p, p x p, unpadded convolution (SigLIP's patch embedding): uint8 NHWC [B, H, W, src_c >= 3] ->
// 16-bit [B * (H / p) * (W / p), kp].  Column k < 3p^2 of the row of patch (hp, wp) is u8_to_unit of channel k % 3 of
// pixel (hp * p + k / (3p), wp * p + (k / 3) % p), i.e. (kh, kw, c) order; columns 3p^2.. are zero.  The floor of H / p
// and W / p drops the last pixel rows and columns, as the convolution does.  One thread per 8-column vector.
template <typename T>
__global__ void image_patches_kernel(const uint8_t* __restrict__ img, T* __restrict__ out, int B, int H, int W,
                                     int src_c, int p, int kp) {
  const int hp_n = H / p, wp_n = W / p, vpr = kp / 8, kreal = 3 * p * p;
  const long long nvec = static_cast<long long>(B) * hp_n * wp_n * vpr;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / vpr;
    const int v = static_cast<int>(i - row * vpr);
    const int wp = static_cast<int>(row % wp_n);
    const int hp = static_cast<int>((row / wp_n) % hp_n);
    const int b = static_cast<int>(row / (static_cast<long long>(wp_n) * hp_n));
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = v * 8 + j;
      o[j] = 0.f;
      if (k < kreal) {
        const int kh = k / (3 * p), kw = (k / 3) % p, c = k % 3;
        const long long px = (static_cast<long long>(b) * H + hp * p + kh) * W + wp * p + kw;
        o[j] = u8_to_unit(img[px * src_c + c]);
      }
    }
    store8(out + row * kp + v * 8, o);
  }
}
__global__ void axpby_kernel(const float* __restrict__ x, const float* __restrict__ y, float* __restrict__ o,
                             long long n, float a, float b) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    o[i] = a * x[i] + b * y[i];
}
// VAE encoder posterior sample (reference mlx/__init__.py:586-594) + latent_format.process_in (:729-730):
//   hidden [pixels, 2C] = (mean | logvar); z = mean + exp(0.5 * clip(logvar, -30, 20)) * noise; out = (z - shift) * scale
template <typename T>
__global__ void vae_sample_latent_kernel(const T* __restrict__ hidden, const float* __restrict__ noise,
                                         float* __restrict__ out, long long pixels, int C, float shift, float scale) {
  const long long n = pixels * C;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i / C;
    const int c = static_cast<int>(i - p * C);
    const float mean = Half16<T>::to_f(hidden[p * 2 * C + c]);
    const float logvar = fminf(fmaxf(Half16<T>::to_f(hidden[p * 2 * C + C + c]), -30.f), 20.f);
    const float z = mean + __expf(0.5f * logvar) * noise[i];
    out[i] = (z - shift) * scale;
  }
}
template <typename T>
__global__ void cast_f32_to_16_kernel(const float* __restrict__ x, T* __restrict__ y, long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    y[i] = Half16<T>::from_f(x[i]);
}
template <typename T>
__global__ void cast_16_to_f32_kernel(const T* __restrict__ x, float* __restrict__ y, long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    y[i] = Half16<T>::to_f(x[i]);
}

// ------------------------------------------------------------------------------------------------
// GroupNorm (VAE).  stats: two-stage, deterministic (no atomics across blocks):
//   stage 1: grid (chunks, B); each block reduces its pixel slab to per-group (sum, sumsq) partials
//   stage 2: one thread per (b, g) folds the partials in double and writes (mean, rstd)
// apply: grid (blocks, B); a thread keeps its 8 channels' (scale, shift) in registers and streams pixels.
// ------------------------------------------------------------------------------------------------
constexpr int GN_MAX_CHUNKS = 1024;
constexpr int GN_THREADS = 256;

static inline int gn_chunks(int HW) {
  // >= 64 pixels per block, at most GN_MAX_CHUNKS blocks per image
  int c = (HW + 63) / 64;
  if (c > GN_MAX_CHUNKS) c = GN_MAX_CHUNKS;
  if (c < 1) c = 1;
  return c;
}

template <typename T>
__global__ void __launch_bounds__(GN_THREADS)
groupnorm_partial_kernel(const T* __restrict__ x, float* __restrict__ partial, int HW, int C, int G, int chunks) {
  extern __shared__ float sm[];  // [2*C] channel totals + 2 x [GN_THREADS*8] staging
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int per = (HW + chunks - 1) / chunks;
  const int p0 = chunk * per;
  const int p1 = min(HW, p0 + per);
  const int vec_per_pix = C / 8;
  const int pix_per_iter = GN_THREADS / vec_per_pix;  // C <= 2048
  const int my_vec = threadIdx.x % vec_per_pix;
  const int my_pix = threadIdx.x / vec_per_pix;
  float s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
  if (my_pix < pix_per_iter) {
    const T* base = x + static_cast<long long>(b) * HW * C + my_vec * 8;
    int p = p0 + my_pix;
    // four independent 128-bit loads in flight per thread (HBM latency hiding)
    for (; p + 3 * pix_per_iter < p1; p += 4 * pix_per_iter) {
      uint4 u[4];
#pragma unroll
      for (int k = 0; k < 4; ++k)
        u[k] = *reinterpret_cast<const uint4*>(base + static_cast<long long>(p + k * pix_per_iter) * C);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t w[4] = {u[k].x, u[k].y, u[k].z, u[k].w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = Half16<T>::unpack(w[i]);
          s[2 * i] += f.x;
          s[2 * i + 1] += f.y;
          q[2 * i] += f.x * f.x;
          q[2 * i + 1] += f.y * f.y;
        }
      }
    }
    for (; p < p1; p += pix_per_iter) {
      float v[8];
      load8(base + static_cast<long long>(p) * C, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        s[j] += v[j];
        q[j] += v[j] * v[j];
      }
    }
  }
  // deterministic in-block reduction (fixed summation order, no atomics): stage every thread's 8 channel sums as
  // [pixel slot][channel], then one thread per channel folds the pixel slots in order
  float* st_s = sm + 2 * C;                    // [pix_per_iter][C]
  float* st_q = st_s + GN_THREADS * 8;         // [pix_per_iter][C]
  if (my_pix < pix_per_iter) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      st_s[my_pix * C + my_vec * 8 + j] = s[j];
      st_q[my_pix * C + my_vec * 8 + j] = q[j];
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += GN_THREADS) {
    float ts = 0.f, tq = 0.f;
    for (int pp = 0; pp < pix_per_iter; ++pp) {
      ts += st_s[pp * C + c];
      tq += st_q[pp * C + c];
    }
    sm[c] = ts;
    sm[C + c] = tq;
  }
  __syncthreads();
  const int cpg = C / G;
  for (int g = threadIdx.x; g < G; g += GN_THREADS) {
    float ts = 0.f, tq = 0.f;
    for (int c = 0; c < cpg; ++c) {
      ts += sm[g * cpg + c];
      tq += sm[C + g * cpg + c];
    }
    float* dst = partial + ((static_cast<long long>(b) * chunks + chunk) * G + g) * 2;
    dst[0] = ts;
    dst[1] = tq;
  }
}
// one 256-thread block per (b, g): threads stride over the chunk partials four at a time (independent loads in
// flight: with one warp per (b, g) the 8192 partials of a 1024^2 image were a 256-deep chain of dependent-latency
// loads per lane, 45 us per launch x 30 launches = 11 % of a batch-1 decode), accumulation in double; fixed
// thread -> chunk assignment, fixed shuffle tree and fixed cross-warp order: deterministic
constexpr int GNF_THREADS = 256;
__global__ void __launch_bounds__(GNF_THREADS)
groupnorm_finalize_kernel(const float* __restrict__ partial, float* __restrict__ stats, int B, int G, int chunks,
                          double count, float eps) {
  const int idx = blockIdx.x;   // b * G + g
  const int b = idx / G, g = idx % G;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const float2* base = reinterpret_cast<const float2*>(partial) + static_cast<long long>(b) * chunks * G + g;
  double s = 0.0, q = 0.0;
  int c = t;
  for (; c + 3 * GNF_THREADS < chunks; c += 4 * GNF_THREADS) {
    const float2 p0 = base[static_cast<long long>(c) * G];
    const float2 p1 = base[static_cast<long long>(c + GNF_THREADS) * G];
    const float2 p2 = base[static_cast<long long>(c + 2 * GNF_THREADS) * G];
    const float2 p3 = base[static_cast<long long>(c + 3 * GNF_THREADS) * G];
    s += (static_cast<double>(p0.x) + p1.x) + (static_cast<double>(p2.x) + p3.x);
    q += (static_cast<double>(p0.y) + p1.y) + (static_cast<double>(p2.y) + p3.y);
  }
  for (; c < chunks; c += GNF_THREADS) {
    const float2 p = base[static_cast<long long>(c) * G];
    s += p.x;
    q += p.y;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  __shared__ double red[2][GNF_THREADS / 32];
  if (lane == 0) {
    red[0][warp] = s;
    red[1][warp] = q;
  }
  __syncthreads();
  if (t == 0) {
    double ss = 0.0, qq = 0.0;
#pragma unroll
    for (int w = 0; w < GNF_THREADS / 32; ++w) {
      ss += red[0][w];
      qq += red[1][w];
    }
    const double mean = ss / count;
    double var = qq / count - mean * mean;
    if (var < 0.0) var = 0.0;
    stats[idx * 2] = static_cast<float>(mean);
    stats[idx * 2 + 1] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  }
}
template <typename T>
__global__ void __launch_bounds__(GN_THREADS)
groupnorm_apply_kernel(const T* __restrict__ x, T* __restrict__ y, const float* __restrict__ stats,
                       const T* __restrict__ gamma, const T* __restrict__ beta, int HW, int C, int G, int silu) {
  const int b = blockIdx.y;
  const int vec_per_pix = C / 8;
  const int pix_per_iter = GN_THREADS / vec_per_pix;
  const int my_vec = threadIdx.x % vec_per_pix;
  const int my_pix = threadIdx.x / vec_per_pix;
  if (my_pix >= pix_per_iter) return;
  const int cpg = C / G;
  float sc[8], sh[8];
  {
    float ga[8], be[8];
    load8(gamma + my_vec * 8, ga);
    load8(beta + my_vec * 8, be);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int g = (my_vec * 8 + j) / cpg;
      const float mean = stats[(b * G + g) * 2], rstd = stats[(b * G + g) * 2 + 1];
      sc[j] = rstd * ga[j];
      sh[j] = be[j] - mean * rstd * ga[j];
    }
  }
  const long long img = static_cast<long long>(b) * HW * C + my_vec * 8;
  const int step = gridDim.x * pix_per_iter;
  int p = blockIdx.x * pix_per_iter + my_pix;
  // four pixels per iteration: all loads issued before the first use
  for (; p + 3 * step < HW; p += 4 * step) {
    uint4 u[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      u[k] = *reinterpret_cast<const uint4*>(x + img + static_cast<long long>(p + k * step) * C);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t w[4] = {u[k].x, u[k].y, u[k].z, u[k].w};
      float v[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = Half16<T>::unpack(w[i]);
        v[2 * i] = f.x;
        v[2 * i + 1] = f.y;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float o = fmaf(v[j], sc[j], sh[j]);
        if (silu) o = silu_f(round16<T>(o));
        v[j] = o;
      }
      store8(y + img + static_cast<long long>(p + k * step) * C, v);
    }
  }
  for (; p < HW; p += step) {
    float v[8];
    load8(x + img + static_cast<long long>(p) * C, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float o = fmaf(v[j], sc[j], sh[j]);
      if (silu) o = silu_f(round16<T>(o));
      v[j] = o;
    }
    store8(y + img + static_cast<long long>(p) * C, v);
  }
}

// nearest 2x: grid (output rows / rows-per-block, B); a thread owns one 128-bit channel vector of one output column
// and walks output rows — no per-element divisions
template <typename T>
__global__ void __launch_bounds__(256)
upsample2x_kernel(const T* __restrict__ x, T* __restrict__ y, int H, int W, int C, int rows_per_block) {
  const int b = blockIdx.y;
  const int vpp = C / 8;                 // vectors per pixel
  const int row_vecs = 2 * W * vpp;      // vectors per output row
  const int oy0 = blockIdx.x * rows_per_block;
  const int oy1 = min(2 * H, oy0 + rows_per_block);
  const T* xin = x + static_cast<long long>(b) * H * W * C;
  T* yout = y + static_cast<long long>(b) * 4 * H * W * C;
  for (int v = threadIdx.x; v < row_vecs; v += blockDim.x) {
    const int ox = v / vpp;
    const int cv = v - ox * vpp;
    const long long in_col = static_cast<long long>(ox >> 1) * C + cv * 8;
    const long long out_col = static_cast<long long>(ox) * C + cv * 8;
    for (int oy = oy0; oy < oy1; oy += 2) {   // rows oy, oy+1 replicate input row oy/2 (oy0 is even)
      const uint4 u = *reinterpret_cast<const uint4*>(xin + static_cast<long long>(oy >> 1) * W * C + in_col);
      __stcs(reinterpret_cast<uint4*>(yout + static_cast<long long>(oy) * 2 * W * C + out_col), u);
      if (oy + 1 < oy1) __stcs(reinterpret_cast<uint4*>(yout + static_cast<long long>(oy + 1) * 2 * W * C + out_col), u);
    }
  }
}

// row softmax (VAE mid-block attention, reference mlx/vae.py:49-52): p = softmax(scale * s), fp32 math, 16-bit out
template <typename T>
__global__ void __launch_bounds__(256)
softmax_rows_kernel(T* __restrict__ x, int n, long long ld, float scale) {
  __shared__ float red[8];
  T* row = x + static_cast<long long>(blockIdx.x) * ld;
  const int nvec = n / 8;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < nvec; i += 256) {
    float v[8];
    load8(row + i * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) mx = fmaxf(mx, v[j]);
  }
  mx = block_max<256>(mx, red);
  const float k = scale * 1.44269504088896341f;
  float sum = 0.f;
  for (int i = threadIdx.x; i < nvec; i += 256) {
    float v[8];
    load8(row + i * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) sum += exp2f((v[j] - mx) * k);
  }
  sum = block_sum<256>(sum, red);
  const float inv = 1.0f / sum;
  for (int i = threadIdx.x; i < nvec; i += 256) {
    float v[8];
    load8(row + i * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = exp2f((v[j] - mx) * k) * inv;
    store8(row + i * 8, v);
  }
}

// decode tail: clip(x/2 + 0.5, 0, 1) in the activation dtype (mlx/__init__.py:583), uint8 = trunc(x * 255) (:526)
template <typename T>
__global__ void image_post_kernel(const T* __restrict__ x, int c_stride, float* __restrict__ img_f32,
                                  uint8_t* __restrict__ img_u8, long long pixels) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < pixels * 3;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i / 3;
    const int c = static_cast<int>(i % 3);
    float v = Half16<T>::to_f(x[p * c_stride + c]);
    v = round16<T>(round16<T>(v * 0.5f) + 0.5f);
    v = fminf(fmaxf(v, 0.f), 1.f);
    if (img_f32 != nullptr) img_f32[i] = v;
    if (img_u8 != nullptr) img_u8[i] = static_cast<uint8_t>(round16<T>(v * 255.f));
  }
}

// ------------------------------------------------------------------------------------------------
// First-block step cache (DESIGN.md §10).  residual_delta: r = fp32(x) - fp32(base) over nseq sequences of `rows`
// rows; optionally stored to r_out [nseq*rows, h] fp32, and with prev [nseq*rows, h] fp32 the per-sequence sums
// (Σ|r - prev|, Σ|prev|).  Deterministic: grid (chunks, nseq), each block folds its row slab in a fixed thread order
// and a fixed shuffle tree into ws[seq][chunk][2]; residual_delta_finalize folds the chunks of a sequence in a fixed
// order in double.  No atomics, so two launches are bit-identical.
// ------------------------------------------------------------------------------------------------
constexpr int RD_THREADS = 256;
constexpr int RD_MAX_CHUNKS = 256;   // per sequence; ws holds nseq * RD_MAX_CHUNKS * 2 floats

template <typename T>
__global__ void __launch_bounds__(RD_THREADS)
residual_delta_kernel(const T* __restrict__ x, long long ldx, int x_seq_rows, const T* __restrict__ base,
                      long long ldb, int b_seq_rows, float* __restrict__ r_out, const float* __restrict__ prev,
                      float* __restrict__ ws, int rows, int h) {
  __shared__ float red[RD_THREADS / 32];
  const int seq = blockIdx.y, chunk = blockIdx.x, chunks = gridDim.x;
  const int per = (rows + chunks - 1) / chunks;
  const int r0 = chunk * per, r1 = min(rows, r0 + per);
  const int vpr = h / 8;   // vectors per row
  const long long nvec = r1 > r0 ? static_cast<long long>(r1 - r0) * vpr : 0;
  float s_diff = 0.f, s_prev = 0.f;
  for (long long i = threadIdx.x; i < nvec; i += RD_THREADS) {
    const int r = r0 + static_cast<int>(i / vpr);
    const int col = static_cast<int>(i % vpr) * 8;
    float a[8], b[8];
    load8(x + (static_cast<long long>(seq) * x_seq_rows + r) * ldx + col, a);
    load8(base + (static_cast<long long>(seq) * b_seq_rows + r) * ldb + col, b);
    const long long o = (static_cast<long long>(seq) * rows + r) * h + col;
    float d[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] = a[j] - b[j];
    if (r_out != nullptr) {
      float4* p = reinterpret_cast<float4*>(r_out + o);
      p[0] = make_float4(d[0], d[1], d[2], d[3]);
      p[1] = make_float4(d[4], d[5], d[6], d[7]);
    }
    if (prev != nullptr) {
      const float4 p0 = reinterpret_cast<const float4*>(prev + o)[0];
      const float4 p1 = reinterpret_cast<const float4*>(prev + o)[1];
      const float pv[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        s_diff += fabsf(d[j] - pv[j]);
        s_prev += fabsf(pv[j]);
      }
    }
  }
  if (prev == nullptr) return;   // uniform across the block
  s_diff = block_sum<RD_THREADS>(s_diff, red);
  s_prev = block_sum<RD_THREADS>(s_prev, red);
  if (threadIdx.x == 0) {
    float* dst = ws + (static_cast<long long>(seq) * chunks + chunk) * 2;
    dst[0] = s_diff;
    dst[1] = s_prev;
  }
}

// one warp per sequence: lanes stride over the chunk partials, then a fixed shuffle tree, all in double
__global__ void residual_delta_finalize_kernel(const float* __restrict__ ws, float* __restrict__ sums, int nseq,
                                               int chunks) {
  const int seq = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (seq >= nseq) return;
  const float2* p = reinterpret_cast<const float2*>(ws) + static_cast<long long>(seq) * chunks;
  double s = 0.0, q = 0.0;
  for (int c = lane; c < chunks; c += 32) {
    const float2 v = p[c];
    s += v.x;
    q += v.y;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if (lane == 0) {
    sums[seq * 2] = static_cast<float>(s);
    sums[seq * 2 + 1] = static_cast<float>(q);
  }
}

static inline int rd_chunks(int rows, int h, int sm_count, int nseq) {
  // about four 8-element vectors per thread, and about four blocks per SM over the whole batch
  const long long vec = static_cast<long long>(rows) * (h / 8);
  long long c = (vec + RD_THREADS * 4 - 1) / (RD_THREADS * 4);
  const long long fill = (4LL * sm_count + nseq - 1) / nseq;
  if (c > fill) c = fill;
  if (c > rows) c = rows;
  if (c > RD_MAX_CHUNKS) c = RD_MAX_CHUNKS;
  if (c < 1) c = 1;
  return static_cast<int>(c);
}

// out = round16(x + r): one fp32 add, one rounding
template <typename T>
__global__ void residual_apply_kernel(const T* __restrict__ x, const float* __restrict__ r, T* __restrict__ out,
                                      long long n) {
  const long long nvec = n / 8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float a[8];
    load8(x + i * 8, a);
    const float4 r0 = reinterpret_cast<const float4*>(r + i * 8)[0];
    const float4 r1 = reinterpret_cast<const float4*>(r + i * 8)[1];
    a[0] += r0.x;
    a[1] += r0.y;
    a[2] += r0.z;
    a[3] += r0.w;
    a[4] += r1.x;
    a[5] += r1.y;
    a[6] += r1.z;
    a[7] += r1.w;
    store8(out + i * 8, a);
  }
}

}  // namespace dk

using namespace dk;

extern "C" int dk_ln_modulate(dk_ctx* ctx, int dtype, const void* x, void* y, const void* shift, const void* scale,
                              long long mod_ld, int rows, int rows_per_batch, int h, float eps, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(rows > 0 && rows_per_batch > 0, "dk_ln_modulate: empty input");
  DK_REQUIRE(h % 8 == 0 && h <= 32 * 8 * LN_MAXV, "dk_ln_modulate: h=%d unsupported (multiple of 8, <= %d)", h,
             32 * 8 * LN_MAXV);
  DK_REQUIRE(mod_ld % 8 == 0, "dk_ln_modulate: mod_ld must be a multiple of 8");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (launch_layernorm<T, true>(x, y, shift, scale, mod_ld, rows, rows_per_batch, h, eps, stream)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_ln_modulate_fp8(dk_ctx* ctx, int dtype, const void* x, void* q, float* q_scale, const void* shift,
                                  const void* scale, long long mod_ld, int rows, int rows_per_batch, int h, float eps,
                                  void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(rows > 0 && rows_per_batch > 0, "dk_ln_modulate_fp8: empty input");
  DK_REQUIRE(h % 8 == 0 && h <= 32 * 8 * LN_MAXV, "dk_ln_modulate_fp8: h=%d unsupported (multiple of 8, <= %d)", h,
             32 * 8 * LN_MAXV);
  DK_REQUIRE(mod_ld % 8 == 0, "dk_ln_modulate_fp8: mod_ld must be a multiple of 8");
  DK_REQUIRE(q_scale != nullptr, "dk_ln_modulate_fp8: q_scale is required");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (launch_layernorm<T, true, true>(x, q, shift, scale, mod_ld, rows, rows_per_batch, h, eps, stream,
                                                      q_scale)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_quantize_rows_e4m3(dk_ctx* ctx, int dtype, const void* x, long long ldx, void* q, float* q_scale,
                                     int rows, int cols, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(rows > 0 && cols > 0, "dk_quantize_rows_e4m3: empty input");
  DK_REQUIRE(cols % 8 == 0 && ldx % 8 == 0 && ldx >= cols,
             "dk_quantize_rows_e4m3: cols (%d) and ldx (%lld) must be multiples of 8, ldx >= cols", cols, ldx);
  DK_REQUIRE(dk_aligned16(x) && (reinterpret_cast<uintptr_t>(q) & 7u) == 0 && q_scale != nullptr,
             "dk_quantize_rows_e4m3: x must be 16-byte and q 8-byte aligned, q_scale non-null");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (launch_quantize_rows<T>(x, ldx, q, q_scale, rows, cols, stream)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_layernorm(dk_ctx* ctx, int dtype, const void* x, void* y, const void* weight, const void* bias,
                            int rows, int h, float eps, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(rows > 0 && h > 0 && h % 8 == 0 && h <= 32 * 8 * LN_MAXV,
             "dk_layernorm: h (%d) must be a multiple of 8, <= %d", h, 32 * 8 * LN_MAXV);
  DK_REQUIRE(weight != nullptr && bias != nullptr, "dk_layernorm: weight and bias are required");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (launch_layernorm<T, false>(x, y, bias, weight, 0, rows, rows, h, eps, stream)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_qk_norm_rope(dk_ctx* ctx, int dtype, void* qkv, int rows, int S, int heads, int d, int split,
                               const void* q_w, const void* k_w, const void* q_w2, const void* k_w2, const float* rope,
                               float eps, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(d == 64 || d == 128, "dk_qk_norm_rope: head dim %d unsupported (64 or 128)", d);
  DK_REQUIRE(rows > 0 && S > 0 && rows % S == 0, "dk_qk_norm_rope: rows %d must be a multiple of S %d", rows, S);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long warps = static_cast<long long>(rows) * heads * 2;
  const int blocks = static_cast<int>((warps * 32 + 255) / 256);
  if (q_w2 == nullptr) q_w2 = q_w;
  if (k_w2 == nullptr) k_w2 = k_w;
  DK_DISPATCH(dtype, {
    if (d == 128)
      qk_norm_rope_kernel<T, 128><<<blocks, 256, 0, stream>>>(
          static_cast<T*>(qkv), rows, S, heads, split, static_cast<const T*>(q_w), static_cast<const T*>(k_w),
          static_cast<const T*>(q_w2), static_cast<const T*>(k_w2), rope, eps);
    else
      qk_norm_rope_kernel<T, 64><<<blocks, 256, 0, stream>>>(
          static_cast<T*>(qkv), rows, S, heads, split, static_cast<const T*>(q_w), static_cast<const T*>(k_w),
          static_cast<const T*>(q_w2), static_cast<const T*>(k_w2), rope, eps);
  });
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_silu_add(dk_ctx* ctx, int dtype, const void* y, const void* temb, void* c, int n_t, int B, int h,
                           void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(h % 8 == 0, "dk_silu_add: h must be a multiple of 8");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long nvec = static_cast<long long>(n_t) * B * h / 8;
  DK_DISPATCH(dtype, (silu_add_kernel<T><<<dk_grid_for(nvec, 256, ctx->sm_count), 256, 0, stream>>>(
                         static_cast<const T*>(y), static_cast<const T*>(temb), static_cast<T*>(c), n_t, B, h)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_act(dk_ctx* ctx, int dtype, const void* x, void* y, long long n, int act, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(n % 8 == 0, "dk_act: n must be a multiple of 8");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (act_kernel<T><<<dk_grid_for(n / 8, 256, ctx->sm_count), 256, 0, stream>>>(
                         static_cast<const T*>(x), static_cast<T*>(y), n, act)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_patchify(dk_ctx* ctx, int dtype, const void* latent, void* rows, int B, int H, int W, int C, int order,
                           void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(H % 2 == 0 && W % 2 == 0, "dk_patchify: latent size must be even (got %dx%d)", H, W);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long total = static_cast<long long>(B) * H * W * C;
  DK_DISPATCH(dtype, (patchify_kernel<T><<<dk_grid_for(total, 256, ctx->sm_count), 256, 0, stream>>>(
                         static_cast<const T*>(latent), static_cast<T*>(rows), B, H, W, C, order)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_unpatchify(dk_ctx* ctx, int dtype, const void* rows, void* latent, int B, int H, int W, int C,
                             int order, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(H % 2 == 0 && W % 2 == 0, "dk_unpatchify: latent size must be even (got %dx%d)", H, W);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long total = static_cast<long long>(B) * H * W * C;
  DK_DISPATCH(dtype, (unpatchify_kernel<T><<<dk_grid_for(total, 256, ctx->sm_count), 256, 0, stream>>>(
                         static_cast<const T*>(rows), static_cast<T*>(latent), B, H, W, C, order)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_pos_embed_crop(dk_ctx* ctx, int dtype, const void* table, void* out, int max_hw, int hp, int wp, int h,
                                 void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(hp <= max_hw && wp <= max_hw, "dk_pos_embed_crop: %dx%d exceeds the %d table", hp, wp, max_hw);
  DK_REQUIRE(h % 8 == 0, "dk_pos_embed_crop: h must be a multiple of 8");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long nvec = static_cast<long long>(hp) * wp * h / 8;
  DK_DISPATCH(dtype, (pos_embed_crop_kernel<T><<<dk_grid_for(nvec, 256, ctx->sm_count), 256, 0, stream>>>(
                         static_cast<const T*>(table), static_cast<T*>(out), max_hw, hp, wp, h)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_copy_rows(dk_ctx* ctx, int dtype, const void* src, void* dst, int B, int rows, int h, int dst_rows,
                            int dst_off, int src_rows, int src_off, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(h % 8 == 0, "dk_copy_rows: h must be a multiple of 8");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long nvec = static_cast<long long>(B) * rows * h / 8;
  DK_DISPATCH(dtype, (copy_rows_kernel<T><<<dk_grid_for(nvec, 256, ctx->sm_count), 256, 0, stream>>>(
                         static_cast<const T*>(src), static_cast<T*>(dst), B, rows, h, dst_rows, dst_off, src_rows,
                         src_off)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_sampler_prepare(dk_ctx* ctx, int dtype, const float* x, void* xin, long long n_per_rep, int reps,
                                  void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (sampler_prepare_kernel<T><<<dk_grid_for(n_per_rep, 256, ctx->sm_count), 256, 0, stream>>>(
                         x, static_cast<T*>(xin), n_per_rep, reps)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_sampler_step(dk_ctx* ctx, int dtype, float* x, const void* xin, const void* out, long long n,
                               float sigma, float sigma_next, float cfg_weight, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(sigma != 0.f, "dk_sampler_step: sigma must be non-zero");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (sampler_step_kernel<T, false><<<dk_grid_for(n, 256, ctx->sm_count), 256, 0, stream>>>(
                         x, static_cast<const T*>(xin), static_cast<const T*>(out), n, sigma, sigma_next, cfg_weight,
                         0.f)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_sampler_heun_predict(dk_ctx* ctx, int dtype, const float* x, const void* xin, const void* out,
                                       float* d, float* x2, long long n, float sigma, float sigma_next,
                                       float cfg_weight, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(sigma != 0.f, "dk_sampler_heun_predict: sigma must be non-zero");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (sampler_heun_predict_kernel<T, false><<<dk_grid_for(n, 256, ctx->sm_count), 256, 0, stream>>>(
                         x, static_cast<const T*>(xin), static_cast<const T*>(out), d, x2, n, sigma, sigma_next,
                         cfg_weight, 0.f)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_sampler_heun_correct(dk_ctx* ctx, int dtype, float* x, const float* d, const float* x2,
                                       const void* xin, const void* out, long long n, float sigma, float sigma_next,
                                       float cfg_weight, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(sigma_next != 0.f, "dk_sampler_heun_correct: sigma_next must be non-zero (the last step is an Euler step)");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (sampler_heun_correct_kernel<T, false><<<dk_grid_for(n, 256, ctx->sm_count), 256, 0, stream>>>(
                         x, d, x2, static_cast<const T*>(xin), static_cast<const T*>(out), n, sigma, sigma_next,
                         cfg_weight, 0.f)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_sampler_dpmpp_2m(dk_ctx* ctx, int dtype, float* x, float* d_prev, const void* xin, const void* out,
                                   long long n, float sigma, float a, float b, float c, float cfg_weight,
                                   void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (sampler_dpmpp_2m_kernel<T, false><<<dk_grid_for(n, 256, ctx->sm_count), 256, 0, stream>>>(
                         x, d_prev, static_cast<const T*>(xin), static_cast<const T*>(out), n, sigma, a, b, c,
                         cfg_weight, 0.f)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

// The same four updates with skip-layer guidance (DESIGN.md §13): xin / out hold three blocks of n elements,
// [positive | negative | positive with joint blocks skipped], so they need CFG.
#define DK_SLG_REQUIRE(cfg_weight, slg)                                                                     \
  DK_REQUIRE((cfg_weight) > 0.f, "%s: skip-layer guidance needs CFG (cfg_weight > 0)", __func__);          \
  DK_REQUIRE(isfinite(slg), "%s: the skip-layer guidance scale must be finite", __func__)

extern "C" int dk_sampler_step_slg(dk_ctx* ctx, int dtype, float* x, const void* xin, const void* out, long long n,
                                   float sigma, float sigma_next, float cfg_weight, float slg, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(sigma != 0.f, "dk_sampler_step_slg: sigma must be non-zero");
  DK_SLG_REQUIRE(cfg_weight, slg);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (sampler_step_kernel<T, true><<<dk_grid_for(n, 256, ctx->sm_count), 256, 0, stream>>>(
                         x, static_cast<const T*>(xin), static_cast<const T*>(out), n, sigma, sigma_next, cfg_weight,
                         slg)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_sampler_heun_predict_slg(dk_ctx* ctx, int dtype, const float* x, const void* xin, const void* out,
                                           float* d, float* x2, long long n, float sigma, float sigma_next,
                                           float cfg_weight, float slg, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(sigma != 0.f, "dk_sampler_heun_predict_slg: sigma must be non-zero");
  DK_SLG_REQUIRE(cfg_weight, slg);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (sampler_heun_predict_kernel<T, true><<<dk_grid_for(n, 256, ctx->sm_count), 256, 0, stream>>>(
                         x, static_cast<const T*>(xin), static_cast<const T*>(out), d, x2, n, sigma, sigma_next,
                         cfg_weight, slg)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_sampler_heun_correct_slg(dk_ctx* ctx, int dtype, float* x, const float* d, const float* x2,
                                           const void* xin, const void* out, long long n, float sigma,
                                           float sigma_next, float cfg_weight, float slg, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(sigma_next != 0.f,
             "dk_sampler_heun_correct_slg: sigma_next must be non-zero (the last step is an Euler step)");
  DK_SLG_REQUIRE(cfg_weight, slg);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (sampler_heun_correct_kernel<T, true><<<dk_grid_for(n, 256, ctx->sm_count), 256, 0, stream>>>(
                         x, d, x2, static_cast<const T*>(xin), static_cast<const T*>(out), n, sigma, sigma_next,
                         cfg_weight, slg)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_sampler_dpmpp_2m_slg(dk_ctx* ctx, int dtype, float* x, float* d_prev, const void* xin,
                                       const void* out, long long n, float sigma, float a, float b, float c,
                                       float cfg_weight, float slg, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_SLG_REQUIRE(cfg_weight, slg);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (sampler_dpmpp_2m_kernel<T, true><<<dk_grid_for(n, 256, ctx->sm_count), 256, 0, stream>>>(
                         x, d_prev, static_cast<const T*>(xin), static_cast<const T*>(out), n, sigma, a, b, c,
                         cfg_weight, slg)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}
#undef DK_SLG_REQUIRE

extern "C" int dk_sampler_sde_step(dk_ctx* ctx, int dtype, float* x, float* d_prev, const void* xin, const void* out,
                                   long long n_per_image, int B, int reps, float sigma, float a, float b, float c,
                                   float noise, float cfg_weight, float slg, const uint64_t* seeds, int step,
                                   void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(reps >= 1 && reps <= 3, "dk_sampler_sde_step: reps must be 1 (no CFG), 2 (CFG) or 3 (CFG + SLG), got %d",
             reps);
  DK_REQUIRE((reps >= 2) == (cfg_weight > 0.f),
             "dk_sampler_sde_step: reps = %d does not match cfg_weight = %g (CFG needs reps 2 or 3)", reps, cfg_weight);
  DK_REQUIRE(reps == 3 || slg == 0.f, "dk_sampler_sde_step: skip-layer guidance needs reps = 3 (CFG + SLG)");
  DK_REQUIRE(isfinite(sigma) && isfinite(a) && isfinite(b) && isfinite(c) && isfinite(noise) && isfinite(cfg_weight) &&
                 isfinite(slg),
             "dk_sampler_sde_step: sigma, a, b, c, noise, cfg_weight and slg must be finite");
  DK_REQUIRE(d_prev != nullptr || c == 0.f, "dk_sampler_sde_step: c != 0 needs d_prev");
  DK_REQUIRE(noise == 0.f || seeds != nullptr, "dk_sampler_sde_step: noise != 0 needs seeds");
  DK_REQUIRE(B >= 1 && B <= 65535, "dk_sampler_sde_step: B must be in [1, 65535], got %d", B);
  DK_REQUIRE(step >= 0, "dk_sampler_sde_step: step must be >= 0, got %d", step);
  DK_REQUIRE(n_per_image > 0 && n_per_image % 4 == 0 && n_per_image / 4 <= 0xFFFFFFFFll,
             "dk_sampler_sde_step: n_per_image must be a positive multiple of 4 below 2^34, got %lld", n_per_image);
  DK_REQUIRE(dk_aligned16(x) && dk_aligned16(d_prev) && dk_aligned16(xin) && dk_aligned16(out),
             "dk_sampler_sde_step: x, d_prev, xin and out must be 16-byte aligned");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long n = n_per_image * B;
  const dim3 grid(dk_grid_for(n_per_image / 4, 256, ctx->sm_count), B);
  if (reps == 3) {
    DK_DISPATCH(dtype, (sampler_sde_step_kernel<T, true><<<grid, 256, 0, stream>>>(
                           x, d_prev, static_cast<const T*>(xin), static_cast<const T*>(out), n_per_image, n, sigma, a,
                           b, c, noise, cfg_weight, slg, seeds, static_cast<uint32_t>(step))));
  } else {
    DK_DISPATCH(dtype, (sampler_sde_step_kernel<T, false><<<grid, 256, 0, stream>>>(
                           x, d_prev, static_cast<const T*>(xin), static_cast<const T*>(out), n_per_image, n, sigma, a,
                           b, c, noise, cfg_weight, 0.f, seeds, static_cast<uint32_t>(step))));
  }
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_inpaint_blend(dk_ctx* ctx, float* x, const float* eps, const float* x0, const uint8_t* mask, int B,
                                long long HW, int C, float a, float b, void* stream_) {
  DK_ENTRY(ctx);
  DK_REQUIRE(x != nullptr && eps != nullptr && x0 != nullptr && mask != nullptr,
             "dk_inpaint_blend: x, eps, x0 and mask are required");
  DK_REQUIRE(dk_aligned16(x) && dk_aligned16(eps) && dk_aligned16(x0),
             "dk_inpaint_blend: x, eps and x0 must be 16-byte aligned");
  DK_REQUIRE(B >= 1 && B <= 65535, "dk_inpaint_blend: B must be in [1, 65535], got %d", B);
  DK_REQUIRE(C > 0 && C % 4 == 0, "dk_inpaint_blend: C must be a positive multiple of 4, got %d", C);
  DK_REQUIRE(HW > 0 && HW * C / 4 < (1ll << 31), "dk_inpaint_blend: HW * C / 4 must be in [1, 2^31), got HW = %lld",
             HW);
  DK_REQUIRE(isfinite(a) && isfinite(b), "dk_inpaint_blend: a and b must be finite");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long n4 = HW * C / 4;
  const dim3 grid(dk_grid_for(n4, 256, ctx->sm_count), B);
  inpaint_blend_kernel<<<grid, 256, 0, stream>>>(x, eps, x0, mask, static_cast<unsigned>(n4),
                                                 static_cast<unsigned>(C / 4), a, b);
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_inpaint_paste(dk_ctx* ctx, uint8_t* img, const uint8_t* src, const uint8_t* mask, int B,
                                long long pixels, void* stream_) {
  DK_ENTRY(ctx);
  DK_REQUIRE(img != nullptr && src != nullptr && mask != nullptr, "dk_inpaint_paste: img, src and mask are required");
  DK_REQUIRE(((reinterpret_cast<uintptr_t>(img) | reinterpret_cast<uintptr_t>(src) |
               reinterpret_cast<uintptr_t>(mask)) & 3u) == 0,
             "dk_inpaint_paste: img, src and mask must be 4-byte aligned");
  DK_REQUIRE(B >= 1 && B <= 65535, "dk_inpaint_paste: B must be in [1, 65535], got %d", B);
  DK_REQUIRE(pixels > 0 && pixels % 4 == 0 && pixels / 4 < (1ll << 31),
             "dk_inpaint_paste: pixels must be a positive multiple of 4 below 2^33, got %lld", pixels);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const dim3 grid(dk_grid_for(pixels / 4, 256, ctx->sm_count), B);
  inpaint_paste_kernel<<<grid, 256, 0, stream>>>(img, src, mask, static_cast<unsigned>(pixels / 4));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_axpb_f32(dk_ctx* ctx, const float* x, float* y, long long n, float a, float b, void* stream_) {
  DK_ENTRY(ctx);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  axpb_kernel<<<dk_grid_for(n, 256, ctx->sm_count), 256, 0, stream>>>(x, y, n, a, b);
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_dequant_q4(dk_ctx* ctx, int dtype, const uint32_t* wq, const void* scales, const void* biases,
                             void* out, long long N, int K, int group_size, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(N > 0 && K > 0, "dk_dequant_q4: empty weight");
  DK_REQUIRE(group_size >= 8 && group_size % 8 == 0 && K % group_size == 0,
             "dk_dequant_q4: K (%d) must be a multiple of group_size (%d), itself a multiple of 8", K, group_size);
  DK_REQUIRE(dk_aligned16(out), "dk_dequant_q4: out must be 16-byte aligned");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (dequant_q4_kernel<T><<<dk_grid_for(N * (K / 8), 256, ctx->sm_count), 256, 0, stream>>>(
                         wq, static_cast<const T*>(scales), static_cast<const T*>(biases), static_cast<T*>(out), N, K,
                         group_size)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_image_pre(dk_ctx* ctx, int dtype, const uint8_t* img, void* out, long long pixels, int src_channels,
                            int cpad, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(src_channels >= 3, "dk_image_pre: image needs at least 3 channels (got %d)", src_channels);
  DK_REQUIRE(cpad >= 8 && cpad % 8 == 0, "dk_image_pre: cpad (%d) must be a positive multiple of 8", cpad);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (image_pre_kernel<T><<<dk_grid_for(pixels * (cpad / 8), 256, ctx->sm_count), 256, 0, stream>>>(
                         img, static_cast<T*>(out), pixels, src_channels, cpad)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_image_pre_masked(dk_ctx* ctx, int dtype, const uint8_t* img, const uint8_t* mask, void* out, int H,
                                   int W, int src_channels, int cpad, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(img != nullptr && mask != nullptr && out != nullptr, "dk_image_pre_masked: img, mask and out are required");
  DK_REQUIRE(dk_aligned16(out), "dk_image_pre_masked: out must be 16-byte aligned");
  DK_REQUIRE(H > 0 && W > 0 && H % 16 == 0 && W % 16 == 0,
             "dk_image_pre_masked: H and W must be positive multiples of 16, got %dx%d", H, W);
  DK_REQUIRE(src_channels >= 3, "dk_image_pre_masked: image needs at least 3 channels (got %d)", src_channels);
  DK_REQUIRE(cpad >= 8 && cpad % 8 == 0, "dk_image_pre_masked: cpad (%d) must be a positive multiple of 8", cpad);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long pixels = static_cast<long long>(H) * W;
  DK_DISPATCH(dtype, (image_pre_masked_kernel<T><<<dk_grid_for(pixels * (cpad / 8), 256, ctx->sm_count), 256, 0,
                                                   stream>>>(img, mask, static_cast<T*>(out), pixels, src_channels,
                                                             cpad)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_fill_cond_rows(dk_ctx* ctx, int dtype, const void* lat, const uint8_t* mask, void* out, int H, int W,
                                 void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(lat != nullptr && mask != nullptr && out != nullptr, "dk_fill_cond_rows: lat, mask and out are required");
  DK_REQUIRE(dk_aligned16(lat) && dk_aligned16(out), "dk_fill_cond_rows: lat and out must be 16-byte aligned");
  DK_REQUIRE(H > 0 && W > 0 && H % 16 == 0 && W % 16 == 0,
             "dk_fill_cond_rows: H and W must be positive multiples of 16, got %dx%d", H, W);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long nvec = static_cast<long long>(H / 16) * (W / 16) * 40;
  DK_DISPATCH(dtype, (fill_cond_rows_kernel<T><<<dk_grid_for(nvec, 256, ctx->sm_count), 256, 0, stream>>>(
                         static_cast<const T*>(lat), mask, static_cast<T*>(out), H, W)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_image_patches(dk_ctx* ctx, int dtype, const uint8_t* img, void* out, int B, int H, int W,
                                int src_channels, int p, int kp, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(src_channels >= 3, "dk_image_patches: image needs at least 3 channels (got %d)", src_channels);
  DK_REQUIRE(B > 0 && p > 0 && H >= p && W >= p, "dk_image_patches: image %dx%d (batch %d) has no %dx%d patch", H, W, B,
             p, p);
  DK_REQUIRE(kp % 8 == 0 && kp >= 3 * p * p, "dk_image_patches: kp (%d) must be a multiple of 8 and >= 3p^2 (%d)", kp,
             3 * p * p);
  DK_REQUIRE(dk_aligned16(out), "dk_image_patches: out must be 16-byte aligned");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long nvec = static_cast<long long>(B) * (H / p) * (W / p) * (kp / 8);
  DK_DISPATCH(dtype, (image_patches_kernel<T><<<dk_grid_for(nvec, 256, ctx->sm_count), 256, 0, stream>>>(
                         img, static_cast<T*>(out), B, H, W, src_channels, p, kp)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_axpby_f32(dk_ctx* ctx, const float* x, const float* y, float* out, long long n, float a, float b,
                            void* stream_) {
  DK_ENTRY(ctx);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  axpby_kernel<<<dk_grid_for(n, 256, ctx->sm_count), 256, 0, stream>>>(x, y, out, n, a, b);
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_vae_sample_latent(dk_ctx* ctx, int dtype, const void* hidden, const float* noise, float* out,
                                    long long pixels, int C, float shift, float scale, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (vae_sample_latent_kernel<T><<<dk_grid_for(pixels * C, 256, ctx->sm_count), 256, 0, stream>>>(
                         static_cast<const T*>(hidden), noise, out, pixels, C, shift, scale)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_cast_f32_to_16(dk_ctx* ctx, int dtype, const float* x, void* y, long long n, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (cast_f32_to_16_kernel<T><<<dk_grid_for(n, 256, ctx->sm_count), 256, 0, stream>>>(
                         x, static_cast<T*>(y), n)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}
extern "C" int dk_cast_16_to_f32(dk_ctx* ctx, int dtype, const void* x, float* y, long long n, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (cast_16_to_f32_kernel<T><<<dk_grid_for(n, 256, ctx->sm_count), 256, 0, stream>>>(
                         static_cast<const T*>(x), y, n)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_groupnorm_ws_floats(int B, int G) { return B * GN_MAX_CHUNKS * G * 2; }

extern "C" int dk_groupnorm_stats(dk_ctx* ctx, int dtype, const void* x, float* stats, float* ws, int B, int HW, int C,
                                  int G, float eps, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(C % 8 == 0 && C % G == 0 && C <= 2048, "dk_groupnorm_stats: C=%d G=%d unsupported", C, G);
  DK_REQUIRE(ws != nullptr, "dk_groupnorm_stats: workspace of dk_groupnorm_ws_floats(B, G) floats required");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int chunks = gn_chunks(HW);
  dim3 grid(chunks, B);
  DK_DISPATCH(dtype, (groupnorm_partial_kernel<T><<<grid, GN_THREADS, (2 * C + 2 * GN_THREADS * 8) * sizeof(float), stream>>>(
                         static_cast<const T*>(x), ws, HW, C, G, chunks)));
  DK_LAUNCH_CHECK(ctx);
  groupnorm_finalize_kernel<<<B * G, GNF_THREADS, 0, stream>>>(ws, stats, B, G, chunks,
                                                                static_cast<double>(HW) * (C / G), eps);
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_groupnorm_finalize(dk_ctx* ctx, const float* partial, float* stats, int B, int G, int slots,
                                     double count, float eps, void* stream_) {
  DK_ENTRY(ctx);
  DK_REQUIRE(partial != nullptr && stats != nullptr && B > 0 && G > 0 && slots > 0 && count > 0,
             "dk_groupnorm_finalize: bad arguments");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  groupnorm_finalize_kernel<<<B * G, GNF_THREADS, 0, stream>>>(partial, stats, B, G, slots, count, eps);
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_groupnorm_apply(dk_ctx* ctx, int dtype, const void* x, void* y, const float* stats, const void* gamma,
                                  const void* beta, int B, int HW, int C, int G, int silu, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(C % 8 == 0 && C % G == 0 && C <= 2048, "dk_groupnorm_apply: C=%d G=%d unsupported", C, G);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int pix_per_iter = GN_THREADS / (C / 8);
  int blocks = (HW + pix_per_iter * 4 - 1) / (pix_per_iter * 4);   // >= 4 pixels per thread
  const int cap = (ctx->sm_count * 16 + B - 1) / B;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  dim3 grid(blocks, B);
  DK_DISPATCH(dtype, (groupnorm_apply_kernel<T><<<grid, GN_THREADS, 0, stream>>>(
                         static_cast<const T*>(x), static_cast<T*>(y), stats, static_cast<const T*>(gamma),
                         static_cast<const T*>(beta), HW, C, G, silu)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_upsample_nearest2x(dk_ctx* ctx, int dtype, const void* x, void* y, int B, int H, int W, int C,
                                     void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(C % 8 == 0, "dk_upsample_nearest2x: C must be a multiple of 8");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int rows_per_block = 2;   // even: both replicas of an input row are written by the same thread
  dim3 grid((2 * H + rows_per_block - 1) / rows_per_block, B);
  DK_DISPATCH(dtype, (upsample2x_kernel<T><<<grid, 256, 0, stream>>>(static_cast<const T*>(x), static_cast<T*>(y), H,
                                                                       W, C, rows_per_block)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_softmax_rows(dk_ctx* ctx, int dtype, void* x, long long rows, int n, long long ld, float scale,
                               void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(n % 8 == 0 && ld % 8 == 0, "dk_softmax_rows: n and ld must be multiples of 8");
  DK_REQUIRE(rows > 0 && rows < (1LL << 31), "dk_softmax_rows: bad row count");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (softmax_rows_kernel<T><<<static_cast<unsigned>(rows), 256, 0, stream>>>(static_cast<T*>(x), n, ld,
                                                                                             scale)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_image_post(dk_ctx* ctx, int dtype, const void* x, int c_stride, float* img_f32, uint8_t* img_u8,
                             long long pixels, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (image_post_kernel<T><<<dk_grid_for(pixels * 3, 256, ctx->sm_count), 256, 0, stream>>>(
                         static_cast<const T*>(x), c_stride, img_f32, img_u8, pixels)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_residual_delta(dk_ctx* ctx, int dtype, const void* x, long long ldx, int x_seq_rows, const void* base,
                                 long long ldb, int b_seq_rows, float* r_out, const float* prev, float* sums, float* ws,
                                 int nseq, int rows, int h, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(x != nullptr && base != nullptr, "dk_residual_delta: x and base are required");
  DK_REQUIRE(nseq > 0 && rows > 0 && h > 0, "dk_residual_delta: empty input (nseq %d, rows %d, h %d)", nseq, rows, h);
  DK_REQUIRE(h % 8 == 0 && ldx % 8 == 0 && ldb % 8 == 0 && ldx >= h && ldb >= h,
             "dk_residual_delta: h (%d), ldx (%lld) and ldb (%lld) must be multiples of 8, ldx and ldb >= h", h, ldx,
             ldb);
  DK_REQUIRE(x_seq_rows >= rows && b_seq_rows >= rows,
             "dk_residual_delta: x_seq_rows (%d) and b_seq_rows (%d) must be >= rows (%d)", x_seq_rows, b_seq_rows, rows);
  DK_REQUIRE(r_out != nullptr || prev != nullptr, "dk_residual_delta: nothing to do (r_out and prev are both null)");
  DK_REQUIRE(prev == nullptr || (sums != nullptr && ws != nullptr), "dk_residual_delta: prev needs sums and ws");
  DK_REQUIRE(dk_aligned16(x) && dk_aligned16(base) && dk_aligned16(r_out) && dk_aligned16(prev),
             "dk_residual_delta: x, base, r_out and prev must be 16-byte aligned");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int chunks = rd_chunks(rows, h, ctx->sm_count, nseq);
  dim3 grid(chunks, nseq);
  DK_DISPATCH(dtype, (residual_delta_kernel<T><<<grid, RD_THREADS, 0, stream>>>(
                         static_cast<const T*>(x), ldx, x_seq_rows, static_cast<const T*>(base), ldb, b_seq_rows, r_out,
                         prev, ws, rows, h)));
  DK_LAUNCH_CHECK(ctx);
  if (prev != nullptr) {
    residual_delta_finalize_kernel<<<dk_ceil_div(nseq, 4), 128, 0, stream>>>(ws, sums, nseq, chunks);
    DK_LAUNCH_CHECK(ctx);
  }
  return 0;
}

extern "C" int dk_residual_apply(dk_ctx* ctx, int dtype, const void* x, const float* r, void* out, long long n,
                                 void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(x != nullptr && r != nullptr && out != nullptr, "dk_residual_apply: x, r and out are required");
  DK_REQUIRE(n > 0 && n % 8 == 0, "dk_residual_apply: n (%lld) must be a positive multiple of 8", n);
  DK_REQUIRE(dk_aligned16(x) && dk_aligned16(r) && dk_aligned16(out),
             "dk_residual_apply: x, r and out must be 16-byte aligned");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, (residual_apply_kernel<T><<<dk_grid_for(n / 8, 256, ctx->sm_count), 256, 0, stream>>>(
                         static_cast<const T*>(x), r, static_cast<T*>(out), n)));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}
