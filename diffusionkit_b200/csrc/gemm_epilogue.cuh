// Shared pieces of the wgmma GEMM kernel: problem/epilogue descriptors and the accumulator -> global
// epilogue (bias / GELU-erf / SiLU / adaLN gate / residual, or QK-RMSNorm + RoPE on a packed QKV projection).
#pragma once

#include "common.cuh"
#include "../../include/dkb200.h"

namespace dk {

struct GemmShape {
  int M, N, K;
  int num_m, num_n, num_k;
};

struct GemmEpi {
  void* out;
  long long ldc;
  const void* bias;
  const void* gate;
  long long gate_ld;
  const void* res;
  long long ldres;
  int rpb;
  int out_batch_rows, out_row_off;
  int res_batch_rows, res_row_off;
  int act;
  int debug;  // timing experiments only (DK_GEMM_EPI_DEBUG): 1 = skip the global stores, 2 = skip everything after the accumulator read
  // fused QK-RMSNorm + RoPE on the q and k thirds of a packed QKV projection (columns [0, 2*qk_h)); qk_d == 0 disables
  const void* qk_qw;   // [d] RMSNorm weight of q (or NULL: no norm)
  const void* qk_kw;   // [d]
  const float* qk_rope;  // [S, d/2, 2] (cos, sin) or NULL
  int qk_h, qk_d;
  float qk_eps;
};

struct ConvGeom {
  int B, H, W, Cin;      // H, W: OUTPUT size
  int stride, pad;       // stride 1 / pad 1 (symmetric), or stride 2 / pad 0 with an implicit zero row+column at the
                         // bottom/right (mlx: pad [(0,1),(0,1)] then stride-2 conv, vae.py:142-144)
  int TH, TW;            // output-pixel tile: TH x TW = 128
  int tiles_x, tiles_y;  // per image
  int cblocks;           // Cin / 64
};


// 16 finished 16-bit values of one row -> global (two 128-bit streaming stores).
__device__ __forceinline__ void store_row16(void* dst, const uint32_t (&w)[8]) {
  __stcs(reinterpret_cast<uint4*>(dst), make_uint4(w[0], w[1], w[2], w[3]));
  __stcs(reinterpret_cast<uint4*>(dst) + 1, make_uint4(w[4], w[5], w[6], w[7]));
}

// Drains NCH 32-column chunks of one accumulator row (this thread = one tile row; load32(c, r) fills r with the fp32
// bits of the 32 columns starting c columns after the thread's first column) and stores the finished 16-bit values.
template <typename T, int NCH, int MODE, typename Load>
__device__ __forceinline__ void gemm_epilogue_drain(const GemmShape& s, const GemmEpi& e, Load load32, int n_half0,
                                                    bool row_ok, long long orow, long long rrow, int batch, int pos) {
  using H16 = Half16<T>;
  const T* bias = reinterpret_cast<const T*>(e.bias);
  const T* gate = reinterpret_cast<const T*>(e.gate);
  const T* res = reinterpret_cast<const T*>(e.res);
  T* out = reinterpret_cast<T*>(e.out);
  if (MODE == 0 && e.qk_d != 0 && n_half0 < 2 * e.qk_h) {
  // ---- q / k columns of a packed QKV projection: RMSNorm over each head (two passes over the staged row), then RoPE.
  //      reference: q = Linear(m) (16-bit) -> nn.RMSNorm (fp32 accumulate, 16-bit out) -> RoPE in fp32
  //      (mlx/mmdit.py:471-488, 754-764, 934-942)
  const int d = e.qk_d;
  const int cph = d >> 5;  // chunks per head
  const T* nw = reinterpret_cast<const T*>(n_half0 < e.qk_h ? e.qk_qw : e.qk_kw);
#pragma unroll 1
  for (int hc = 0; hc < NCH; hc += cph) {
    float ss = 0.f;
    if (nw != nullptr) {
#pragma unroll 1
      for (int c = 0; c < cph; ++c) {
        uint32_t r[32];
        load32((hc + c) * 32, r);
        const int n0 = n_half0 + (hc + c) * 32;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float bv[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) bv[i] = 0.f;
          if (bias != nullptr) {
            const uint4 b4 = *reinterpret_cast<const uint4*>(bias + n0 + j * 8);
            const uint32_t bw[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float2 f = H16::unpack(bw[i]);
              bv[2 * i] = f.x;
              bv[2 * i + 1] = f.y;
            }
          }
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float v = H16::to_f(H16::from_f(__uint_as_float(r[j * 8 + i]) + bv[i]));
            ss += v * v;
          }
        }
      }
    }
    const float rstd = rsqrtf(ss / d + e.qk_eps);
    const int head_col0 = (n_half0 + hc * 32) % d;  // 0: tiles are head aligned
#pragma unroll 1
    for (int c = 0; c < cph; ++c) {
      uint32_t r[32];
      load32((hc + c) * 32, r);
      if (!row_ok || e.debug >= 2) continue;
      const int n0 = n_half0 + (hc + c) * 32;
      const int dcol0 = head_col0 + c * 32;  // column inside the head
      uint32_t w16[8];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = n0 + j * 8;
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = __uint_as_float(r[j * 8 + i]);
        if (bias != nullptr) {
          const uint4 b4 = *reinterpret_cast<const uint4*>(bias + n);
          const uint32_t bw[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = H16::unpack(bw[i]);
            v[2 * i] += f.x;
            v[2 * i + 1] += f.y;
          }
        }
        if (nw != nullptr) {
          const uint4 w4 = *reinterpret_cast<const uint4*>(nw + dcol0 + j * 8);
          const uint32_t ww[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = H16::unpack(ww[i]);
            v[2 * i] = H16::to_f(H16::from_f(H16::to_f(H16::from_f(v[2 * i])) * rstd * f.x));
            v[2 * i + 1] = H16::to_f(H16::from_f(H16::to_f(H16::from_f(v[2 * i + 1])) * rstd * f.y));
          }
        }
        if (e.qk_rope != nullptr) {
          const float4* rp = reinterpret_cast<const float4*>(
              e.qk_rope + (static_cast<long long>(pos) * (d >> 1) + ((dcol0 + j * 8) >> 1)) * 2);
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const float4 cs = rp[i];  // (cos0, sin0, cos1, sin1)
            const float a0 = v[4 * i], a1 = v[4 * i + 1], b0 = v[4 * i + 2], b1 = v[4 * i + 3];
            v[4 * i] = a0 * cs.x - a1 * cs.y;
            v[4 * i + 1] = a0 * cs.y + a1 * cs.x;
            v[4 * i + 2] = b0 * cs.z - b1 * cs.w;
            v[4 * i + 3] = b0 * cs.w + b1 * cs.z;
          }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) w16[(j & 1) * 4 + i] = H16::pack(v[2 * i], v[2 * i + 1]);
        if ((j & 1) && e.debug == 0) {
          T* dst = out + orow * e.ldc + (n - 8);
          store_row16(dst, w16);
        }
      }
    }
  }
  return;
}

#pragma unroll 1
for (int chunk = 0; chunk < NCH; ++chunk) {
  uint32_t r[32];
  load32(chunk * 32, r);
  const int n0 = n_half0 + chunk * 32;
  if (!row_ok || e.debug >= 2) continue;
#pragma unroll
  for (int j16 = 0; j16 < 2; ++j16) {
    const int nb = n0 + j16 * 16;
    if (nb >= s.N) break;
    uint32_t w[8];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int j = j16 * 2 + hh;
      const int n = n0 + j * 8;
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = __uint_as_float(r[j * 8 + i]);
      if (n < s.N) {
        if (bias != nullptr) {
          const uint4 b4 = *reinterpret_cast<const uint4*>(bias + n);
          const uint32_t bw[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = H16::unpack(bw[i]);
            v[2 * i] += f.x;
            v[2 * i + 1] += f.y;
          }
        }
        if (e.act == DK_ACT_GELU_ERF) {
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = gelu_erf(v[i]);
        } else if (e.act == DK_ACT_SILU) {
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = silu_f(v[i]);
        } else if (e.act == DK_ACT_QUICK_GELU) {
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = quick_gelu_f(v[i]);
        }
        if (gate != nullptr) {
          const uint4 g4 = *reinterpret_cast<const uint4*>(gate + static_cast<long long>(batch) * e.gate_ld + n);
          const uint32_t gw[4] = {g4.x, g4.y, g4.z, g4.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = H16::unpack(gw[i]);
            v[2 * i] *= f.x;
            v[2 * i + 1] *= f.y;
          }
        }
        if (res != nullptr) {
          const uint4 r4 = *reinterpret_cast<const uint4*>(res + rrow * e.ldres + n);
          const uint32_t rw[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = H16::unpack(rw[i]);
            v[2 * i] += f.x;
            v[2 * i + 1] += f.y;
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) w[hh * 4 + i] = H16::pack(v[2 * i], v[2 * i + 1]);
    }
    if (e.debug != 0) continue;
    T* dst = out + orow * e.ldc + nb;
    if (nb + 16 <= s.N) {
      store_row16(dst, w);
    } else {
      __stcs(reinterpret_cast<uint4*>(dst), make_uint4(w[0], w[1], w[2], w[3]));   // 8-column tail
    }
  }
}
}

}  // namespace dk
