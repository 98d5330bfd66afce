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

// Where row r (0..127) of the output tile of m-block m_blk goes.  A whole tile may lie past the end (the idle partner
// of the last m-block of a 2-CTA cluster): its rows are not ok.
struct EpiRow {
  bool ok;
  int batch, pos;          // pos: position in the joint sequence (RoPE)
  long long orow, rrow;    // destination row of out / of the residual
};
template <int MODE>
__device__ __forceinline__ EpiRow epi_row(const GemmShape& s, const GemmEpi& e, const ConvGeom& g, int m_blk, int r) {
  EpiRow o;
  if (MODE == 0) {
    const int m = m_blk * 128 + r;
    o.ok = m < s.M;
    o.batch = m / e.rpb;
    const int in_b = m - o.batch * e.rpb;
    o.pos = e.out_row_off + in_b;
    o.orow = static_cast<long long>(o.batch) * e.out_batch_rows + e.out_row_off + in_b;
    o.rrow = static_cast<long long>(o.batch) * e.res_batch_rows + e.res_row_off + in_b;
  } else {
    const int per_img = g.tiles_x * g.tiles_y;
    const int img = m_blk / per_img;
    const int t = m_blk - img * per_img;
    const int y = (t / g.tiles_x) * g.TH + r / g.TW;
    const int x = (t % g.tiles_x) * g.TW + r % g.TW;
    o.ok = img < g.B && y < g.H && x < g.W;
    o.batch = img;
    o.pos = 0;
    o.orow = (static_cast<long long>(img) * g.H + y) * g.W + x;
    o.rrow = o.orow;
  }
  return o;
}

template <typename T>
__device__ __forceinline__ uint32_t ld_u32(const T* p) {
  return *reinterpret_cast<const uint32_t*>(p);
}

// Epilogue of one 128 x BN tile, run by consumer warpgroup cw on its 64 rows straight from the wgmma accumulator
// fragment (layout above stage_acc_rows: row 16*warp + lane/4 + 8i, columns 8j + 2*(lane%4) + {0,1}).  The columns go
// in passes of EC <= 128: the finished 16-bit values of a pass are written to this warpgroup's 64 x EC staging tile
// `stg` (16-byte chunk c of row r at chunk c ^ (r & 7): conflict-free fragment writes and row reads), then every row
// leaves as coalesced 16-byte stores to its destination row.  `rstd` holds 128 floats for this warpgroup.
// Per element the fp32 order is that of the reference: bias, activation, gate, residual, one rounding; the QK path
// rounds (acc + bias) to 16 bits for the head's sum of squares, which one thread per (row, head) adds in column order.
template <typename T, int BN, int MODE>
__device__ __forceinline__ void gemm_epilogue_tile(const float (&acc)[BN / 2], const GemmShape& s, const GemmEpi& e,
                                                   const ConvGeom& g, int m_blk, int n_blk, int cw, uint8_t* stg,
                                                   float* rstd) {
  using H16 = Half16<T>;
  constexpr int EC = BN < 128 ? BN : 128;  // columns per pass
  constexpr int JP = EC / 8;               // 8-column fragment groups per pass = 16-byte chunks per staged row
  constexpr int ROWB = EC * 2;
  constexpr int G = 4;                     // fragment groups whose global loads are issued together
  constexpr int GQ = 2;                    // the same on the QK path, which holds more per group
  const uint32_t bar = 1 + cw;             // named barrier of this warpgroup
  const int t = threadIdx.x & 127;
  const int lane = t & 31;
  const int q = lane & 3;
  const int rl0 = (t >> 5) * 16 + (lane >> 2);   // fragment rows rl0 and rl0 + 8 of this warpgroup's 64
  const int row0 = cw * 64;
  const T* bias = reinterpret_cast<const T*>(e.bias);
  const T* gate = reinterpret_cast<const T*>(e.gate);
  const T* res = reinterpret_cast<const T*>(e.res);
  T* out = reinterpret_cast<T*>(e.out);
  // this thread's two columns of fragment group jj in staged row rl
  auto slot = [&](int rl, int jj) { return rl * ROWB + ((jj ^ (rl & 7)) << 4) + q * 4; };
  const uint32_t stg_s = smem_u32(stg);
  auto put = [&](int rl, int jj, float lo, float hi) { st_shared_u32(stg_s + slot(rl, jj), H16::pack(lo, hi)); };

#pragma unroll
  for (int p = 0; p < BN / EC; ++p) {
    const int n_pass = n_blk * BN + p * EC;
    if (MODE == 0 && e.qk_d != 0 && n_pass < 2 * e.qk_h) {
      // ---- q / k columns of a packed QKV projection: RMSNorm over each head, then RoPE.  Passes are head aligned
      //      (heads*d % 128 == 0, d in {64, 128}).
      //      reference: q = Linear(m) (16-bit) -> nn.RMSNorm (fp32 accumulate, 16-bit out) -> RoPE in fp32
      //      (mlx/mmdit.py:471-488, 754-764, 934-942)
      const int d = e.qk_d;
      const EpiRow fr[2] = {epi_row<MODE>(s, e, g, m_blk, row0 + rl0), epi_row<MODE>(s, e, g, m_blk, row0 + rl0 + 8)};
      const T* nw = reinterpret_cast<const T*>(n_pass < e.qk_h ? e.qk_qw : e.qk_kw);
      // (cos, sin) row of each fragment row; a row past the end reads row 0 and stores nothing
      const float* rope[2];
#pragma unroll
      for (int i = 0; i < 2; ++i)
        rope[i] = e.qk_rope + (fr[i].ok ? static_cast<long long>(fr[i].pos) * d : 0);
      if (nw != nullptr) {
        // the norm sees only (acc + bias) rounded to 16 bits: stage that, then sum each head's squares in column order
#pragma unroll
        for (int j0 = 0; j0 < JP; j0 += G) {
          uint32_t bw[G];
          if (bias != nullptr) {
#pragma unroll
            for (int u = 0; u < G; ++u) bw[u] = ld_u32(bias + n_pass + 8 * (j0 + u) + 2 * q);
          }
#pragma unroll
          for (int u = 0; u < G; ++u) {
            const int a = p * (EC / 2) + 4 * (j0 + u);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              float v0 = acc[a + 2 * i], v1 = acc[a + 2 * i + 1];
              if (bias != nullptr) {
                const float2 b = H16::unpack(bw[u]);
                v0 += b.x;
                v1 += b.y;
              }
              put(rl0 + 8 * i, j0 + u, v0, v1);
            }
          }
        }
        named_bar_sync(bar, 128);
        if (t < 64 * (EC / d)) {
          const int rl = t & 63, hd = t >> 6;
          const int cph = d >> 3;
          float ss = 0.f;
#pragma unroll 1
          for (int c = 0; c < cph; ++c) {
            const uint4 v4 = *reinterpret_cast<const uint4*>(stg + rl * ROWB + (((hd * cph + c) ^ (rl & 7)) << 4));
            const uint32_t w[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float2 f = H16::unpack(w[k]);
              ss += f.x * f.x;
              ss += f.y * f.y;
            }
          }
          rstd[hd * 64 + rl] = rsqrtf(ss / d + e.qk_eps);
        }
        named_bar_sync(bar, 128);
      }
#pragma unroll
      for (int j0 = 0; j0 < JP; j0 += GQ) {
        uint32_t bw[GQ], ww[GQ];
        float2 cs[2][GQ];
        if (nw != nullptr) {
#pragma unroll
          for (int u = 0; u < GQ; ++u) ww[u] = ld_u32(nw + ((8 * (j0 + u) + 2 * q) & (d - 1)));
        } else if (bias != nullptr) {
#pragma unroll
          for (int u = 0; u < GQ; ++u) bw[u] = ld_u32(bias + n_pass + 8 * (j0 + u) + 2 * q);
        }
        if (e.qk_rope != nullptr) {
#pragma unroll
          for (int u = 0; u < GQ; ++u)
#pragma unroll
            for (int i = 0; i < 2; ++i)
              cs[i][u] = *reinterpret_cast<const float2*>(rope[i] + ((8 * (j0 + u) + 2 * q) & (d - 1)));
        }
        // one branch per group, not per element pair: the group's chains interleave
        float v[GQ][2][2];
        if (nw != nullptr) {
#pragma unroll
          for (int u = 0; u < GQ; ++u) {
            const int hd = 8 * (j0 + u) >= d ? 1 : 0;   // head inside the pass
            const float2 w = H16::unpack(ww[u]);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const float2 h = H16::unpack(*reinterpret_cast<const uint32_t*>(stg + slot(rl0 + 8 * i, j0 + u)));
              const float r = rstd[hd * 64 + rl0 + 8 * i];
              v[u][i][0] = H16::to_f(H16::from_f(h.x * r * w.x));   // h: the staged, rounded acc + bias
              v[u][i][1] = H16::to_f(H16::from_f(h.y * r * w.y));
            }
          }
        } else {
#pragma unroll
          for (int u = 0; u < GQ; ++u)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const int a = p * (EC / 2) + 4 * (j0 + u) + 2 * i;
              v[u][i][0] = acc[a];
              v[u][i][1] = acc[a + 1];
              if (bias != nullptr) {
                const float2 b = H16::unpack(bw[u]);
                v[u][i][0] += b.x;
                v[u][i][1] += b.y;
              }
            }
        }
        if (e.qk_rope != nullptr) {
#pragma unroll
          for (int u = 0; u < GQ; ++u)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const float a0 = v[u][i][0], a1 = v[u][i][1];
              v[u][i][0] = a0 * cs[i][u].x - a1 * cs[i][u].y;
              v[u][i][1] = a0 * cs[i][u].y + a1 * cs[i][u].x;
            }
        }
#pragma unroll
        for (int u = 0; u < GQ; ++u)
#pragma unroll
          for (int i = 0; i < 2; ++i) put(rl0 + 8 * i, j0 + u, v[u][i][0], v[u][i][1]);
      }
    } else {
      const EpiRow fr[2] = {epi_row<MODE>(s, e, g, m_blk, row0 + rl0), epi_row<MODE>(s, e, g, m_blk, row0 + rl0 + 8)};
      // gate / residual row of each fragment row; a row past the end reads row 0 and stores nothing
      const T* grow[2];
      const T* rrow[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        grow[i] = gate + (fr[i].ok ? static_cast<long long>(fr[i].batch) * e.gate_ld : 0);
        rrow[i] = res + (fr[i].ok ? fr[i].rrow * e.ldres : 0);
      }
#pragma unroll
      for (int j0 = 0; j0 < JP; j0 += G) {
        // the loads of a group are issued together (column clamped to N: groups past N are computed, not stored)
        uint32_t bw[G], gw[2][G], rw[2][G];
        int n[G];
#pragma unroll
        for (int u = 0; u < G; ++u) n[u] = min(n_pass + 8 * (j0 + u), s.N - 8) + 2 * q;
        if (bias != nullptr) {
#pragma unroll
          for (int u = 0; u < G; ++u) bw[u] = ld_u32(bias + n[u]);
        }
        if (gate != nullptr) {
#pragma unroll
          for (int u = 0; u < G; ++u)
#pragma unroll
            for (int i = 0; i < 2; ++i) gw[i][u] = ld_u32(grow[i] + n[u]);
        }
        if (res != nullptr) {
#pragma unroll
          for (int u = 0; u < G; ++u)
#pragma unroll
            for (int i = 0; i < 2; ++i) rw[i][u] = ld_u32(rrow[i] + n[u]);
        }
        // one branch per group and step, not per element pair: the group's chains (GELU-erf) interleave
        float v[G][2][2];
#pragma unroll
        for (int u = 0; u < G; ++u)
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int a = p * (EC / 2) + 4 * (j0 + u) + 2 * i;
            v[u][i][0] = acc[a];
            v[u][i][1] = acc[a + 1];
          }
        if (bias != nullptr) {
#pragma unroll
          for (int u = 0; u < G; ++u)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const float2 b = H16::unpack(bw[u]);
              v[u][i][0] += b.x;
              v[u][i][1] += b.y;
            }
        }
        if (e.act == DK_ACT_GELU_ERF) {
#pragma unroll
          for (int u = 0; u < G; ++u)
#pragma unroll
            for (int k = 0; k < 4; ++k) v[u][k >> 1][k & 1] = gelu_erf(v[u][k >> 1][k & 1]);
        } else if (e.act == DK_ACT_SILU) {
#pragma unroll
          for (int u = 0; u < G; ++u)
#pragma unroll
            for (int k = 0; k < 4; ++k) v[u][k >> 1][k & 1] = silu_f(v[u][k >> 1][k & 1]);
        } else if (e.act == DK_ACT_QUICK_GELU) {
#pragma unroll
          for (int u = 0; u < G; ++u)
#pragma unroll
            for (int k = 0; k < 4; ++k) v[u][k >> 1][k & 1] = quick_gelu_f(v[u][k >> 1][k & 1]);
        }
        if (gate != nullptr) {
#pragma unroll
          for (int u = 0; u < G; ++u)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const float2 gv = H16::unpack(gw[i][u]);
              v[u][i][0] *= gv.x;
              v[u][i][1] *= gv.y;
            }
        }
        if (res != nullptr) {
#pragma unroll
          for (int u = 0; u < G; ++u)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const float2 rv = H16::unpack(rw[i][u]);
              v[u][i][0] += rv.x;
              v[u][i][1] += rv.y;
            }
        }
#pragma unroll
        for (int u = 0; u < G; ++u)
#pragma unroll
          for (int i = 0; i < 2; ++i) put(rl0 + 8 * i, j0 + u, v[u][i][0], v[u][i][1]);
      }
    }
    named_bar_sync(bar, 128);

    // ---- staged rows -> destination rows, JP threads per row
    const int c = t % JP;
    const int n = n_pass + 8 * c;
#pragma unroll 2
    for (int r0 = 0; r0 < 64; r0 += 128 / JP) {
      const int rl = r0 + t / JP;
      const EpiRow row = epi_row<MODE>(s, e, g, m_blk, row0 + rl);
      if (row.ok && n < s.N)
        __stcs(reinterpret_cast<uint4*>(out + row.orow * e.ldc + n),
               *reinterpret_cast<const uint4*>(stg + rl * ROWB + ((c ^ (rl & 7)) << 4)));
    }
    named_bar_sync(bar, 128);
  }
}

}  // namespace dk
