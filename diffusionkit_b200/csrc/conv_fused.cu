// K7 — fused VAE convolution for sm_90a: [GroupNorm-apply + SiLU] -> [nearest 2x] -> conv 3x3 -> [+bias, +skip]
// -> output + GroupNorm partial statistics of the output, one kernel.
// Replaces, per ResnetBlock2D / upsample stage of the reference decoder (mlx/vae.py:60-101, 20-25, 146-147):
//   nn.GroupNorm + nn.SiLU (a separate HBM round trip in round 1), upsample_nearest (a 4x-sized tensor written and read
//   back), nn.Conv2d, the skip add, and the statistics pass of the NEXT GroupNorm (another full read of the output).
//
// Im2col-free, halo-tiled: a CTA owns R = 2 output rows x 128 output pixels; for every block of 64 input channels ONE
// TMA box brings the (R+2) x 130 pixel halo of the raw input into shared memory (128B-swizzled, one 128-byte line per
// pixel; out-of-image pixels are zero-filled by the TMA unit = the zero padding).  The nine taps are NOT nine loads:
// tap (dy, dx) of output row r is the run of 128 consecutive pixel lines starting at halo pixel (r + dy, dx), i.e. the
// same shared-memory tile read through a wgmma descriptor whose start address is shifted by whole lines.  Every input
// byte crosses L2 -> SM once per 64-channel block and n-tile (round 1: nine times).
//
// Because the halo is staged once, the GroupNorm affine + SiLU can run ON it: the consumer threads rewrite the tile in
// place (normalise with the per-(image, channel) scale/shift table, SiLU with one MUFU.TANH, back to 16 bits; padding
// pixels stay zero, as the reference pads AFTER the activation) before the MMAs read it — once per input element, not
// once per tap.
//
// Nearest-2x upsampling never materialises: out(2y+py, 2x+px) of conv3x3(upsample(x)) only sees a 2x2 neighbourhood
// of x, with the 3x3 weights that fall on the same source pixel pre-added (dk_conv_up_weights).  The four output
// phases (py, px) are four 4-tap convolutions over the SAME halo tile (2.25x fewer FLOPs than convolving the
// upsampled tensor); the epilogue scatters each phase to its stride-2 output pixels.
//
// One CTA per work item (R x 128 output pixels x 128 output channels of one image / phase), 384 threads:
//   warpgroup 0 (warp 0) TMA producer: halo boxes (double buffered per 64-channel block) and 128 x 64 weight tiles
//                        (ring)
//   warpgroups 1, 2      output row r = warpgroup - 1: two wgmma m64n128k16 chains (pixels 0-63 and 64-127 of the
//                        row) per tap, A = the halo tile read through a line-shifted descriptor.  Before the MMAs of
//                        a block the 256 threads apply GroupNorm affine + SiLU in place on the halo (a pass-through
//                        when there is no norm).
//   epilogue             the accumulators go through an fp32 staging tile in the (then idle) pipeline buffers; bias,
//                        skip, store, per-(pixel row, group) statistics of the stored values.
#include <stdlib.h>

#include "common.cuh"
#include "host.h"

namespace dk {

constexpr int CF_TW = 128;
constexpr int CF_R = 2;
constexpr int CF_BN = 128;
constexpr int CF_HW = CF_TW + 2;                       // halo width in pixels
constexpr int CF_HR = CF_R + 2;                        // halo rows
constexpr int CF_A_BYTES = CF_HR * CF_HW * 128;        // 66,560 (65 KB) per 64-channel block
constexpr int CF_B_BYTES = CF_BN * 64 * 2;             // 16 KB: one tap's 128 x 64 weight tile
constexpr int CF_A_BUFS = 2;                            // halo buffers
constexpr int CF_B_STAGES = 4;                          // weight ring
constexpr int CF_THREADS = 384;
constexpr int CF_STAGE_LD = CF_BN + 4;                  // fp32 staging row stride (floats)
constexpr int CF_STAT_BYTES = 8 * CF_R * 2 * 8 * 2 * 4;  // [warp][row][chunk][group<=8][sum,sumsq]
constexpr int CF_OFF_B = CF_A_BUFS * CF_A_BYTES;
constexpr int CF_OFF_STAT = CF_OFF_B + CF_B_STAGES * CF_B_BYTES;
constexpr int CF_OFF_BAR = CF_OFF_STAT + CF_STAT_BYTES;
constexpr int CF_SMEM_BYTES = CF_OFF_BAR + 256 + 1024;
static_assert(CF_OFF_STAT >= CF_R * CF_TW * CF_STAGE_LD * 4, "conv_fused: the staging tile reuses the pipeline buffers");
static_assert(CF_SMEM_BYTES <= 232448, "conv_fused: shared memory budget");

struct ConvFParams {
  int B, H, W;          // grid of tile coordinates = the conv INPUT image (source image in upsample mode)
  int Cin, Cout;
  int up;               // 0: 3x3 conv (output H x W); 1: nearest 2x then 3x3 conv, by sub-pixel phases (output 2H x 2W)
  int tiles_x, tiles_y; // W / 128, H / R
  int n_tiles;          // Cout / 128
  const void* bias;     // [Cout] or null
  const void* res;      // output-shaped skip tensor or null
  void* out;
  const float* gn_stats;   // [B, G, 2] (mean, rstd) of the input, or null: no normalisation
  const void* gamma;
  const void* beta;
  int G;
  int silu;
  float* out_partial;   // [B, slots, out_G, 2] per-(128-pixel row segment, group) (sum, sumsq) of the output, or null
  int out_G;
};

__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// work item -> (image, row block, x block, phase, n tile); n tile and phase vary fastest so that the items in flight
// share their halo through L2
struct CfItem {
  int b, ty, tx, phase, nt;
};
__device__ __forceinline__ void cf_decode(const ConvFParams& p, int item, CfItem& it) {
  const int phases = p.up ? 4 : 1;
  it.nt = item % p.n_tiles;
  item /= p.n_tiles;
  it.phase = item % phases;
  item /= phases;
  it.tx = item % p.tiles_x;
  item /= p.tiles_x;
  it.ty = item % p.tiles_y;
  it.b = item / p.tiles_y;
}

// Sum N values (N = 16, 8 or 4) over the 32 lanes of a warp with N + log-many shuffles instead of 5 N: at every step a
// lane keeps one half of its values and hands the other half to its partner (recursive halving), then the last value is
// reduced over the remaining lane bits.  On return lane l holds in v[0] the complete sum of value index
// warp_multi_index<N>(l); lanes that differ only in the low (plain-reduced) bits hold copies.
template <int N>
__device__ __forceinline__ void warp_multi_sum(float (&v)[N], int lane) {
  int off = 16;
#pragma unroll
  for (int n = N; n > 1; n >>= 1, off >>= 1) {
    const bool hi = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < n / 2; ++i) {
      const float keep = hi ? v[i + n / 2] : v[i];
      const float send = hi ? v[i] : v[i + n / 2];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
#pragma unroll
  for (; off > 0; off >>= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], off);
}
template <int N>
__device__ __forceinline__ int warp_multi_index(int lane) {
  int idx = 0, off = 16;
#pragma unroll
  for (int n = N; n > 1; n >>= 1, off >>= 1) idx += (lane & off) ? n / 2 : 0;
  return idx;
}

// per group of CPG channels of one 32-channel chunk: sum and sum of squares over the warp's 32 pixels -> dst[g][2]
template <int CPG>
__device__ __forceinline__ void cf_chunk_stats(const float (&v)[32], float* dst, int lane) {
  constexpr int NG = 32 / CPG;          // groups in the chunk
  constexpr int N = 2 * NG;             // values to reduce: NG sums then NG sums of squares
  float a[N];
#pragma unroll
  for (int g = 0; g < NG; ++g) {
    float s = 0.f, q = 0.f;
#pragma unroll
    for (int c = 0; c < CPG; ++c) {
      const float t = v[g * CPG + c];
      s += t;
      q = fmaf(t, t, q);
    }
    a[g] = s;
    a[NG + g] = q;
  }
  warp_multi_sum<N>(a, lane);
  constexpr int LOW = 32 / N;           // lanes per value (copies)
  if ((lane & (LOW - 1)) == 0) {
    const int idx = warp_multi_index<N>(lane);
    const int g = idx % NG, which = idx / NG;
    dst[g * 2 + which] = a[0];
  }
}

template <typename T>
__global__ void __launch_bounds__(CF_THREADS, 1)
conv_fused_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const ConvFParams p) {
  using H16 = Half16<T>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;                       // [CF_A_BUFS][CF_A_BYTES]
  uint8_t* sB = smem + CF_OFF_B;            // [CF_B_STAGES][CF_B_BYTES]
  float* sstat = reinterpret_cast<float*>(smem + CF_OFF_STAT);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + CF_OFF_BAR);
  uint64_t* a_land = bars;                  // [CF_A_BUFS] TMA halo landed
  uint64_t* a_empty = a_land + CF_A_BUFS;   // [CF_A_BUFS] the MMAs reading the buffer have retired (8 consumer warps)
  uint64_t* b_full = a_empty + CF_A_BUFS;   // [CF_B_STAGES]
  uint64_t* b_empty = b_full + CF_B_STAGES; // [CF_B_STAGES] (8 consumer warps)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int cblocks = p.Cin / 64;
  const int ntaps = p.up ? 4 : 9;
  CfItem it;
  cf_decode(p, blockIdx.x, it);
  const int py = it.phase >> 1, px = it.phase & 1;
  const int y0 = it.ty * CF_R;
  const int x0 = it.tx * CF_TW;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmW);
    for (int i = 0; i < CF_A_BUFS; ++i) {
      mbar_init(&a_land[i], 1);
      mbar_init(&a_empty[i], 8);
    }
    for (int i = 0; i < CF_B_STAGES; ++i) {
      mbar_init(&b_full[i], 1);
      mbar_init(&b_empty[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer, converged warp
    if (warp != 0) return;
    uint32_t bst = 0, bph = 0;     // weight ring
    uint32_t abuf = 0, aph = 0;    // halo double buffer
    const int w_row = it.phase * p.Cout + it.nt * CF_BN;
    for (int cb = 0; cb < cblocks; ++cb) {
      mbar_wait_warp(&a_empty[abuf], aph ^ 1);
      if (elect_one_sync()) {
        mbar_arrive_expect_tx(&a_land[abuf], CF_A_BYTES);
        tma_load_4d(sA + abuf * CF_A_BYTES, &tmX, &a_land[abuf], cb * 64, x0 - 1, y0 - 1, it.b);
      }
      __syncwarp();
      if (++abuf == CF_A_BUFS) {
        abuf = 0;
        aph ^= 1;
      }
      for (int tap = 0; tap < ntaps; ++tap) {
        mbar_wait_warp(&b_empty[bst], bph ^ 1);
        if (elect_one_sync()) {
          mbar_arrive_expect_tx(&b_full[bst], CF_B_BYTES);
          tma_load_2d(sB + bst * CF_B_BYTES, &tmW, &b_full[bst], tap * p.Cin + cb * 64, w_row);
        }
        __syncwarp();
        if (++bst == CF_B_STAGES) {
          bst = 0;
          bph ^= 1;
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: output row rr of the item
  const int rr = wg - 1;
  const int tid = threadIdx.x - 128;          // 0..255
  float acc0[CF_BN / 2], acc1[CF_BN / 2];     // pixels 0-63 / 64-127 of the row
#pragma unroll
  for (int i = 0; i < CF_BN / 2; ++i) {
    acc0[i] = 0.f;
    acc1[i] = 0.f;
  }
  {
    constexpr int TT = 256;
    const int chunk = tid & 7;                 // logical 16-byte chunk = 8 channels of the 64-channel block
    const int cpg = p.gn_stats != nullptr ? p.Cin / p.G : 1;
    uint32_t bst = 0, bph = 0, abuf = 0, aph = 0;
    for (int cb = 0; cb < cblocks; ++cb) {
      mbar_wait(&a_land[abuf], aph);
      if (p.gn_stats != nullptr) {
        // GroupNorm affine + SiLU in place.  Per-channel (scale, shift) of this image: y = x * (rstd * gamma) +
        // (beta - mean * rstd * gamma); the 8 channels of this thread's chunk come straight from global memory
        float sc[8], sh[8];
        {
          const int c0 = cb * 64 + chunk * 8;
          const uint4 g4 = *reinterpret_cast<const uint4*>(reinterpret_cast<const T*>(p.gamma) + c0);
          const uint4 b4 = *reinterpret_cast<const uint4*>(reinterpret_cast<const T*>(p.beta) + c0);
          const uint32_t gw[4] = {g4.x, g4.y, g4.z, g4.w}, bw[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 gf = H16::unpack(gw[i]), bf = H16::unpack(bw[i]);
#pragma unroll
            for (int h2 = 0; h2 < 2; ++h2) {
              const int g = (c0 + 2 * i + h2) / cpg;
              const float mean = __ldg(p.gn_stats + (it.b * p.G + g) * 2), rstd = __ldg(p.gn_stats + (it.b * p.G + g) * 2 + 1);
              const float ga = h2 ? gf.y : gf.x, be = h2 ? bf.y : bf.x;
              sc[2 * i + h2] = rstd * ga;
              sh[2 * i + h2] = be - mean * rstd * ga;
            }
          }
        }
        const uint32_t base = smem_u32(sA) + abuf * CF_A_BYTES;
        const bool do_silu = p.silu != 0;
        // padding pixels (outside the image) stay zero: the reference pads AFTER the activation
        auto in_image = [&](int q) {
          const int hr = q / CF_HW, hx = q - hr * CF_HW;
          const int gy = y0 - 1 + hr, gx = x0 - 1 + hx;
          return q < CF_HR * CF_HW && gy >= 0 && gy < p.H && gx >= 0 && gx < p.W;
        };
        auto xform = [&](uint32_t (&w)[4]) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = H16::unpack(w[i]);
            float a = fmaf(f.x, sc[2 * i], sh[2 * i]);
            float b = fmaf(f.y, sc[2 * i + 1], sh[2 * i + 1]);
            if (do_silu) {   // x * sigmoid(x) = h + h * tanh(h), h = x / 2: one MUFU op per element
              const float ha = 0.5f * a, hb = 0.5f * b;
              a = fmaf(ha, tanh_approx(ha), ha);
              b = fmaf(hb, tanh_approx(hb), hb);
            }
            w[i] = H16::pack(a, b);
          }
        };
        for (int q0 = tid >> 3; q0 < CF_HR * CF_HW; q0 += 2 * (TT / 8)) {
          const int q1 = q0 + TT / 8;
          const bool ok0 = in_image(q0), ok1 = in_image(q1);
          const uint32_t addr0 = base + q0 * 128 + ((chunk ^ (q0 & 7)) << 4);
          const uint32_t addr1 = base + q1 * 128 + ((chunk ^ (q1 & 7)) << 4);
          uint32_t w0[4] = {0u, 0u, 0u, 0u}, w1[4] = {0u, 0u, 0u, 0u};
          if (ok0) asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(w0[0]), "=r"(w0[1]), "=r"(w0[2]), "=r"(w0[3]) : "r"(addr0));
          if (ok1) asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(w1[0]), "=r"(w1[1]), "=r"(w1[2]), "=r"(w1[3]) : "r"(addr1));
          xform(w0);
          xform(w1);
          if (ok0) asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr0), "r"(w0[0]), "r"(w0[1]), "r"(w0[2]), "r"(w0[3]) : "memory");
          if (ok1) asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr1), "r"(w1[0]), "r"(w1[1]), "r"(w1[2]), "r"(w1[3]) : "memory");
        }
        fence_proxy_async_smem();   // generic-proxy writes -> visible to the tensor core's operand reads
        named_bar_sync(1, 256);     // the whole halo is transformed before either warpgroup reads it
      }
      const uint32_t a_addr0 = smem_u32(sA) + abuf * CF_A_BYTES;
      uint32_t prev = 0;
      for (int tap = 0; tap < ntaps; ++tap) {
        // halo offset of this tap: 3x3 -> (tap / 3, tap % 3); phase (py, px) of the upsampled conv -> (a + py, b + px)
        const int dy = p.up ? ((tap >> 1) + py) : (tap / 3);
        const int dx = p.up ? ((tap & 1) + px) : (tap - (tap / 3) * 3);
        mbar_wait(&b_full[bst], bph);
        const uint32_t b_addr = smem_u32(sB) + bst * CF_B_BYTES;
        const uint32_t a_addr = a_addr0 + ((rr + dy) * CF_HW + dx) * 128;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint32_t acc_on = (cb | tap | k) != 0 ? 1u : 0u;
          const uint64_t db = make_smem_desc_sw128(b_addr + k * 32, 16, 1024);
          Wgmma<CF_BN, H16::is_bf16, 0>::ss(acc0, make_smem_desc_sw128(a_addr + k * 32, 16, 1024), db, acc_on);
          Wgmma<CF_BN, H16::is_bf16, 0>::ss(acc1, make_smem_desc_sw128(a_addr + 64 * 128 + k * 32, 16, 1024), db, acc_on);
        }
        wgmma_commit();
        if (tap > 0) {   // the previous tap's MMAs have retired: its weight stage can be refilled
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&b_empty[prev]);
        }
        prev = bst;
        if (++bst == CF_B_STAGES) {
          bst = 0;
          bph ^= 1;
        }
      }
      wgmma_wait<0>();
      if (lane == 0) {
        mbar_arrive(&b_empty[prev]);
        mbar_arrive(&a_empty[abuf]);
      }
      if (++abuf == CF_A_BUFS) {
        abuf = 0;
        aph ^= 1;
      }
    }
    reg_fence(acc0);
    reg_fence(acc1);
  }

  // ------------------------------------------------------------------ epilogue: R x 128 output pixels
  // every load has landed and every MMA has retired once both warpgroups pass this barrier: the pipeline buffers
  // become the fp32 staging tile [R * 128 pixels][CF_STAGE_LD]
  float* stg = reinterpret_cast<float*>(smem);
  named_bar_sync(1, 256);
  stage_acc_rows<CF_BN>(stg, CF_STAGE_LD, rr * CF_TW, acc0);
  stage_acc_rows<CF_BN>(stg, CF_STAGE_LD, rr * CF_TW + 64, acc1);
  named_bar_sync(1, 256);

  const int ew = warp - 4;                    // 0..7
  const int quarter = ew & 3;
  const int half = ew >> 2;                   // 64-channel half of the 128-channel tile
  const int xl = quarter * 32 + lane;         // pixel inside the 128-pixel segment
  const T* bias = reinterpret_cast<const T*>(p.bias);
  const T* res = reinterpret_cast<const T*>(p.res);
  T* out = reinterpret_cast<T*>(p.out);
  const int Hout = p.up ? 2 * p.H : p.H, Wout = p.up ? 2 * p.W : p.W;
  const int cpg_out = p.out_partial != nullptr ? p.Cout / p.out_G : 8;
  const int slots = (Hout * Wout) / CF_TW;
  const int x = x0 + xl;
  const int n_base = it.nt * CF_BN + half * 64;
  float* st_my = sstat + (ew * CF_R) * (2 * 8 * 2);
#pragma unroll 1
  for (int r2 = 0; r2 < CF_R; ++r2) {
    const int oy = p.up ? 2 * (y0 + r2) + py : (y0 + r2);
    const int ox = p.up ? 2 * x + px : x;
    const long long orow = (static_cast<long long>(it.b) * Hout + oy) * Wout + ox;
#pragma unroll
    for (int ch = 0; ch < 2; ++ch) {
      const float* src = stg + (r2 * CF_TW + xl) * CF_STAGE_LD + half * 64 + ch * 32;
      const int n0 = n_base + ch * 32;
      float v[32];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (n0 + j * 8 >= p.Cout) {   // narrow output tile (conv_out): channels beyond Cout do not exist
#pragma unroll
          for (int i = 0; i < 8; ++i) v[j * 8 + i] = 0.f;
          continue;
        }
        const float4 a4 = *reinterpret_cast<const float4*>(src + j * 8);
        const float4 b4f = *reinterpret_cast<const float4*>(src + j * 8 + 4);
        const float r[8] = {a4.x, a4.y, a4.z, a4.w, b4f.x, b4f.y, b4f.z, b4f.w};
        float bv[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
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
        float rv[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (res != nullptr) {
          const uint4 r4 = *reinterpret_cast<const uint4*>(res + orow * p.Cout + n0 + j * 8);
          const uint32_t rw[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = H16::unpack(rw[i]);
            rv[2 * i] = f.x;
            rv[2 * i + 1] = f.y;
          }
        }
        uint32_t w16[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float a = r[2 * i] + bv[2 * i] + rv[2 * i];
          const float b = r[2 * i + 1] + bv[2 * i + 1] + rv[2 * i + 1];
          w16[i] = H16::pack(a, b);
          const float2 back = H16::unpack(w16[i]);   // statistics of what is STORED
          v[j * 8 + 2 * i] = back.x;
          v[j * 8 + 2 * i + 1] = back.y;
        }
        *reinterpret_cast<uint4*>(out + orow * p.Cout + n0 + j * 8) = make_uint4(w16[0], w16[1], w16[2], w16[3]);
      }
      if (p.out_partial != nullptr) {
        float* dst = st_my + ((r2 * 2 + ch) * 8) * 2;
        if (cpg_out == 4)
          cf_chunk_stats<4>(v, dst, lane);
        else if (cpg_out == 8)
          cf_chunk_stats<8>(v, dst, lane);
        else
          cf_chunk_stats<16>(v, dst, lane);
      }
    }
  }
  if (p.out_partial != nullptr) {
    // fold the four pixel quarters in fixed order (deterministic) and publish one (sum, sumsq) per 128-pixel row
    // segment and group
    named_bar_sync(1, 256);
    const int ng = 32 / cpg_out;
    const int per_row = 2 * 2 * ng;         // halves x chunks x groups of this tile, per output row
    if (tid < CF_R * per_row) {
      const int r2 = tid / per_row;
      const int rem = tid - r2 * per_row;
      const int hf = rem / (2 * ng);
      const int ch = (rem / ng) & 1;
      const int g = rem % ng;
      float s = 0.f, q = 0.f;
#pragma unroll
      for (int qd = 0; qd < 4; ++qd) {
        const float* src = sstat + ((hf * 4 + qd) * CF_R) * (2 * 8 * 2) + ((r2 * 2 + ch) * 8 + g) * 2;
        s += src[0];
        q += src[1];
      }
      const int oy = p.up ? 2 * (y0 + r2) + py : (y0 + r2);
      // slot: one per (output row, 128 consecutive stored pixels of one phase)
      const int slot = p.up ? ((oy * p.tiles_x + it.tx) * 2 + px) : (oy * p.tiles_x + it.tx);
      const int gidx = (it.nt * CF_BN + hf * 64 + ch * 32) / cpg_out + g;
      float* dst = p.out_partial + ((static_cast<long long>(it.b) * slots + slot) * p.out_G + gidx) * 2;
      dst[0] = s;
      dst[1] = q;
    }
  }
}

// w [Cout, 3, 3, Cin] -> wp [4 phases][Cout][2 x 2 taps][Cin]: the 3x3 taps that land on the same source pixel of a
// nearest-2x upsampled input, added in fp32 and rounded once.  Phase (py, px), tap (a, b):
//   py = 0: a = 0 <- ky {0}, a = 1 <- ky {1, 2};   py = 1: a = 0 <- ky {0, 1}, a = 1 <- ky {2}      (same for x)
template <typename T>
__global__ void conv_up_weights_kernel(const T* __restrict__ w, T* __restrict__ wp, int Cout, int Cin) {
  const long long total = 4LL * Cout * 4 * Cin;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % Cin);
    long long t = i / Cin;
    const int tap = static_cast<int>(t % 4);
    t /= 4;
    const int n = static_cast<int>(t % Cout);
    const int phase = static_cast<int>(t / Cout);
    const int py = phase >> 1, px = phase & 1, a = tap >> 1, b = tap & 1;
    const int ky0 = (py == 0) ? (a == 0 ? 0 : 1) : (a == 0 ? 0 : 2);
    const int ky1 = (py == 0) ? (a == 0 ? 0 : 2) : (a == 0 ? 1 : 2);
    const int kx0 = (px == 0) ? (b == 0 ? 0 : 1) : (b == 0 ? 0 : 2);
    const int kx1 = (px == 0) ? (b == 0 ? 0 : 2) : (b == 0 ? 1 : 2);
    float acc = 0.f;
    for (int ky = ky0; ky <= ky1; ++ky)
      for (int kx = kx0; kx <= kx1; ++kx) acc += Half16<T>::to_f(w[((static_cast<long long>(n) * 3 + ky) * 3 + kx) * Cin + c]);
    wp[i] = Half16<T>::from_f(acc);
  }
}

}  // namespace dk

using namespace dk;

static bool cf_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

extern "C" int dk_conv_fused_supported(int H, int W, int Cin, int Cout) {
  // Cout: whole 128-channel tiles, or ONE narrow tile of 8..120 channels (conv_out: the weight rows beyond Cout are
  // zero-filled by the TMA unit, the epilogue stores only the real channels)
  const bool cout_ok = Cout % CF_BN == 0 || (Cout > 0 && Cout < CF_BN && Cout % 8 == 0);
  return (W % CF_TW == 0 && H % (2 * CF_R) == 0 && Cin % 64 == 0 && Cin <= 512 && cout_ok) ? 1 : 0;
}

extern "C" int dk_conv_up_weights(dk_ctx* ctx, int dtype, const void* w, void* wp, int Cout, int Cin, void* stream_) {
  DK_REQUIRE(ctx != nullptr, "dk_conv_up_weights: null ctx");
  DkDeviceGuard dk_guard_(ctx);
  DK_REQUIRE(dtype == DK_BF16 || dtype == DK_FP16, "dk_conv_up_weights: bad dtype %d", dtype);
  DK_REQUIRE(w != nullptr && wp != nullptr && Cout > 0 && Cin > 0, "dk_conv_up_weights: bad arguments");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long total = 16LL * Cout * Cin;
  const int grid = static_cast<int>((total + 255) / 256 < 4096 ? (total + 255) / 256 : 4096);
  if (dtype == DK_BF16)
    conv_up_weights_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(w),
                                                                      static_cast<__nv_bfloat16*>(wp), Cout, Cin);
  else
    conv_up_weights_kernel<__half><<<grid, 256, 0, stream>>>(static_cast<const __half*>(w), static_cast<__half*>(wp), Cout, Cin);
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

// x NHWC [B, H, W, Cin]; w: [Cout, 3, 3, Cin] (up = 0) or the phase weights of dk_conv_up_weights [4*Cout, 4*Cin] (up = 1);
// out NHWC [B, H, W, Cout] (up = 0) / [B, 2H, 2W, Cout] (up = 1); res like out or NULL.
// gn_stats [B, G, 2] + gamma/beta [Cin] (+ silu) normalise the INPUT on the fly (NULL: raw input);
// out_partial [B, slots, out_G, 2] (slots = out pixels / 128) receives the output's GroupNorm partial sums (NULL: none).
extern "C" int dk_conv3x3_fused(dk_ctx* ctx, int dtype, const void* x, const void* w, const void* bias, const void* res,
                                void* out, int B, int H, int W, int Cin, int Cout, int up, const float* gn_stats,
                                const void* gamma, const void* beta, int G, int silu, float* out_partial, int out_G,
                                void* stream_) {
  DK_REQUIRE(ctx != nullptr, "dk_conv3x3_fused: null ctx");
  DkDeviceGuard dk_guard_(ctx);
  DK_REQUIRE(dtype == DK_BF16 || dtype == DK_FP16, "dk_conv3x3_fused: bad dtype %d", dtype);
  DK_REQUIRE(B > 0 && dk_conv_fused_supported(H, W, Cin, Cout),
             "dk_conv3x3_fused: needs W %% 128 == 0, H %% 4 == 0, Cin %% 64 == 0 (<= 512), Cout %% 128 == 0 or a multiple "
             "of 8 below 128 (got %dx%d, %d -> %d)",
             H, W, Cin, Cout);
  DK_REQUIRE(Cout % CF_BN == 0 || (up == 0 && out_partial == nullptr),
             "dk_conv3x3_fused: a narrow output tile (Cout = %d) has no upsampling and no output statistics", Cout);
  DK_REQUIRE(cf_aligned16(x) && cf_aligned16(w) && cf_aligned16(out) && (bias == nullptr || cf_aligned16(bias)) &&
                 (res == nullptr || cf_aligned16(res)),
             "dk_conv3x3_fused: buffers must be 16-byte aligned");
  DK_REQUIRE(gn_stats == nullptr || (gamma != nullptr && beta != nullptr && G > 0 && Cin % G == 0),
             "dk_conv3x3_fused: GroupNorm needs gamma, beta and G dividing Cin");
  DK_REQUIRE(gn_stats == nullptr || up == 0, "dk_conv3x3_fused: normalisation and upsampling are not combined");
  DK_REQUIRE(out_partial == nullptr || (out_G > 0 && Cout % out_G == 0 && (Cout / out_G == 4 || Cout / out_G == 8 || Cout / out_G == 16)),
             "dk_conv3x3_fused: output statistics need 4, 8 or 16 channels per group");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  ConvFParams p = {};
  p.B = B;
  p.H = H;
  p.W = W;
  p.Cin = Cin;
  p.Cout = Cout;
  p.up = up ? 1 : 0;
  p.tiles_x = W / CF_TW;
  p.tiles_y = H / CF_R;
  p.n_tiles = (Cout + CF_BN - 1) / CF_BN;
  p.bias = bias;
  p.res = res;
  p.out = out;
  p.gn_stats = gn_stats;
  p.gamma = gamma;
  p.beta = beta;
  p.G = G;
  p.silu = silu;
  p.out_partial = out_partial;
  p.out_G = out_G;

  CUtensorMap tmX, tmW;
  {
    const uint64_t dims[4] = {static_cast<uint64_t>(Cin), static_cast<uint64_t>(W), static_cast<uint64_t>(H),
                              static_cast<uint64_t>(B)};
    const uint64_t strides[3] = {static_cast<uint64_t>(Cin) * 2, static_cast<uint64_t>(W) * Cin * 2,
                                 static_cast<uint64_t>(H) * W * Cin * 2};
    const uint32_t box[4] = {64, CF_HW, CF_HR, 1};
    if (int rc = dk_make_tmap_16b(ctx, &tmX, x, 4, dims, strides, box)) return rc;
  }
  {
    const int taps = up ? 4 : 9;
    const uint64_t dims[2] = {static_cast<uint64_t>(taps) * Cin, static_cast<uint64_t>(up ? 4 : 1) * Cout};
    const uint64_t strides[1] = {static_cast<uint64_t>(taps) * Cin * 2};
    const uint32_t box[2] = {64, CF_BN};
    if (int rc = dk_make_tmap_16b(ctx, &tmW, w, 2, dims, strides, box)) return rc;
  }
  const long long items = static_cast<long long>(B) * p.tiles_y * p.tiles_x * (up ? 4 : 1) * p.n_tiles;
  DK_REQUIRE(items < (1LL << 31), "dk_conv3x3_fused: problem too large");
  if (dtype == DK_BF16) {
    auto kern = conv_fused_kernel<__nv_bfloat16>;
    static bool configured = false;
    if (!configured) {
      DK_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, CF_SMEM_BYTES));
      configured = true;
    }
    kern<<<static_cast<int>(items), CF_THREADS, CF_SMEM_BYTES, stream>>>(tmX, tmW, p);
  } else {
    auto kern = conv_fused_kernel<__half>;
    static bool configured = false;
    if (!configured) {
      DK_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, CF_SMEM_BYTES));
      configured = true;
    }
    kern<<<static_cast<int>(items), CF_THREADS, CF_SMEM_BYTES, stream>>>(tmX, tmW, p);
  }
  DK_LAUNCH_CHECK(ctx);
  return 0;
}
