// K1 / K7 — warp-specialised, persistent wgmma GEMM for sm_90a, and its implicit-GEMM 3x3 convolution variant.
//
//   out = epilogue( A[M,K] * W[N,K]^T )        (nn.Linear — reference mlx/mmdit.py:471-473,532,830-835, ...)
//   out = epilogue( conv3x3(x NHWC, w OHWI) )  (nn.Conv2d — reference mlx/vae.py:73-81,134-136,349-351,384)
//
// Structure (2-CTA clusters along M, 384 threads per CTA, as many CTAs as can be resident):
//   schedule            : a cluster tile is (m-block pair, n-block); every cluster walks the cluster tiles with a static
//                         stride, grouped 16 m-blocks per group so the resident clusters share A bands and W column
//                         blocks in L2.  The two CTAs of a cluster take the two m-blocks of the pair.
//   warpgroup 0 (warp 0): TMA producer — streams its 128x64 A tile and half of the BNx64 W tile (128B swizzle) through
//                         a STAGES-deep mbarrier ring; the W half is multicast to both CTAs, so each CTA fetches
//                         A + W/2 per k-block.  Ring stage and phase carry over from tile to tile, so the next tile's
//                         loads start while the consumers are still in the epilogue.  For the convolution the A tile of
//                         tap (dy,dx) is a shifted 4-D TMA box of the NHWC input; out-of-bounds elements are zero-filled
//                         by the TMA unit, which *is* the zero padding — no im2col buffer exists anywhere.
//   warpgroups 1, 2     : MMA consumers — each owns 64 rows of the tile: wgmma m64nBNk16 from shared memory into
//                         register accumulators, one k-block group in flight while the next is issued.  A stage is
//                         released to the producers of both CTAs (it may be refilled only when both have read it).
//   epilogue            : on the accumulator fragments in registers (gemm_epilogue_tile): fused bias / GELU-erf /
//                         adaLN gate / residual, or QK-RMSNorm + RoPE on the q/k thirds of a packed QKV projection;
//                         16-bit results go through a dedicated shared-memory tile to 16-byte row stores (row remap =
//                         joint-sequence scatter).
#include <algorithm>

#include "common.cuh"
#include "gemm_epilogue.cuh"
#include "host.h"

namespace dk {

constexpr int BM = 128;
constexpr int ROW_BYTES = 128;    // one swizzled shared-memory row of an operand tile
constexpr int BK = ROW_BYTES / 2;  // K elements per k-block of the 16-bit operands
constexpr int GEMM_THREADS = 384;
constexpr int CLUSTER = 2;

// e4m3 operand element: one byte, only ever moved by TMA and read by wgmma
struct E4m3 {
  uint8_t bits;
};
// K elements per k-block: a tile row is 128 bytes whatever the element, so every byte count below (stage sizes, ring
// depth, descriptor steps) is the same for 16-bit and 8-bit operands
template <typename E>
constexpr int BK_OF = ROW_BYTES / static_cast<int>(sizeof(E));
static_assert(BK_OF<__nv_bfloat16> == BK && BK_OF<__half> == BK && BK_OF<E4m3> == 2 * BK, "k-block is one 128-byte row");

// Accumulation of the e4m3 MMAs: one fp32 fragment across all of K, like the 16-bit operands.  Hopper's FP8 wgmma is
// reported to keep fewer than 32 bits inside the tensor core (DeepSeek-V3 technical report, section 3.3.2); measured on
// an H100 at K = 15360 against an fp32 product of the same e4m3 operands this costs 3.4e-3 .. 3.7e-3 relative L2 after
// bf16 rounding (1.7e-3 is the rounding alone), inside the 4e-3 bound of the 16-bit kernel, while adding each k-block to
// a second fragment with CUDA-core adds (1.7e-3) ran at 0.65 of the rate.  DESIGN.md "FP8 linears".

template <int BN>
struct GemmCfg {
  static constexpr int STAGES = (BN == 256) ? 4 : (BN == 128 ? 6 : 8);
  static constexpr int A_BYTES = BM * ROW_BYTES;
  static constexpr int B_BYTES = BN * ROW_BYTES;
  static constexpr int PIPE_BYTES = STAGES * (A_BYTES + B_BYTES);
  static constexpr int EPI_BYTES = BM * (BN < 128 ? BN : 128) * 2;   // 16-bit output staging, one column pass
  static constexpr int RSTD_BYTES = BM * 2 * 4;                       // QK-RMSNorm: 1/rms per (row, head of a pass)
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_BYTES = PIPE_BYTES + EPI_BYTES + RSTD_BYTES + BAR_BYTES + 1024;  // +1024: alignment slack
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory per block");
  static_assert(A_BYTES == BM * BK * 2 && B_BYTES == BN * BK * 2, "stage sizes do not depend on the operand element");
};

// Cluster tile ct -> this CTA's (m-block, n-block).  When num_m is odd the partner of the last m-block gets
// m_blk == num_m: its loads are zero-filled and its epilogue stores nothing.
__device__ __forceinline__ void cluster_tile(int ct, const GemmShape& s, uint32_t rank, int& m_blk, int& n_blk) {
  constexpr int GC = 8;  // m-block pairs per rasterisation group (16 m-blocks)
  const int num_cm = (s.num_m + 1) >> 1;
  const int group_size = GC * s.num_n;
  const int group = ct / group_size;
  const int first = group * GC;
  const int gsz = min(num_cm - first, GC);
  const int in_group = ct - group * group_size;
  m_blk = 2 * (first + in_group % gsz) + static_cast<int>(rank);
  n_blk = in_group / gsz;
}

// MODE 0: plain GEMM.  MODE 1: conv3x3 implicit GEMM (A via 4-D TMA boxes).
// B_MN: W operand given as [K, N] row-major (MN-major wgmma operand, transposed B).
// T: 16-bit type of the epilogue's operands and of out.  E: element of A and W, T itself or E4m3 (K-major only,
// MODE 0 only; the epilogue then applies the row and column scales).
// GELU_TANH: the instance whose epilogue has the DK_ACT_GELU_TANH case (gemm_epilogue_tile).
// Launched in clusters of 2 along x with an even grid of at most (resident clusters) x 2 CTAs.
template <typename T, int BN, bool B_MN, int MODE, typename E, bool GELU_TANH>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmShape s,
                  const GemmEpi e, const ConvGeom g) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int A_BYTES = Cfg::A_BYTES;
  constexpr int B_BYTES = Cfg::B_BYTES;
  constexpr bool FP8 = sizeof(E) == 1;
  constexpr int BKE = BK_OF<E>;
  static_assert(!FP8 || (!B_MN && MODE == 0), "8-bit operands are K-major and have no convolution form");

  extern __shared__ uint8_t smem_raw[];
  // 128B-swizzled tiles need 1024-byte aligned bases.  The multicast writes the partner's shared memory at the same
  // offsets, so the layout must be identical in both CTAs (same kernel, same dynamic size, same base alignment).
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  uint8_t* stg = smem + Cfg::PIPE_BYTES;
  float* rstd = reinterpret_cast<float*>(stg + Cfg::EPI_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stg + Cfg::EPI_BYTES + Cfg::RSTD_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const uint32_t rank = cluster_ctarank();

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8 * CLUSTER);  // one arrive per consumer warp of each CTA of the cluster
    }
    fence_barrier_init();
  }
  // the partner's multicast loads and stage releases target this CTA's barriers: both must be initialised first
  cluster_sync();

  const int num_ctiles = ((s.num_m + 1) >> 1) * s.num_n;
  const int first_ct = blockIdx.x / CLUSTER;
  const int ct_stride = gridDim.x / CLUSTER;

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer, converged warp
    setmaxnreg_dec<40>();
    if (warp == 0) {
      uint32_t stage = 0, phase = 0;
      for (int ct = first_ct; ct < num_ctiles; ct += ct_stride) {
        int m_blk, n_blk;
        cluster_tile(ct, s, rank, m_blk, n_blk);
        int img = 0, y0 = 0, x0 = 0;
        if (MODE == 1) {
          const int per_img = g.tiles_x * g.tiles_y;
          img = m_blk / per_img;
          const int t = m_blk - img * per_img;
          y0 = (t / g.tiles_x) * g.TH;
          x0 = (t % g.tiles_x) * g.TW;
        }
        for (int kb = 0; kb < s.num_k; ++kb) {
          if (lane == 0) mbar_wait(&empty_bar[stage], phase ^ 1);
          __syncwarp();
          if (elect_one_sync()) {
            // A (own) + the whole W tile: this CTA's half and the partner's multicast half
            mbar_arrive_expect_tx(&full_bar[stage], A_BYTES + B_BYTES);
            uint8_t* a_dst = sA + stage * A_BYTES;
            uint8_t* b_dst = sB + stage * B_BYTES;
            if (MODE == 0) {
              tma_load_2d(a_dst, &tmA, &full_bar[stage], kb * BKE, m_blk * BM);
            } else {
              const int tap = kb / g.cblocks;
              const int c0 = (kb - tap * g.cblocks) * BK;
              const int dy = tap / 3, dx = tap - dy * 3;
              tma_load_4d(a_dst, &tmA, &full_bar[stage], c0, x0 * g.stride + dx - g.pad, y0 * g.stride + dy - g.pad,
                          img);
            }
            if (!B_MN) {
              // rows [rank*BN/2, (rank+1)*BN/2) of the W tile
              tma_load_2d_multicast(b_dst + rank * (B_BYTES / 2), &tmB, &full_bar[stage], kb * BKE,
                                    n_blk * BN + static_cast<int>(rank) * (BN / 2), 0x3);
            } else {
#pragma unroll
              for (int j = 0; j < BN / 64; ++j)
                if (j % CLUSTER == static_cast<int>(rank))
                  tma_load_2d_multicast(b_dst + j * (BK * 128), &tmB, &full_bar[stage], n_blk * BN + j * 64, kb * BK,
                                        0x3);
            }
          }
          __syncwarp();
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ MMA consumers: rows 64*cw .. 64*cw+63
    setmaxnreg_inc<232>();
    const int cw = wg - 1;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    uint32_t stage = 0, phase = 0;
    for (int ct = first_ct; ct < num_ctiles; ct += ct_stride) {
      int m_blk, n_blk;
      cluster_tile(ct, s, rank, m_blk, n_blk);
      uint32_t prev = 0;
      for (int kb = 0; kb < s.num_k; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_base = smem_u32(sA + stage * A_BYTES) + cw * 64 * 128;
        const uint32_t b_base = smem_u32(sB + stage * B_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < ROW_BYTES / 32; ++k) {   // one MMA per 32 bytes of K: k16 of 16-bit, k32 of 8-bit elements
          const uint64_t da = make_smem_desc_sw128(a_base + k * 32, 16, 1024);
          const uint64_t db = B_MN ? make_smem_desc_sw128(b_base + k * 16 * 128, BK * 128, 1024)
                                   : make_smem_desc_sw128(b_base + k * 32, 16, 1024);
          if constexpr (FP8)
            WgmmaE4m3<BN>::ss(acc, da, db, (kb | k) != 0 ? 1u : 0u);
          else
            Wgmma<BN, Half16<T>::is_bf16, B_MN ? 1 : 0>::ss(acc, da, db, (kb | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        // the previous k-block's MMAs have retired: its stage can be refilled, in both CTAs of the cluster
        wgmma_wait<1>();
        if (kb > 0 && lane == 0) {
          mbar_arrive_cluster(&empty_bar[prev], 0);
          mbar_arrive_cluster(&empty_bar[prev], 1);
        }
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      reg_fence(acc);
      if (lane == 0) {
        mbar_arrive_cluster(&empty_bar[prev], 0);
        mbar_arrive_cluster(&empty_bar[prev], 1);
      }
      gemm_epilogue_tile<T, BN, MODE, FP8, GELU_TANH>(acc, s, e, g, m_blk, n_blk, cw, stg + cw * (Cfg::EPI_BYTES / 2),
                                                      rstd + cw * 128);
    }
  }
  // no CTA may leave while its partner can still multicast into its shared memory or arrive on its barriers
  cluster_sync();
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
template <typename T, int BN, bool B_MN, int MODE, typename E = T, bool GELU_TANH = false>
static int launch_gemm_inst(const char* fn, dk_ctx* ctx, const CUtensorMap& tmA, const CUtensorMap& tmB,
                            const GemmShape& s, const GemmEpi& e, const ConvGeom& g, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_wgmma_kernel<T, BN, B_MN, MODE, E, GELU_TANH>;
  cudaLaunchAttribute cluster;
  cluster.id = cudaLaunchAttributeClusterDimension;
  cluster.val.clusterDim.x = CLUSTER;
  cluster.val.clusterDim.y = 1;
  cluster.val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(CLUSTER);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
  cfg.stream = stream;
  cfg.attrs = &cluster;
  cfg.numAttrs = 1;
  // resident clusters: a GPC whose SM count is odd leaves one SM without a partner
  int& max_clusters = ctx->max_clusters[reinterpret_cast<const void*>(kern)];
  if (max_clusters == 0) {
    if (int rc = dk_kernel_smem(ctx, reinterpret_cast<const void*>(kern), Cfg::SMEM_BYTES)) return rc;
    int n = 0;
    DK_CHECK_CUDA(cudaOccupancyMaxActiveClusters(&n, kern, &cfg));
    DK_REQUIRE(n > 0, "%s: no 2-CTA cluster of the GEMM kernel fits on the device", fn);
    max_clusters = n;
  }
  const int cluster_tiles = dk_ceil_div(s.num_m, CLUSTER) * s.num_n;
  cfg.gridDim = dim3(CLUSTER * std::min(cluster_tiles, max_clusters));
  DK_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, s, e, g));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

template <typename T, bool B_MN, int MODE, typename E = T, bool GELU_TANH = false>
static int launch_gemm_bn(const char* fn, dk_ctx* ctx, int bn, const CUtensorMap& tmA, const CUtensorMap& tmB,
                          const GemmShape& s, const GemmEpi& e, const ConvGeom& g, cudaStream_t stream) {
  if (bn == 256) return launch_gemm_inst<T, 256, B_MN, MODE, E, GELU_TANH>(fn, ctx, tmA, tmB, s, e, g, stream);
  if (bn == 128) return launch_gemm_inst<T, 128, B_MN, MODE, E, GELU_TANH>(fn, ctx, tmA, tmB, s, e, g, stream);
  return launch_gemm_inst<T, 64, B_MN, MODE, E, GELU_TANH>(fn, ctx, tmA, tmB, s, e, g, stream);
}

// Tile-N choice: 256 wide tiles keep the shared-memory operand traffic per MMA lowest; fall back to narrower tiles
// when N is small or when 256-wide tiles would leave most of the SMs idle.
static int pick_bn(const dk_ctx* ctx, int num_m, int N) {
  if (N <= 64) return 64;
  if (N <= 128) return 128;
  const int tiles256 = num_m * dk_ceil_div(N, 256);
  if (tiles256 >= ctx->sm_count) return 256;
  const int tiles128 = num_m * dk_ceil_div(N, 128);
  if (tiles128 >= ctx->sm_count || N % 256 != 0) return 128;
  return (tiles256 * 2 > ctx->sm_count) ? 256 : 128;
}

}  // namespace dk

using namespace dk;

// dk_gemm and dk_gemm_fp8.  The entry point named fn has run DK_ENTRY and DK_DTYPE_OK.  E is the element of A and W:
// the 16-bit type of a->dtype, or E4m3 with the two scale vectors.
static int gemm_impl(const char* fn, dk_ctx* ctx, const dk_gemm_args* a, const float* a_scale, const float* w_scale,
                     cudaStream_t stream) {
  const bool fp8 = a_scale != nullptr;
  const int esize = fp8 ? 1 : 2;
  const int kmul = 16 / esize;   // TMA global strides are multiples of 16 bytes
  DK_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0, "%s: empty problem M=%d N=%d K=%d", fn, a->M, a->N, a->K);
  DK_REQUIRE(a->N % 8 == 0 && a->K % kmul == 0, "%s: N (%d) must be a multiple of 8 and K (%d) of %d", fn, a->N, a->K,
             kmul);
  DK_REQUIRE(a->lda % kmul == 0 && a->ldw % kmul == 0 && a->ldc % 8 == 0,
             "%s: lda and ldw must be multiples of %d, ldc of 8", fn, kmul);
  DK_REQUIRE(dk_aligned16(a->A) && dk_aligned16(a->W) && dk_aligned16(a->out), "%s: A/W/out must be 16-byte aligned", fn);
  DK_REQUIRE(a->bias == nullptr || dk_aligned16(a->bias), "%s: bias must be 16-byte aligned", fn);
  DK_REQUIRE(a->gate == nullptr || (dk_aligned16(a->gate) && a->gate_ld % 8 == 0), "%s: gate alignment", fn);
  DK_REQUIRE(a->res == nullptr || (dk_aligned16(a->res) && a->ldres % 8 == 0), "%s: residual alignment", fn);

  const int bk = ROW_BYTES / esize;
  GemmShape s = {};
  s.M = a->M;
  s.N = a->N;
  s.K = a->K;
  s.num_m = dk_ceil_div(a->M, BM);
  s.num_k = dk_ceil_div(a->K, bk);
  const int bn = a->w_n_major ? 128 : (a->qk_head_dim != 0 ? 256 : pick_bn(ctx, s.num_m, a->N));
  s.num_n = dk_ceil_div(a->N, bn);

  GemmEpi e;
  e.out = a->out;
  e.ldc = a->ldc;
  e.bias = a->bias;
  e.gate = a->gate;
  e.gate_ld = a->gate_ld;
  e.res = a->res;
  e.ldres = a->ldres;
  e.rpb = a->rows_per_batch > 0 ? a->rows_per_batch : a->M;
  e.out_batch_rows = a->rows_per_batch > 0 ? a->out_batch_rows : a->M;
  e.out_row_off = a->out_row_off;
  e.res_batch_rows = a->rows_per_batch > 0 ? a->res_batch_rows : a->M;
  e.res_row_off = a->res_row_off;
  e.act = a->act;
  e.qk_qw = a->qk_q_weight;
  e.qk_kw = a->qk_k_weight;
  e.qk_rope = a->qk_rope;
  e.qk_d = a->qk_head_dim;
  e.qk_h = a->qk_heads * a->qk_head_dim;
  e.qk_eps = a->qk_eps;
  e.a_scale = a_scale;
  e.w_scale = w_scale;
  if (e.qk_d != 0) {
    DK_REQUIRE(e.qk_d == 64 || e.qk_d == 128, "%s: fused QK norm/RoPE supports head dims 64 and 128 (got %d)", fn, e.qk_d);
    DK_REQUIRE(a->N == 3 * e.qk_h && e.qk_h % 128 == 0, "%s: fused QK epilogue needs N == 3*heads*d, heads*d %% 128 == 0", fn);
    DK_REQUIRE(!a->w_n_major && a->act == DK_ACT_NONE && a->gate == nullptr && a->res == nullptr,
               "%s: fused QK epilogue excludes act/gate/residual", fn);
    DK_REQUIRE(a->qk_rope == nullptr || dk_aligned16(a->qk_rope), "%s: rope table alignment", fn);
  }
  DK_REQUIRE(a->act != DK_ACT_GELU_TANH || (!fp8 && !a->w_n_major),
             "%s: the tanh-GELU epilogue runs on 16-bit K-major operands only", fn);
  ConvGeom g = {};

  CUtensorMap tmA, tmB;
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(a->K), static_cast<uint64_t>(a->M)};
    const uint64_t strides[1] = {static_cast<uint64_t>(a->lda) * esize};
    const uint32_t box[2] = {static_cast<uint32_t>(bk), BM};
    if (int rc = dk_make_tmap(ctx, &tmA, esize, a->A, 2, dims, strides, box)) return rc;
  }
  if (!a->w_n_major) {
    const uint64_t dims[2] = {static_cast<uint64_t>(a->K), static_cast<uint64_t>(a->N)};
    const uint64_t strides[1] = {static_cast<uint64_t>(a->ldw) * esize};
    const uint32_t box[2] = {static_cast<uint32_t>(bk), static_cast<uint32_t>(bn / CLUSTER)};   // each CTA of a cluster loads half the tile
    if (int rc = dk_make_tmap(ctx, &tmB, esize, a->W, 2, dims, strides, box)) return rc;
  } else {
    const uint64_t dims[2] = {static_cast<uint64_t>(a->N), static_cast<uint64_t>(a->K)};
    const uint64_t strides[1] = {static_cast<uint64_t>(a->ldw) * 2};
    const uint32_t box[2] = {64, BK};
    if (int rc = dk_make_tmap_16b(ctx, &tmB, a->W, 2, dims, strides, box)) return rc;
  }

  DK_DISPATCH(a->dtype, {
    if (fp8) return launch_gemm_bn<T, false, 0, E4m3>(fn, ctx, bn, tmA, tmB, s, e, g, stream);
    if (a->w_n_major) return launch_gemm_inst<T, 128, true, 0>(fn, ctx, tmA, tmB, s, e, g, stream);
    if (a->act == DK_ACT_GELU_TANH) return launch_gemm_bn<T, false, 0, T, true>(fn, ctx, bn, tmA, tmB, s, e, g, stream);
    return launch_gemm_bn<T, false, 0>(fn, ctx, bn, tmA, tmB, s, e, g, stream);
  });
}

extern "C" int dk_gemm(dk_ctx* ctx, const dk_gemm_args* a, void* stream_) {
  DK_ENTRY(ctx);
  DK_REQUIRE(a != nullptr, "dk_gemm: null argument");
  DK_DTYPE_OK(a->dtype);
  return gemm_impl(__func__, ctx, a, nullptr, nullptr, static_cast<cudaStream_t>(stream_));
}

extern "C" int dk_gemm_fp8(dk_ctx* ctx, const dk_gemm_args* a, const float* a_scale, const float* w_scale,
                           void* stream_) {
  DK_ENTRY(ctx);
  DK_REQUIRE(a != nullptr, "dk_gemm_fp8: null argument");
  DK_DTYPE_OK(a->dtype);
  DK_REQUIRE(!a->w_n_major, "dk_gemm_fp8: e4m3 operands are K-major only (w_n_major is not supported)");
  DK_REQUIRE(a_scale != nullptr && w_scale != nullptr, "dk_gemm_fp8: a_scale and w_scale are required");
  DK_REQUIRE(dk_aligned16(a_scale) && dk_aligned16(w_scale), "dk_gemm_fp8: a_scale/w_scale must be 16-byte aligned");
  return gemm_impl(__func__, ctx, a, a_scale, w_scale, static_cast<cudaStream_t>(stream_));
}

// The entry point named fn has run DK_ENTRY and DK_DTYPE_OK.
static int conv3x3_impl(const char* fn, dk_ctx* ctx, int dtype, const void* x, const void* w, const void* bias,
                        const void* res, void* out, int B, int Hin, int Win, int Cin, int Cout, int stride, int pad,
                        cudaStream_t stream) {
  DK_REQUIRE(B > 0 && Hin > 0 && Win > 0, "%s: empty input", fn);
  DK_REQUIRE(Cin % 64 == 0, "%s: Cin (%d) must be a multiple of 64 (pad the channels)", fn, Cin);
  DK_REQUIRE(Cout % 8 == 0, "%s: Cout (%d) must be a multiple of 8 (pad the filters)", fn, Cout);
  DK_REQUIRE(dk_aligned16(x) && dk_aligned16(w) && dk_aligned16(out), "%s: x/w/out must be 16-byte aligned", fn);
  DK_REQUIRE(bias == nullptr || dk_aligned16(bias), "%s: bias alignment", fn);
  DK_REQUIRE(res == nullptr || dk_aligned16(res), "%s: residual alignment", fn);
  DK_REQUIRE(stride == 1 || pad == 1 || (Hin % 2 == 0 && Win % 2 == 0), "%s: input size must be even (got %dx%d)", fn,
             Hin, Win);

  // output size: stride 1 keeps it; stride 2 halves it (pad 0: even input), or rounds up with a pad of 1 on every side
  const int H = (Hin + (stride - 1) * pad) / stride, W = (Win + (stride - 1) * pad) / stride;
  ConvGeom g;
  g.B = B;
  g.H = H;
  g.W = W;
  g.Cin = Cin;
  g.stride = stride;
  g.pad = pad;
  if (W < 128 && 128 % W == 0) {
    g.TW = W;
    g.TH = 128 / W;
  } else {
    g.TW = 128;
    g.TH = 1;
  }
  g.tiles_x = dk_ceil_div(W, g.TW);
  g.tiles_y = dk_ceil_div(H, g.TH);
  g.cblocks = Cin / 64;

  GemmShape s = {};
  s.M = B * H * W;
  s.N = Cout;
  s.K = 9 * Cin;
  s.num_m = B * g.tiles_x * g.tiles_y;
  s.num_k = 9 * g.cblocks;
  const int bn = pick_bn(ctx, s.num_m, Cout);
  s.num_n = dk_ceil_div(Cout, bn);

  GemmEpi e = {};
  e.out = out;
  e.ldc = Cout;
  e.bias = bias;
  e.res = res;
  e.ldres = Cout;
  e.rpb = 1;
  e.act = DK_ACT_NONE;

  CUtensorMap tmA, tmB;
  {
    const uint64_t dims[4] = {static_cast<uint64_t>(Cin), static_cast<uint64_t>(Win), static_cast<uint64_t>(Hin),
                              static_cast<uint64_t>(B)};
    const uint64_t strides[3] = {static_cast<uint64_t>(Cin) * 2, static_cast<uint64_t>(Win) * Cin * 2,
                                 static_cast<uint64_t>(Hin) * Win * Cin * 2};
    // strided traversal: N elements with stride s need a box entry of N * s
    const uint32_t box[4] = {BK, static_cast<uint32_t>(g.TW * stride), static_cast<uint32_t>(g.TH * stride), 1};
    const uint32_t estr[4] = {1, static_cast<uint32_t>(stride), static_cast<uint32_t>(stride), 1};
    DK_REQUIRE(box[1] <= 256 && box[2] <= 256, "%s: TMA box too large", fn);
    if (int rc = dk_make_tmap_16b(ctx, &tmA, x, 4, dims, strides, box, estr)) return rc;
  }
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(9 * Cin), static_cast<uint64_t>(Cout)};
    const uint64_t strides[1] = {static_cast<uint64_t>(9 * Cin) * 2};
    const uint32_t box[2] = {BK, static_cast<uint32_t>(bn / CLUSTER)};
    if (int rc = dk_make_tmap_16b(ctx, &tmB, w, 2, dims, strides, box)) return rc;
  }
  DK_DISPATCH(dtype, return launch_gemm_bn<T, false, 1>(fn, ctx, bn, tmA, tmB, s, e, g, stream));
}

extern "C" int dk_conv3x3(dk_ctx* ctx, int dtype, const void* x, const void* w, const void* bias, const void* res,
                          void* out, int B, int H, int W, int Cin, int Cout, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  return conv3x3_impl(__func__, ctx, dtype, x, w, bias, res, out, B, H, W, Cin, Cout, 1, 1,
                      static_cast<cudaStream_t>(stream_));
}

extern "C" int dk_conv3x3_s2(dk_ctx* ctx, int dtype, const void* x, const void* w, const void* bias, void* out, int B,
                             int H, int W, int Cin, int Cout, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  return conv3x3_impl(__func__, ctx, dtype, x, w, bias, nullptr, out, B, H, W, Cin, Cout, 2, 0,
                      static_cast<cudaStream_t>(stream_));
}

// The taps of output pixel (y, x) start at input (2y - 1, 2x - 1): the negative coordinate and the row / column past an
// odd input's end are zero-filled by the TMA unit, so an odd size needs no special case.
extern "C" int dk_conv3x3_s2_p1(dk_ctx* ctx, int dtype, const void* x, const void* w, const void* bias, void* out,
                                int B, int H, int W, int Cin, int Cout, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  return conv3x3_impl(__func__, ctx, dtype, x, w, bias, nullptr, out, B, H, W, Cin, Cout, 2, 1,
                      static_cast<cudaStream_t>(stream_));
}
