// K1 / K7 — warp-specialised wgmma GEMM for sm_90a, and its implicit-GEMM 3x3 convolution variant.
//
//   out = epilogue( A[M,K] * W[N,K]^T )        (nn.Linear — reference mlx/mmdit.py:471-473,532,830-835, ...)
//   out = epilogue( conv3x3(x NHWC, w OHWI) )  (nn.Conv2d — reference mlx/vae.py:73-81,134-136,349-351,384)
//
// Structure (one 128 x BN output tile per CTA, 384 threads):
//   warpgroup 0 (warp 0): TMA producer — streams 128x64 A tiles and BNx64 W tiles (128B swizzle) through a
//                         STAGES-deep mbarrier ring.  For the convolution the A tile of tap (dy,dx) is a shifted 4-D
//                         TMA box of the NHWC input; out-of-bounds elements are zero-filled by the TMA unit, which
//                         *is* the zero padding — no im2col buffer exists anywhere.
//   warpgroups 1, 2     : MMA consumers — each owns 64 rows of the tile: wgmma m64nBNk16 from shared memory into
//                         register accumulators, one k-block group in flight while the next is issued.
//   epilogue            : the accumulators go through an fp32 staging tile in the (then idle) pipeline buffers, so
//                         that each thread owns one tile row: fused bias / GELU-erf / adaLN gate / residual, or
//                         QK-RMSNorm + RoPE on the q/k thirds of a packed QKV projection; 128-bit stores straight to
//                         the destination row (row remap = joint-sequence scatter).
#include <stdlib.h>

#include "common.cuh"
#include "gemm_epilogue.cuh"
#include "host.h"

namespace dk {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int GEMM_THREADS = 384;

template <int BN>
struct GemmCfg {
  static constexpr int STAGES = (BN == 256) ? 4 : (BN == 128 ? 6 : 8);
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int PIPE_BYTES = STAGES * (A_BYTES + B_BYTES);
  static constexpr int STAGE_LD = BN + 4;   // fp32 staging row stride (floats): +4 spreads the rows over the banks
  static_assert(PIPE_BYTES >= BM * STAGE_LD * 4, "the epilogue staging tile reuses the pipeline buffers");
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_BYTES = PIPE_BYTES + BAR_BYTES + 1024;  // +1024: manual alignment slack
};

// MODE 0: plain GEMM.  MODE 1: conv3x3 implicit GEMM (A via 4-D TMA boxes).
// B_MN: W operand given as [K, N] row-major (MN-major wgmma operand, transposed B).
template <typename T, int BN, bool B_MN, int MODE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmShape s,
                  const GemmEpi e, const ConvGeom g) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int A_BYTES = Cfg::A_BYTES;
  constexpr int B_BYTES = Cfg::B_BYTES;

  extern __shared__ uint8_t smem_raw[];
  // 128B-swizzled tiles need 1024-byte aligned bases.
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::PIPE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  // Grouped rasterisation: consecutive tile ids walk GM m-blocks for one n-block, so the CTAs resident at a time
  // share a band of A rows and a handful of W column blocks (L2 reuse).
  constexpr int GM = 16;
  int m_blk, n_blk;
  {
    const int tile = blockIdx.x;
    const int group_size = GM * s.num_n;
    const int group = tile / group_size;
    const int first_m = group * GM;
    const int gsz = min(s.num_m - first_m, GM);
    const int in_group = tile - group * group_size;
    m_blk = first_m + in_group % gsz;
    n_blk = in_group / gsz;
  }

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer, converged warp
    if (warp != 0) return;
    int img = 0, y0 = 0, x0 = 0;
    if (MODE == 1) {
      const int per_img = g.tiles_x * g.tiles_y;
      img = m_blk / per_img;
      const int t = m_blk - img * per_img;
      y0 = (t / g.tiles_x) * g.TH;
      x0 = (t % g.tiles_x) * g.TW;
    }
    uint32_t stage = 0, phase = 0;
    for (int kb = 0; kb < s.num_k; ++kb) {
      mbar_wait_warp(&empty_bar[stage], phase ^ 1);
      if (elect_one_sync()) {
        mbar_arrive_expect_tx(&full_bar[stage], A_BYTES + B_BYTES);
        uint8_t* a_dst = sA + stage * A_BYTES;
        uint8_t* b_dst = sB + stage * B_BYTES;
        if (MODE == 0) {
          tma_load_2d(a_dst, &tmA, &full_bar[stage], kb * BK, m_blk * BM);
        } else {
          const int tap = kb / g.cblocks;
          const int c0 = (kb - tap * g.cblocks) * BK;
          const int dy = tap / 3, dx = tap - dy * 3;
          tma_load_4d(a_dst, &tmA, &full_bar[stage], c0, x0 * g.stride + dx - g.pad, y0 * g.stride + dy - g.pad, img);
        }
        if (!B_MN) {
          tma_load_2d(b_dst, &tmB, &full_bar[stage], kb * BK, n_blk * BN);
        } else {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j)
            tma_load_2d(b_dst + j * (BK * 128), &tmB, &full_bar[stage], n_blk * BN + j * 64, kb * BK);
        }
      }
      __syncwarp();
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    return;
  }

  // -------------------------------------------------------------------- MMA consumers: rows 64*cw .. 64*cw+63
  const int cw = wg - 1;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  {
    uint32_t stage = 0, phase = 0, prev = 0;
    for (int kb = 0; kb < s.num_k; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_base = smem_u32(sA + stage * A_BYTES) + cw * 64 * 128;
      const uint32_t b_base = smem_u32(sB + stage * B_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t da = make_smem_desc_sw128(a_base + k * 32, 16, 1024);
        const uint64_t db = B_MN ? make_smem_desc_sw128(b_base + k * 16 * 128, BK * 128, 1024)
                                 : make_smem_desc_sw128(b_base + k * 32, 16, 1024);
        Wgmma<BN, Half16<T>::is_bf16, B_MN ? 1 : 0>::ss(acc, da, db, (kb | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      // the previous k-block's MMAs have retired: its stage can be refilled
      wgmma_wait<1>();
      if (kb > 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    reg_fence(acc);
  }

  // ------------------------------------------------------------------ epilogue (256 threads, thread = tile row)
  // every TMA load has landed and every MMA has retired once both warpgroups pass this barrier: the pipeline buffers
  // become the fp32 staging tile
  float* stg = reinterpret_cast<float*>(smem);
  named_bar_sync(1, 256);
  stage_acc_rows<BN>(stg, Cfg::STAGE_LD, cw * 64, acc);
  named_bar_sync(1, 256);

  const int ew = warp - 4;               // 0..7
  const int quarter = ew & 3;            // rows 32*quarter .. 32*quarter+31
  const int half = ew >> 2;              // which half of the tile's columns this warp drains
  constexpr int NCH = BN / 64;           // 32-column chunks per thread
  const int r_in_tile = quarter * 32 + lane;

  // destination rows
  bool row_ok;
  long long orow, rrow;
  int batch, pos = 0;
  if (MODE == 0) {
    const int m = m_blk * BM + r_in_tile;
    row_ok = m < s.M;
    batch = m / e.rpb;
    const int in_b = m - batch * e.rpb;
    pos = e.out_row_off + in_b;  // position in the joint sequence (RoPE)
    orow = static_cast<long long>(batch) * e.out_batch_rows + e.out_row_off + in_b;
    rrow = static_cast<long long>(batch) * e.res_batch_rows + e.res_row_off + in_b;
  } else {
    const int per_img = g.tiles_x * g.tiles_y;
    const int img = m_blk / per_img;
    const int t = m_blk - img * per_img;
    const int y = (t / g.tiles_x) * g.TH + r_in_tile / g.TW;
    const int x = (t % g.tiles_x) * g.TW + r_in_tile % g.TW;
    row_ok = (y < g.H) && (x < g.W);
    batch = img;
    orow = (static_cast<long long>(img) * g.H + y) * g.W + x;
    rrow = orow;
  }
  const float* srow = stg + r_in_tile * Cfg::STAGE_LD + half * (BN / 2);
  auto load32 = [&](int c, uint32_t (&r)[32]) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 v = *reinterpret_cast<const float4*>(srow + c + 4 * q);
      r[4 * q] = __float_as_uint(v.x);
      r[4 * q + 1] = __float_as_uint(v.y);
      r[4 * q + 2] = __float_as_uint(v.z);
      r[4 * q + 3] = __float_as_uint(v.w);
    }
  };
  gemm_epilogue_drain<T, NCH, MODE>(s, e, load32, n_blk * BN + half * (BN / 2), row_ok, orow, rrow, batch, pos);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
template <typename T, int BN, bool B_MN, int MODE>
static int launch_gemm_inst(dk_ctx* ctx, const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmShape& s,
                            const GemmEpi& e, const ConvGeom& g, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  auto kern = gemm_wgmma_kernel<T, BN, B_MN, MODE>;
  static bool configured = false;
  if (!configured) {
    DK_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    configured = true;
  }
  kern<<<s.num_m * s.num_n, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(tmA, tmB, s, e, g);
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

template <typename T, bool B_MN, int MODE>
static int launch_gemm_bn(dk_ctx* ctx, int bn, const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmShape& s,
                          const GemmEpi& e, const ConvGeom& g, cudaStream_t stream) {
  if (bn == 256) return launch_gemm_inst<T, 256, B_MN, MODE>(ctx, tmA, tmB, s, e, g, stream);
  if (bn == 128) return launch_gemm_inst<T, 128, B_MN, MODE>(ctx, tmA, tmB, s, e, g, stream);
  return launch_gemm_inst<T, 64, B_MN, MODE>(ctx, tmA, tmB, s, e, g, stream);
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

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace dk

using namespace dk;

extern "C" int dk_gemm(dk_ctx* ctx, const dk_gemm_args* a, void* stream_) {
  DK_REQUIRE(ctx != nullptr && a != nullptr, "dk_gemm: null argument");
  DkDeviceGuard dk_guard_(ctx);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_REQUIRE(a->dtype == DK_BF16 || a->dtype == DK_FP16, "dk_gemm: bad dtype %d", a->dtype);
  DK_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0, "dk_gemm: empty problem M=%d N=%d K=%d", a->M, a->N, a->K);
  DK_REQUIRE(a->N % 8 == 0 && a->K % 8 == 0, "dk_gemm: N (%d) and K (%d) must be multiples of 8", a->N, a->K);
  DK_REQUIRE(a->lda % 8 == 0 && a->ldw % 8 == 0 && a->ldc % 8 == 0, "dk_gemm: leading dims must be multiples of 8");
  DK_REQUIRE(aligned16(a->A) && aligned16(a->W) && aligned16(a->out), "dk_gemm: A/W/out must be 16-byte aligned");
  DK_REQUIRE(a->bias == nullptr || aligned16(a->bias), "dk_gemm: bias must be 16-byte aligned");
  DK_REQUIRE(a->gate == nullptr || (aligned16(a->gate) && a->gate_ld % 8 == 0), "dk_gemm: gate alignment");
  DK_REQUIRE(a->res == nullptr || (aligned16(a->res) && a->ldres % 8 == 0), "dk_gemm: residual alignment");

  GemmShape s = {};
  s.M = a->M;
  s.N = a->N;
  s.K = a->K;
  s.num_m = dk_ceil_div(a->M, BM);
  s.num_k = dk_ceil_div(a->K, BK);
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
  {
    static const int dbg = [] { const char* v = getenv("DK_GEMM_EPI_DEBUG"); return v ? atoi(v) : 0; }();
    e.debug = dbg;
  }
  e.qk_qw = a->qk_q_weight;
  e.qk_kw = a->qk_k_weight;
  e.qk_rope = a->qk_rope;
  e.qk_d = a->qk_head_dim;
  e.qk_h = a->qk_heads * a->qk_head_dim;
  e.qk_eps = a->qk_eps;
  if (e.qk_d != 0) {
    DK_REQUIRE(e.qk_d == 64 || e.qk_d == 128, "dk_gemm: fused QK norm/RoPE supports head dims 64 and 128 (got %d)", e.qk_d);
    DK_REQUIRE(a->N == 3 * e.qk_h && e.qk_h % 128 == 0, "dk_gemm: fused QK epilogue needs N == 3*heads*d, heads*d %% 128 == 0");
    DK_REQUIRE(!a->w_n_major && a->act == DK_ACT_NONE && a->gate == nullptr && a->res == nullptr,
               "dk_gemm: fused QK epilogue excludes act/gate/residual");
    DK_REQUIRE(a->qk_rope == nullptr || (reinterpret_cast<uintptr_t>(a->qk_rope) & 15u) == 0, "dk_gemm: rope table alignment");
  }
  ConvGeom g = {};

  CUtensorMap tmA, tmB;
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(a->K), static_cast<uint64_t>(a->M)};
    const uint64_t strides[1] = {static_cast<uint64_t>(a->lda) * 2};
    const uint32_t box[2] = {BK, BM};
    if (int rc = dk_make_tmap_16b(ctx, &tmA, a->A, 2, dims, strides, box)) return rc;
  }
  if (!a->w_n_major) {
    const uint64_t dims[2] = {static_cast<uint64_t>(a->K), static_cast<uint64_t>(a->N)};
    const uint64_t strides[1] = {static_cast<uint64_t>(a->ldw) * 2};
    const uint32_t box[2] = {BK, static_cast<uint32_t>(bn)};
    if (int rc = dk_make_tmap_16b(ctx, &tmB, a->W, 2, dims, strides, box)) return rc;
  } else {
    const uint64_t dims[2] = {static_cast<uint64_t>(a->N), static_cast<uint64_t>(a->K)};
    const uint64_t strides[1] = {static_cast<uint64_t>(a->ldw) * 2};
    const uint32_t box[2] = {64, BK};
    if (int rc = dk_make_tmap_16b(ctx, &tmB, a->W, 2, dims, strides, box)) return rc;
  }

  if (a->dtype == DK_BF16) {
    if (a->w_n_major) return launch_gemm_inst<__nv_bfloat16, 128, true, 0>(ctx, tmA, tmB, s, e, g, stream);
    return launch_gemm_bn<__nv_bfloat16, false, 0>(ctx, bn, tmA, tmB, s, e, g, stream);
  } else {
    if (a->w_n_major) return launch_gemm_inst<__half, 128, true, 0>(ctx, tmA, tmB, s, e, g, stream);
    return launch_gemm_bn<__half, false, 0>(ctx, bn, tmA, tmB, s, e, g, stream);
  }
}

static int conv3x3_impl(dk_ctx* ctx, int dtype, const void* x, const void* w, const void* bias, const void* res,
                        void* out, int B, int Hin, int Win, int Cin, int Cout, int stride, cudaStream_t stream) {
  DK_REQUIRE(ctx != nullptr, "dk_conv3x3: null ctx");
  DkDeviceGuard dk_guard_(ctx);
  DK_REQUIRE(dtype == DK_BF16 || dtype == DK_FP16, "dk_conv3x3: bad dtype %d", dtype);
  DK_REQUIRE(B > 0 && Hin > 0 && Win > 0, "dk_conv3x3: empty input");
  DK_REQUIRE(Cin % 64 == 0, "dk_conv3x3: Cin (%d) must be a multiple of 64 (pad the channels)", Cin);
  DK_REQUIRE(Cout % 8 == 0, "dk_conv3x3: Cout (%d) must be a multiple of 8 (pad the filters)", Cout);
  DK_REQUIRE(aligned16(x) && aligned16(w) && aligned16(out), "dk_conv3x3: x/w/out must be 16-byte aligned");
  DK_REQUIRE(bias == nullptr || aligned16(bias), "dk_conv3x3: bias alignment");
  DK_REQUIRE(res == nullptr || aligned16(res), "dk_conv3x3: residual alignment");
  DK_REQUIRE(stride == 1 || (Hin % 2 == 0 && Win % 2 == 0), "dk_conv3x3_s2: input size must be even (got %dx%d)", Hin, Win);

  const int H = Hin / stride, W = Win / stride;   // output size
  ConvGeom g;
  g.B = B;
  g.H = H;
  g.W = W;
  g.Cin = Cin;
  g.stride = stride;
  g.pad = stride == 1 ? 1 : 0;
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
    DK_REQUIRE(box[1] <= 256 && box[2] <= 256, "dk_conv3x3: TMA box too large");
    if (int rc = dk_make_tmap_16b(ctx, &tmA, x, 4, dims, strides, box, estr)) return rc;
  }
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(9 * Cin), static_cast<uint64_t>(Cout)};
    const uint64_t strides[1] = {static_cast<uint64_t>(9 * Cin) * 2};
    const uint32_t box[2] = {BK, static_cast<uint32_t>(bn)};
    if (int rc = dk_make_tmap_16b(ctx, &tmB, w, 2, dims, strides, box)) return rc;
  }
  if (dtype == DK_BF16) return launch_gemm_bn<__nv_bfloat16, false, 1>(ctx, bn, tmA, tmB, s, e, g, stream);
  return launch_gemm_bn<__half, false, 1>(ctx, bn, tmA, tmB, s, e, g, stream);
}

extern "C" int dk_conv3x3(dk_ctx* ctx, int dtype, const void* x, const void* w, const void* bias, const void* res,
                          void* out, int B, int H, int W, int Cin, int Cout, void* stream_) {
  return conv3x3_impl(ctx, dtype, x, w, bias, res, out, B, H, W, Cin, Cout, 1, static_cast<cudaStream_t>(stream_));
}

extern "C" int dk_conv3x3_s2(dk_ctx* ctx, int dtype, const void* x, const void* w, const void* bias, void* out, int B,
                             int H, int W, int Cin, int Cout, void* stream_) {
  return conv3x3_impl(ctx, dtype, x, w, bias, nullptr, out, B, H, W, Cin, Cout, 2, static_cast<cudaStream_t>(stream_));
}
