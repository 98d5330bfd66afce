// K3 — attention forward softmax(scale * Q K^T) V for sm_90a: wgmma with S and O accumulators in registers,
// TMA-fed 128B-swizzled Q/K/V tiles, online softmax in registers, P fed back to the PV wgmma as a register operand.
// Replaces mx.fast.scaled_dot_product_attention (reference mlx/mmdit.py:562-563,643,687-688,736): no mask,
// non-causal, joint [text|image] sequence, head dim 64 (SD3) or 128 (FLUX).
//
// One CTA per (128-row Q tile, head, batch), 384 threads:
//   warpgroup 0 (warp 0): TMA producer — Q once, then K and V tiles of 128 keys through a two-deep ring (K and V on
//                         separate barriers, so S = Q K^T starts before V has landed)
//   warpgroups 1, 2     : 64 query rows each — S = Q K^T (m64n128, A and B from shared memory), masked online softmax
//                         on the S fragment (a row is spread over the four lanes of a quad), O = O * alpha + P V
//                         (m64nD, P from registers: the S accumulator layout of 16 key columns IS the A fragment
//                         layout of one k16 step), O / l -> global.
#include "common.cuh"
#include "host.h"

namespace dk {

constexpr int ATT_BQ = 128;
constexpr int ATT_BKV = 128;
constexpr int ATT_THREADS = 384;

struct AttParams {
  int B, S, heads, split;
  float scale_log2;  // scale * log2(e)
  void* out0;
  long long ld0;
  void* out1;
  long long ld1;
};

// one 128-row Q tile per CTA, K / V ring of KS tiles of 128 keys
template <int D>
struct AttCfg {
  static constexpr int KS = 2;
  static constexpr int TILE_BYTES = 128 * D * 2;
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = TILE_BYTES;
  static constexpr int OFF_V = OFF_K + KS * TILE_BYTES;
  static constexpr int OFF_BAR = OFF_V + KS * TILE_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
};

template <typename T, int D>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tm, const AttParams p) {
  using H16 = Half16<T>;
  using Cfg = AttCfg<D>;
  constexpr int KS = Cfg::KS;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem + Cfg::OFF_Q;
  uint8_t* sK = smem + Cfg::OFF_K;
  uint8_t* sV = smem + Cfg::OFF_V;
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* k_full = q_full + 1;
  uint64_t* v_full = k_full + KS;
  uint64_t* kv_empty = v_full + KS;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int q0 = blockIdx.x * ATT_BQ;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int h = p.heads * D;
  const int row0 = b * p.S;               // first row of this batch in the packed [B*S, 3h] tensor
  const int nkv = (p.S + ATT_BKV - 1) / ATT_BKV;
  constexpr uint32_t TILE_BYTES = ATT_BKV * D * 2;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm);
    mbar_init(q_full, 1);
    for (int i = 0; i < KS; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&kv_empty[i], 8);   // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer, converged warp
    if (warp != 0) return;
    if (elect_one_sync()) {
      mbar_arrive_expect_tx(q_full, ATT_BQ * D * 2);
#pragma unroll
      for (int c = 0; c < D / 64; ++c) tma_load_2d(sQ + c * (ATT_BQ * 128), &tm, q_full, head * D + c * 64, row0 + q0);
    }
    __syncwarp();
    uint32_t stage = 0, phase = 0;
    for (int j = 0; j < nkv; ++j) {
      mbar_wait_warp(&kv_empty[stage], phase ^ 1);
      if (elect_one_sync()) {
        const int kr = row0 + j * ATT_BKV;
        mbar_arrive_expect_tx(&k_full[stage], TILE_BYTES);
#pragma unroll
        for (int c = 0; c < D / 64; ++c)
          tma_load_2d(sK + stage * TILE_BYTES + c * (ATT_BKV * 128), &tm, &k_full[stage], h + head * D + c * 64, kr);
        mbar_arrive_expect_tx(&v_full[stage], TILE_BYTES);
#pragma unroll
        for (int c = 0; c < D / 64; ++c)
          tma_load_2d(sV + stage * TILE_BYTES + c * (ATT_BKV * 128), &tm, &v_full[stage], 2 * h + head * D + c * 64, kr);
      }
      __syncwarp();
      if (++stage == KS) {
        stage = 0;
        phase ^= 1;
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: query rows q0 + 64*cw ..
  const int cw = wg - 1;
  const float sl2 = p.scale_log2;
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};   // running max (log2 domain) of rows lane/4 and lane/4 + 8
  float l_run[2] = {0.f, 0.f};               // this thread's share of the running row sums
  const int col0 = 2 * (lane & 3);

  mbar_wait(q_full, 0);
  const uint32_t q_base = smem_u32(sQ) + cw * 64 * 128;
  uint32_t stage = 0, phase = 0;
  for (int j = 0; j < nkv; ++j) {
    const int kv_valid = p.S - j * ATT_BKV;
    const uint32_t k_base = smem_u32(sK + stage * TILE_BYTES);
    const uint32_t v_base = smem_u32(sV + stage * TILE_BYTES);
    float s[ATT_BKV / 2];
    mbar_wait(&k_full[stage], phase);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const uint32_t koff = (kk >> 2) * (ATT_BKV * 128) + (kk & 3) * 32;
      Wgmma<ATT_BKV, H16::is_bf16, 0>::ss(s, make_smem_desc_sw128(q_base + (kk >> 2) * (ATT_BQ * 128) + (kk & 3) * 32, 16, 1024),
                                         make_smem_desc_sw128(k_base + koff, 16, 1024), kk != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);

    // masked online softmax; s[4*jj + 2*i + e] is row lane/4 + 8i, key 8*jj + col0 + e
    float alpha[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < ATT_BKV / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = s[4 * jj + 2 * i + e];
          if (kv_valid < ATT_BKV && 8 * jj + col0 + e >= kv_valid) v = -INFINITY;   // only the last tile is ragged
          mx = fmaxf(mx, v);
        }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[i], mx * sl2);
      alpha[i] = ex2_approx(m_run[i] - m_new);
      m_run[i] = m_new;
      float ls = 0.f;
#pragma unroll
      for (int jj = 0; jj < ATT_BKV / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = s[4 * jj + 2 * i + e];
          v = ex2_approx(fmaf(v, sl2, -m_new));
          ls += v;
        }
      l_run[i] = l_run[i] * alpha[i] + ls;
    }
#pragma unroll
    for (int jj = 0; jj < D / 8; ++jj)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        o[4 * jj + 2 * i] *= alpha[i];
        o[4 * jj + 2 * i + 1] *= alpha[i];
      }
    uint32_t pa[ATT_BKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < ATT_BKV / 16; ++kk) {
      pa[kk][0] = H16::pack(s[8 * kk + 0], s[8 * kk + 1]);
      pa[kk][1] = H16::pack(s[8 * kk + 2], s[8 * kk + 3]);
      pa[kk][2] = H16::pack(s[8 * kk + 4], s[8 * kk + 5]);
      pa[kk][3] = H16::pack(s[8 * kk + 6], s[8 * kk + 7]);
    }

    // O += P V: V tile rows = keys (K of the MMA), 128-byte lines = 64 head-dim columns (MN-major, transposed B)
    mbar_wait(&v_full[stage], phase);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < ATT_BKV / 16; ++kk)
      Wgmma<D, H16::is_bf16, 1>::rs(o, pa[kk], make_smem_desc_sw128(v_base + kk * 16 * 128, ATT_BKV * 128, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[stage]);
    if (++stage == KS) {
      stage = 0;
      phase ^= 1;
    }
  }

  // epilogue: complete the row sums over the quad, O / l -> global
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float l = l_run[i];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv_l = 1.0f / l;
    const int s_idx = q0 + cw * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
    if (s_idx >= p.S) continue;
    T* dst;
    if (s_idx < p.split)
      dst = reinterpret_cast<T*>(p.out0) + (static_cast<long long>(b) * p.split + s_idx) * p.ld0 + head * D;
    else
      dst = reinterpret_cast<T*>(p.out1) + (static_cast<long long>(b) * (p.S - p.split) + (s_idx - p.split)) * p.ld1 +
            head * D;
#pragma unroll
    for (int jj = 0; jj < D / 8; ++jj)
      *reinterpret_cast<uint32_t*>(dst + 8 * jj + col0) =
          H16::pack(o[4 * jj + 2 * i] * inv_l, o[4 * jj + 2 * i + 1] * inv_l);
  }
}

template <typename T, int D>
static int launch_attention(dk_ctx* ctx, const CUtensorMap& tm, const AttParams& p, cudaStream_t stream) {
  auto kern = attention_fwd_kernel<T, D>;
  if (int rc = dk_kernel_smem(ctx, reinterpret_cast<const void*>(kern), AttCfg<D>::SMEM_BYTES)) return rc;
  dim3 grid(dk_ceil_div(p.S, ATT_BQ), p.heads, p.B);
  kern<<<grid, ATT_THREADS, AttCfg<D>::SMEM_BYTES, stream>>>(tm, p);
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

}  // namespace dk

using namespace dk;

extern "C" int dk_attention_fwd(dk_ctx* ctx, int dtype, const void* qkv, int B, int S, int heads, int d, float scale,
                                int split, void* out0, long long ld0, void* out1, long long ld1, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(d == 64 || d == 128, "dk_attention_fwd: head dim %d unsupported (64 or 128)", d);
  DK_REQUIRE(B > 0 && S > 0 && heads > 0, "dk_attention_fwd: empty problem");
  DK_REQUIRE(split >= 0 && split <= S, "dk_attention_fwd: split %d outside [0, %d]", split, S);
  DK_REQUIRE(out0 != nullptr || split == 0, "dk_attention_fwd: out0 is NULL");
  DK_REQUIRE(out1 != nullptr || split == S, "dk_attention_fwd: out1 is NULL but split < S");
  DK_REQUIRE(ld0 % 8 == 0 && ld1 % 8 == 0, "dk_attention_fwd: output leading dims must be multiples of 8");
  DK_REQUIRE(dk_aligned16(qkv) && dk_aligned16(out0) && dk_aligned16(out1),
             "dk_attention_fwd: buffers must be 16-byte aligned");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int h = heads * d;
  CUtensorMap tm;
  const uint64_t dims[2] = {static_cast<uint64_t>(3 * h), static_cast<uint64_t>(B) * S};
  const uint64_t strides[1] = {static_cast<uint64_t>(3 * h) * 2};
  const uint32_t box[2] = {64, 128};
  if (int rc = dk_make_tmap_16b(ctx, &tm, qkv, 2, dims, strides, box)) return rc;
  AttParams p;
  p.B = B;
  p.S = S;
  p.heads = heads;
  p.split = split;
  p.scale_log2 = scale * 1.44269504088896341f;
  p.out0 = out0;
  p.ld0 = ld0;
  p.out1 = out1;
  p.ld1 = ld1;
  DK_DISPATCH(dtype, {
    if (d == 128) return launch_attention<T, 128>(ctx, tm, p, stream);
    return launch_attention<T, 64>(ctx, tm, p, stream);
  });
}
