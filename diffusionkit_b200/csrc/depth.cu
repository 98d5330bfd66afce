// FLUX.1 Depth's depth estimator (DESIGN.md §20): the kernels Depth Anything's DPT neck and head need beside the
// engine's GEMM, convolution, attention and LayerNorm.
//   dk_resample:       separable linear resampling of an NHWC map through per-axis tap tables made on the host
//                      (bilinear with either align_corners, PyTorch's bicubic and its antialiased bicubic); 16-bit or
//                      fp32 in and out, fp32 arithmetic; optionally BFL's depth / 127.5 - 1 replicated to 3 channels.
//   dk_depth_add_relu: sum = a (+ b) and relu(sum), each to its own buffer, 16-bit (the DPT pre-activations).
//   dk_depth_head:     relu(w . relu(x) + b) per pixel, the head's last 1 x 1 convolution to fp32 depth.
#include "common.cuh"
#include "host.h"

namespace dk {

template <typename T>
struct DepthVal {
  __device__ static __forceinline__ float to_f(T v) { return Half16<T>::to_f(v); }
  __device__ static __forceinline__ T from_f(float v) { return Half16<T>::from_f(v); }
};
template <>
struct DepthVal<float> {
  __device__ static __forceinline__ float to_f(float v) { return v; }
  __device__ static __forceinline__ float from_f(float v) { return v; }
};

// out(y, x, c) = sum_t wy[y, t] * sum_u wx[x, u] * in(y0[y] + t, x0[x] + u, c), rows then columns, in fp32.  A tap
// index outside the input is clamped (the host's tables never produce one; the clamp keeps a bad table in bounds).
// One thread per output element; mode 1 writes v / 127.5 - 1 to channels 0, 1 and 2 of a 3-channel output (C == 1).
template <typename Tin, typename Tout>
__global__ void resample_kernel(const Tin* __restrict__ in, Tout* __restrict__ out, int Hi, int Wi, int C, int Ho,
                                int Wo, const int* __restrict__ y0, const float* __restrict__ wy, int ty,
                                const int* __restrict__ x0, const float* __restrict__ wx, int tx, int mode) {
  const long long n = static_cast<long long>(Ho) * Wo * C;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    const long long p = i / C;
    const int x = static_cast<int>(p % Wo), y = static_cast<int>(p / Wo);
    float acc = 0.f;
    for (int t = 0; t < ty; ++t) {
      const int r = min(max(y0[y] + t, 0), Hi - 1);
      const Tin* row = in + static_cast<long long>(r) * Wi * C + c;
      float s = 0.f;
      for (int u = 0; u < tx; ++u) {
        const int q = min(max(x0[x] + u, 0), Wi - 1);
        s = __fmaf_rn(wx[static_cast<long long>(x) * tx + u], DepthVal<Tin>::to_f(row[static_cast<long long>(q) * C]),
                      s);
      }
      acc = __fmaf_rn(wy[static_cast<long long>(y) * ty + t], s, acc);
    }
    if (mode == 0) {
      out[i] = DepthVal<Tout>::from_f(acc);
    } else {
      const Tout v = DepthVal<Tout>::from_f(__fsub_rn(__fdiv_rn(acc, 127.5f), 1.f));
      out[3 * p] = v;
      out[3 * p + 1] = v;
      out[3 * p + 2] = v;
    }
  }
}

// sum = round(a + b) (b null: a), relu = max(sum, 0); either output may be null, and may alias a (in place).
template <typename T>
__global__ void depth_add_relu_kernel(const T* a, const T* b, T* sum, T* relu, long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    T v = a[i];
    if (b != nullptr) v = Half16<T>::from_f(__fadd_rn(Half16<T>::to_f(v), Half16<T>::to_f(b[i])));
    if (sum != nullptr) sum[i] = v;
    if (relu != nullptr) relu[i] = Half16<T>::from_f(fmaxf(Half16<T>::to_f(v), 0.f));
  }
}

// out[p] = max(((w[0] r0 + w[1] r1) + ...) + b, 0) with r_k = max(x[p, k], 0): every product and sum rounded on its
// own (no contraction), in channel order.
template <typename T>
__global__ void depth_head_kernel(const T* __restrict__ x, const float* __restrict__ w, float b, float* __restrict__ out,
                                  long long pixels, int C) {
  for (long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; p < pixels;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    const T* px = x + p * C;
    float acc = 0.f;
    for (int k = 0; k < C; ++k) acc = __fadd_rn(acc, __fmul_rn(w[k], fmaxf(Half16<T>::to_f(px[k]), 0.f)));
    out[p] = fmaxf(__fadd_rn(acc, b), 0.f);
  }
}

template <typename Tin, typename Tout>
static int launch_resample(dk_ctx* ctx, const void* in, void* out, int Hi, int Wi, int C, int Ho, int Wo,
                           const int* y0, const float* wy, int ty, const int* x0, const float* wx, int tx, int mode,
                           cudaStream_t stream) {
  const long long n = static_cast<long long>(Ho) * Wo * C;
  resample_kernel<Tin, Tout><<<dk_grid_for(n, 256, ctx->sm_count), 256, 0, stream>>>(
      static_cast<const Tin*>(in), static_cast<Tout*>(out), Hi, Wi, C, Ho, Wo, y0, wy, ty, x0, wx, tx, mode);
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

template <typename Tin>
static int resample_out(dk_ctx* ctx, int out_dtype, const void* in, void* out, int Hi, int Wi, int C, int Ho, int Wo,
                        const int* y0, const float* wy, int ty, const int* x0, const float* wx, int tx, int mode,
                        cudaStream_t stream) {
  if (out_dtype == DK_F32)
    return launch_resample<Tin, float>(ctx, in, out, Hi, Wi, C, Ho, Wo, y0, wy, ty, x0, wx, tx, mode, stream);
  if (out_dtype == DK_BF16)
    return launch_resample<Tin, __nv_bfloat16>(ctx, in, out, Hi, Wi, C, Ho, Wo, y0, wy, ty, x0, wx, tx, mode, stream);
  return launch_resample<Tin, __half>(ctx, in, out, Hi, Wi, C, Ho, Wo, y0, wy, ty, x0, wx, tx, mode, stream);
}

}  // namespace dk

using namespace dk;

extern "C" int dk_resample(dk_ctx* ctx, int in_dtype, int out_dtype, const void* in, void* out, int Hi, int Wi, int C,
                           int Ho, int Wo, const int* y0, const float* wy, int ty, const int* x0, const float* wx,
                           int tx, int mode, void* stream_) {
  DK_ENTRY(ctx);
  DK_REQUIRE(in_dtype == DK_BF16 || in_dtype == DK_FP16 || in_dtype == DK_F32, "dk_resample: bad input dtype %d",
             in_dtype);
  DK_REQUIRE(out_dtype == DK_BF16 || out_dtype == DK_FP16 || out_dtype == DK_F32, "dk_resample: bad output dtype %d",
             out_dtype);
  DK_REQUIRE(in != nullptr && out != nullptr && y0 != nullptr && wy != nullptr && x0 != nullptr && wx != nullptr,
             "dk_resample: in, out and the four tap tables are required");
  DK_REQUIRE(Hi > 0 && Wi > 0 && C > 0 && Ho > 0 && Wo > 0, "dk_resample: empty map %dx%dx%d -> %dx%d", Hi, Wi, C, Ho,
             Wo);
  DK_REQUIRE(static_cast<long long>(Hi) * Wi * C < (1ll << 40) && static_cast<long long>(Ho) * Wo * C * 3 < (1ll << 40),
             "dk_resample: map too large");
  DK_REQUIRE(ty >= 1 && ty <= 64 && tx >= 1 && tx <= 64, "dk_resample: taps per output must be 1..64, got %d, %d", ty,
             tx);
  DK_REQUIRE(mode == 0 || (mode == 1 && C == 1), "dk_resample: mode must be 0, or 1 with one input channel");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (in_dtype == DK_F32)
    return resample_out<float>(ctx, out_dtype, in, out, Hi, Wi, C, Ho, Wo, y0, wy, ty, x0, wx, tx, mode, stream);
  if (in_dtype == DK_BF16)
    return resample_out<__nv_bfloat16>(ctx, out_dtype, in, out, Hi, Wi, C, Ho, Wo, y0, wy, ty, x0, wx, tx, mode,
                                       stream);
  return resample_out<__half>(ctx, out_dtype, in, out, Hi, Wi, C, Ho, Wo, y0, wy, ty, x0, wx, tx, mode, stream);
}

extern "C" int dk_depth_add_relu(dk_ctx* ctx, int dtype, const void* a, const void* b, void* sum, void* relu,
                                 long long n, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(a != nullptr && (sum != nullptr || relu != nullptr), "dk_depth_add_relu: needs a and sum or relu");
  DK_REQUIRE(n > 0, "dk_depth_add_relu: empty tensor");
  const int grid = dk_grid_for(n, 256, ctx->sm_count);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, depth_add_relu_kernel<T><<<grid, 256, 0, stream>>>(
                         static_cast<const T*>(a), static_cast<const T*>(b), static_cast<T*>(sum),
                         static_cast<T*>(relu), n));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}

extern "C" int dk_depth_head(dk_ctx* ctx, int dtype, const void* x, const float* w, float b, float* out,
                             long long pixels, int C, void* stream_) {
  DK_ENTRY(ctx);
  DK_DTYPE_OK(dtype);
  DK_REQUIRE(x != nullptr && w != nullptr && out != nullptr, "dk_depth_head: x, w and out are required");
  DK_REQUIRE(pixels > 0 && C > 0 && C <= 1024, "dk_depth_head: needs pixels > 0 and 0 < C <= 1024, got %lld, %d",
             pixels, C);
  const int grid = dk_grid_for(pixels, 256, ctx->sm_count);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DK_DISPATCH(dtype, depth_head_kernel<T><<<grid, 256, 0, stream>>>(static_cast<const T*>(x), w, b, out, pixels, C));
  DK_LAUNCH_CHECK(ctx);
  return 0;
}
