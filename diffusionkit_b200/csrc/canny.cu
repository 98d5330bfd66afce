// FLUX.1 Canny [dev]'s preprocessor (DESIGN.md §19): OpenCV's cv2.Canny(img, low, high) with the L1 gradient, on a
// 3-channel uint8 image whose values first go through a 256-entry table (BFL's float round trip).  Five launches:
//   1. canny_grad_kernel:   table, 3 x 3 Sobel dx / dy per channel with replicated borders, the channel of largest
//                           |dx| + |dy| (first wins a tie) -> (dx, dy) per pixel;
//   2. canny_nms_kernel:    non-maximum suppression in OpenCV's integer tangent test, magnitude 0 outside the image,
//                           then 0 / candidate (m > low) / strong (m > high); every pixel's union-find label is set;
//   3. canny_merge_kernel:  every candidate is united with its candidate neighbours W, NW, N and NE (each 8-connected
//                           pair once) by lock-free union-find on labels that only decrease;
//   4. canny_resolve_kernel: each candidate's label becomes its root, and the root of every strong pixel is flagged;
//   5. canny_edges_kernel:  255 in all three channels for a candidate whose root is flagged, 0 elsewhere.
// After launch 3 the labels describe the 8-connected components of the candidates exactly, so the output is the exact
// hysteresis fixpoint in a fixed number of launches with no host synchronisation.
#include "host.h"

namespace dk {

__device__ __forceinline__ int canny_px(const uint8_t* __restrict__ img, const uint8_t* __restrict__ lut, int H, int W,
                                        int C, int y, int x, int c) {
  y = min(max(y, 0), H - 1);
  x = min(max(x, 0), W - 1);
  return lut[img[(static_cast<long long>(y) * W + x) * C + c]];
}

// One thread per pixel: Sobel of the three table-mapped channels, the channel of largest L1 magnitude
__global__ void canny_grad_kernel(const uint8_t* __restrict__ img, const uint8_t* __restrict__ lut,
                                  short2* __restrict__ dxy, int H, int W, int C) {
  const long long n = static_cast<long long>(H) * W;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int y = static_cast<int>(i / W), x = static_cast<int>(i - static_cast<long long>(y) * W);
    int best_dx = 0, best_dy = 0, best_m = -1;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int a = canny_px(img, lut, H, W, C, y - 1, x - 1, c), b = canny_px(img, lut, H, W, C, y - 1, x, c),
                d = canny_px(img, lut, H, W, C, y - 1, x + 1, c), e = canny_px(img, lut, H, W, C, y, x - 1, c),
                f = canny_px(img, lut, H, W, C, y, x + 1, c), g = canny_px(img, lut, H, W, C, y + 1, x - 1, c),
                h = canny_px(img, lut, H, W, C, y + 1, x, c), k = canny_px(img, lut, H, W, C, y + 1, x + 1, c);
      const int dx = (d + 2 * f + k) - (a + 2 * e + g);
      const int dy = (g + 2 * h + k) - (a + 2 * b + d);
      const int m = abs(dx) + abs(dy);
      if (m > best_m) {
        best_m = m;
        best_dx = dx;
        best_dy = dy;
      }
    }
    dxy[i] = make_short2(static_cast<short>(best_dx), static_cast<short>(best_dy));
  }
}

__device__ __forceinline__ int canny_mag(const short2* __restrict__ dxy, int H, int W, int y, int x) {
  if (y < 0 || y >= H || x < 0 || x >= W) return 0;
  const short2 v = dxy[static_cast<long long>(y) * W + x];
  return abs(static_cast<int>(v.x)) + abs(static_cast<int>(v.y));
}

// cls: 0 none, 1 candidate, 2 strong.  label = own index (candidates) or -1; flag = 0.
__global__ void canny_nms_kernel(const short2* __restrict__ dxy, uint8_t* __restrict__ cls, int* __restrict__ label,
                                 uint8_t* __restrict__ flag, int H, int W, int low, int high) {
  const long long n = static_cast<long long>(H) * W;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int y = static_cast<int>(i / W), x = static_cast<int>(i - static_cast<long long>(y) * W);
    const short2 v = dxy[i];
    const int dx = v.x, dy = v.y;
    const int ax = abs(dx), m = ax + abs(dy);
    uint8_t k = 0;
    if (m > low) {
      const int yy = abs(dy) << 15, tg22x = ax * 13573;
      bool keep;
      if (yy < tg22x) {
        keep = m > canny_mag(dxy, H, W, y, x - 1) && m >= canny_mag(dxy, H, W, y, x + 1);
      } else if (yy > tg22x + (ax << 16)) {
        keep = m > canny_mag(dxy, H, W, y - 1, x) && m >= canny_mag(dxy, H, W, y + 1, x);
      } else {
        const int s = (dx ^ dy) < 0 ? -1 : 1;
        keep = m > canny_mag(dxy, H, W, y - 1, x - s) && m > canny_mag(dxy, H, W, y + 1, x + s);
      }
      if (keep) k = m > high ? 2 : 1;
    }
    cls[i] = k;
    label[i] = k ? static_cast<int>(i) : -1;
    flag[i] = 0;
  }
}

// Labels only ever decrease and label[i] <= i, so every chain ends at a root.  Reads bypass L1, which is not coherent
// with the atomics of other SMs.
__device__ __forceinline__ int canny_find(const int* label, int i) {
  int p = __ldcg(label + i);
  while (p != i) {
    i = p;
    p = __ldcg(label + i);
  }
  return i;
}

__device__ __forceinline__ void canny_unite(int* label, int a, int b) {
  while (true) {
    a = canny_find(label, a);
    b = canny_find(label, b);
    if (a == b) return;
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    // hang the larger root under the smaller one; if b stopped being a root meanwhile, retry from its new parent
    const int old = atomicMin(label + b, a);
    if (old == b) return;
    b = old;
  }
}

__global__ void canny_merge_kernel(const uint8_t* __restrict__ cls, int* label, int H, int W) {
  const long long n = static_cast<long long>(H) * W;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    if (!cls[i]) continue;
    const int y = static_cast<int>(i / W), x = static_cast<int>(i - static_cast<long long>(y) * W);
    if (x > 0 && cls[i - 1]) canny_unite(label, static_cast<int>(i), static_cast<int>(i - 1));
    if (y > 0) {
      const long long up = i - W;
      if (x > 0 && cls[up - 1]) canny_unite(label, static_cast<int>(i), static_cast<int>(up - 1));
      if (cls[up]) canny_unite(label, static_cast<int>(i), static_cast<int>(up));
      if (x + 1 < W && cls[up + 1]) canny_unite(label, static_cast<int>(i), static_cast<int>(up + 1));
    }
  }
}

// The forest is final here: writing a root into label[i] keeps every chain ending at the same root.
__global__ void canny_resolve_kernel(const uint8_t* __restrict__ cls, int* label, uint8_t* __restrict__ flag,
                                     long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint8_t k = cls[i];
    if (!k) continue;
    const int r = canny_find(label, static_cast<int>(i));
    label[i] = r;
    if (k == 2) flag[r] = 1;
  }
}

__global__ void canny_edges_kernel(const uint8_t* __restrict__ cls, const int* __restrict__ label,
                                   const uint8_t* __restrict__ flag, uint8_t* __restrict__ out, long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint8_t e = (cls[i] && flag[label[i]]) ? 255 : 0;
    out[3 * i] = e;
    out[3 * i + 1] = e;
    out[3 * i + 2] = e;
  }
}

}  // namespace dk

using namespace dk;

extern "C" int dk_canny(dk_ctx* ctx, const uint8_t* img, const uint8_t* lut, uint8_t* out, void* ws, int H, int W,
                        int src_channels, int low, int high, void* stream_) {
  DK_ENTRY(ctx);
  DK_REQUIRE(img != nullptr && lut != nullptr && out != nullptr && ws != nullptr,
             "dk_canny: img, lut, out and ws are required");
  DK_REQUIRE(dk_aligned16(ws), "dk_canny: ws must be 16-byte aligned");
  DK_REQUIRE(H > 0 && W > 0 && static_cast<long long>(H) * W < (1ll << 31),
             "dk_canny: H and W must be positive with H * W < 2^31, got %dx%d", H, W);
  DK_REQUIRE(src_channels >= 3, "dk_canny: image needs at least 3 channels (got %d)", src_channels);
  DK_REQUIRE(low >= 0 && low <= high, "dk_canny: thresholds must satisfy 0 <= low <= high, got %d / %d", low, high);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long n = static_cast<long long>(H) * W;
  // workspace (DK_CANNY_WS_BYTES_PER_PIXEL per pixel): labels, (dx, dy), classes, root flags
  int* label = static_cast<int*>(ws);
  short2* dxy = reinterpret_cast<short2*>(static_cast<char*>(ws) + 4 * n);
  uint8_t* cls = static_cast<uint8_t*>(ws) + 8 * n;
  uint8_t* flag = cls + n;
  const int grid = dk_grid_for(n, 256, ctx->sm_count);
  canny_grad_kernel<<<grid, 256, 0, stream>>>(img, lut, dxy, H, W, src_channels);
  DK_LAUNCH_CHECK(ctx);
  canny_nms_kernel<<<grid, 256, 0, stream>>>(dxy, cls, label, flag, H, W, low, high);
  DK_LAUNCH_CHECK(ctx);
  canny_merge_kernel<<<grid, 256, 0, stream>>>(cls, label, H, W);
  DK_LAUNCH_CHECK(ctx);
  canny_resolve_kernel<<<grid, 256, 0, stream>>>(cls, label, flag, n);
  DK_LAUNCH_CHECK(ctx);
  canny_edges_kernel<<<grid, 256, 0, stream>>>(cls, label, flag, out, n);
  DK_LAUNCH_CHECK(ctx);
  return 0;
}
