// Image preparation of the eval loader (datasets/general_eval.py:112-131, 210-211) on the device: the edge pad and
// cv2.resize of each decoded uint8 image, once per scene, and the ToTensor + Normalize of each view set, gathered from the
// resident uint8 scene by view index.
//
// Both are bit-exact restatements (oracle/image_prep.py spells out the same rules in numpy):
//   - resize: cv2's INTER_LINEAR for uint8.  The coefficients come from the double scale rounded to float, so the double
//     product and sum and the float products are written as __dmul_rn / __dadd_rn / __fmul_rn: nvcc would otherwise
//     contract (dx + 0.5) * scale - 0.5 into an FMA, which moves fx.  The weights are 11-bit fixed point and the vertical
//     pass is cv2's SIMD one (VResizeLinearVec_32s8u): each horizontal sum loses 4 bits before a 16-bit high multiply.
//   - normalize: (u8 / 255 - mean) / std, and the colour test.py saves for fusion, trunc(clip((x std + mean) 255)) / 255,
//     each step one rounded fp32 operation as torch and numpy perform them.
// One thread per output pixel, 3 channels; both kernels are memory-bound.
#include "common.cuh"

namespace mvsf {

constexpr int IMG_BLOCK = 256;
constexpr int IMG_MAX_VIEWS = 64;
constexpr int RESIZE_COEF = 2048;   // cv2's INTER_RESIZE_COEF_SCALE

struct ImgViews { int idx[IMG_MAX_VIEWS]; };

// cv2::resize's source coordinate of output index d: floor and fraction of (d + 0.5) * scale - 0.5, rounded to float
__device__ __forceinline__ void resize_coord(int d, double scale, int& s, float& f) {
  const float x = __double2float_rn(__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5));
  const float fl = floorf(x);
  s = (int)fl;
  f = __fsub_rn(x, fl);
}

// saturate_cast<short>(w * 2048) of cv2: round half to even
__device__ __forceinline__ int resize_weight(float w) { return __float2int_rn(__fmul_rn(w, (float)RESIZE_COEF)); }

__global__ void __launch_bounds__(IMG_BLOCK) image_resize_kernel(const uint8_t* __restrict__ src, int h, int w, int pad,
                                                                 uint8_t* __restrict__ dst, int H, int W, double scale_y,
                                                                 double scale_x, long long total) {
  const long long i = (long long)blockIdx.x * IMG_BLOCK + threadIdx.x;
  if (i >= total) return;
  const int dx = (int)(i % W);
  const long long r = i / W;
  const int dy = (int)(r % H);
  const long long n = r / H;

  int sx;
  float fx;
  resize_coord(dx, scale_x, sx, fx);
  if (sx < 0) sx = 0, fx = 0.f;
  if (sx >= w - 1) sx = w - 1, fx = 0.f;
  const int x1 = min(sx + 1, w - 1);
  const int a0 = resize_weight(__fsub_rn(1.f, fx)), a1 = resize_weight(fx);

  int sy;
  float fy;
  resize_coord(dy, scale_y, sy, fy);   // rows keep their fraction; both rows are clamped to the padded image
  const int hp = h + 2 * pad;
  const int b0 = resize_weight(__fsub_rn(1.f, fy)), b1 = resize_weight(fy);
  // padded row -> source row: the edge pad repeats the first and last rows
  const int y0 = min(max(min(max(sy, 0), hp - 1) - pad, 0), h - 1);
  const int y1 = min(max(min(max(sy + 1, 0), hp - 1) - pad, 0), h - 1);

  const uint8_t* img = src + (size_t)n * h * w * 3;
  const uint8_t* p00 = img + ((size_t)y0 * w + sx) * 3;
  const uint8_t* p01 = img + ((size_t)y0 * w + x1) * 3;
  const uint8_t* p10 = img + ((size_t)y1 * w + sx) * 3;
  const uint8_t* p11 = img + ((size_t)y1 * w + x1) * 3;
  uint8_t* o = dst + (size_t)i * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int s0 = (a0 * (int)__ldg(p00 + c) + a1 * (int)__ldg(p01 + c)) >> 4;
    const int s1 = (a0 * (int)__ldg(p10 + c) + a1 * (int)__ldg(p11 + c)) >> 4;
    const int v = (((s0 * b0) >> 16) + ((s1 * b1) >> 16) + 2) >> 2;
    o[c] = (uint8_t)min(max(v, 0), 255);
  }
}

__device__ __constant__ float IMG_MEAN[3] = {0.485f, 0.456f, 0.406f};   // general_eval.py:31
__device__ __constant__ float IMG_STD[3] = {0.229f, 0.224f, 0.225f};

__global__ void __launch_bounds__(IMG_BLOCK) image_normalize_kernel(const uint8_t* __restrict__ scene, ImgViews views, int V,
                                                                    int H, int W, float* __restrict__ norm,
                                                                    float* __restrict__ colour) {
  const long long HW = (long long)H * W;
  const long long i = (long long)blockIdx.x * IMG_BLOCK + threadIdx.x;
  if (i >= (long long)V * HW) return;
  const int v = (int)(i / HW);
  const long long p = i - (long long)v * HW;
  const uint8_t* px = scene + ((size_t)views.idx[v] * HW + p) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float x = __fdiv_rn(__fsub_rn(__fdiv_rn((float)__ldg(px + c), 255.f), IMG_MEAN[c]), IMG_STD[c]);
    const size_t o = ((size_t)v * 3 + c) * HW + p;
    if (norm) norm[o] = x;
    if (colour) {
      const float u = __fmul_rn(__fadd_rn(__fmul_rn(x, IMG_STD[c]), IMG_MEAN[c]), 255.f);
      colour[o] = __fdiv_rn(truncf(fminf(fmaxf(u, 0.f), 255.f)), 255.f);
    }
  }
}

}  // namespace mvsf

extern "C" {

int mvsf_image_resize_u8(const unsigned char* src, int N, int h, int w, int pad_rows, unsigned char* dst, int H, int W,
                         mvsf_stream_t stream) {
  MVSF_REQUIRE(src && dst, "image_resize_u8: null pointer");
  MVSF_REQUIRE(N > 0 && h > 0 && w > 0 && H > 0 && W > 0, "image_resize_u8: N = %d, %d x %d -> %d x %d: every size must be >= 1",
               N, h, w, H, W);
  MVSF_REQUIRE(pad_rows >= 0 && (long long)h + 2ll * pad_rows < (1ll << 30), "image_resize_u8: pad_rows = %d", pad_rows);
  MVSF_REQUIRE((long long)h * w < (1ll << 31) && (long long)H * W < (1ll << 31),
               "image_resize_u8: %d x %d -> %d x %d: an image must have fewer than 2^31 pixels", h, w, H, W);
  const long long total = (long long)N * H * W;
  MVSF_REQUIRE(total / mvsf::IMG_BLOCK < (1ll << 31) - 1, "image_resize_u8: %lld output pixels", total);
  // cv2: inv_scale = (double)dsize / ssize, scale = 1. / inv_scale
  const double scale_x = 1.0 / ((double)W / w), scale_y = 1.0 / ((double)H / (h + 2 * pad_rows));
  mvsf::image_resize_kernel<<<(unsigned)((total + mvsf::IMG_BLOCK - 1) / mvsf::IMG_BLOCK), mvsf::IMG_BLOCK, 0,
                              (cudaStream_t)stream>>>(src, h, w, pad_rows, dst, H, W, scale_y, scale_x, total);
  MVSF_LAUNCH_CHECK("image_resize_u8");
  return MVSF_OK;
}

int mvsf_image_normalize(const unsigned char* scene, int N, const int* views, int V, int H, int W, float* norm,
                         float* colour, mvsf_stream_t stream) {
  MVSF_REQUIRE(scene && views, "image_normalize: null pointer");
  MVSF_REQUIRE(norm || colour, "image_normalize: neither output requested");
  MVSF_REQUIRE(V >= 1 && V <= mvsf::IMG_MAX_VIEWS, "image_normalize: %d views outside [1, %d]", V, mvsf::IMG_MAX_VIEWS);
  MVSF_REQUIRE(H > 0 && W > 0 && (long long)H * W < (1ll << 31), "image_normalize: H x W = %d x %d outside [1, 2^31)", H, W);
  mvsf::ImgViews s;
  for (int i = 0; i < mvsf::IMG_MAX_VIEWS; ++i) s.idx[i] = 0;
  for (int i = 0; i < V; ++i) {
    MVSF_REQUIRE(N > 0 && views[i] >= 0 && views[i] < N, "image_normalize: view %d outside the scene's %d images", views[i], N);
    s.idx[i] = views[i];
  }
  const long long total = (long long)V * H * W;
  mvsf::image_normalize_kernel<<<(unsigned)((total + mvsf::IMG_BLOCK - 1) / mvsf::IMG_BLOCK), mvsf::IMG_BLOCK, 0,
                                 (cudaStream_t)stream>>>(scene, s, V, H, W, norm, colour);
  MVSF_LAUNCH_CHECK("image_normalize");
  return MVSF_OK;
}
}
