// Image preprocessing and reductions of the image-symmetry and prompt-consistency rewards
// (reference ddpo/training/callbacks.py:122-140, 166-344), on uint8 NHWC RGB batches.
//
//   resample_u8        Image.resize((w, h), BICUBIC) with reducing_gap=None, one axis per call (Pillow's
//                      ImagingResample: the width pass runs first and stores uint8, then the height pass).  The
//                      22-bit fixed-point coefficient table comes from the host (ddpo_b200/clip_vision.py,
//                      resample_table); the first pass reads the source through a transform: identity,
//                      ImageOps.mirror, rotate(90 / 180 / 270) (Pillow's transposes; 90 / 270 need a square image).
//   clip_normalize_u8  CLIPProcessor's rescale + normalise of a centre crop: (float32(x) / 255 - mean) / std with the
//                      division in fp32 and the normalisation in double, as clip_vision.preprocess computes it.
//   pair_stats_u8      per image against its mirror or 180-degree rotation: sum(((a - T a) mod 256)^2 mod 256) (numpy's
//                      uint8 wrap in the reference's (pils - mirrored) ** 2), sum a, sum a^2, sum a T(a).
//   feature_angles     mean over variants v >= 1 of degrees(arccos(clip(cos(f_0, f_v), 0, 1))).
//   scaled_cosine      exp(logit_scale) cos(img_i, txt_i), the diagonal of CLIP's logits_per_image.
//
// Integer sums are exact; the float reductions run in double over a fixed tree, so every result is independent of
// the batch and bit-reproducible.  No atomics.
#include <cmath>

#include "common.cuh"

namespace ddpo {
namespace {

constexpr int IR_THREADS = 256;
constexpr int IR_BITS = 22;   // Pillow's PRECISION_BITS = 32 - 8 - 2

// The source image seen through a transform: pixel (y, x) of the transformed view is src[off + y * sy + x * sx]
// (in pixels, within one image).  Pillow's rotate(90) equals np.rot90(a, 1): out[y, x] = a[x, W - 1 - y].
struct View {
  int64_t off, sy, sx;
  int th, tw;
};

View make_view(int h, int w, int transform) {
  switch (transform) {
    case DDPO_IMAGE_MIRROR: return {w - 1, w, -1, h, w};
    case DDPO_IMAGE_ROT90: return {w - 1, -1, w, w, h};
    case DDPO_IMAGE_ROT180: return {static_cast<int64_t>(h) * w - 1, -w, -1, h, w};
    case DDPO_IMAGE_ROT270: return {static_cast<int64_t>(h - 1) * w, 1, -w, w, h};
    default: return {0, w, 1, h, w};
  }
}

// One output pixel per thread.  axis 0: out [B, th, n_out, 3] resampled along the view's columns; axis 1:
// out [B, n_out, tw, 3] along its rows.  table: per output index xmin, n, then ksize coefficients.
__global__ void __launch_bounds__(IR_THREADS) resample_u8_kernel(const uint8_t* __restrict__ src, View v, int64_t img_px,
                                                                 int axis, int n_out, const int32_t* __restrict__ table,
                                                                 int ksize, int B, uint8_t* __restrict__ dst) {
  const int rows = axis == 0 ? v.th : n_out, cols = axis == 0 ? n_out : v.tw;
  const int64_t total = static_cast<int64_t>(B) * rows * cols;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * IR_THREADS + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * IR_THREADS) {
    const int x = static_cast<int>(i % cols);
    const int y = static_cast<int>((i / cols) % rows);
    const int b = static_cast<int>(i / (static_cast<int64_t>(cols) * rows));
    const int o = axis == 0 ? x : y;
    const int32_t* rec = table + static_cast<int64_t>(o) * (2 + ksize);
    const int xmin = rec[0], n = rec[1];
    const int64_t step = axis == 0 ? v.sx : v.sy;
    int64_t px = static_cast<int64_t>(b) * img_px + v.off + (axis == 0 ? y * v.sy + static_cast<int64_t>(xmin) * v.sx
                                                                      : static_cast<int64_t>(xmin) * v.sy + x * v.sx);
    int32_t a0 = 1 << (IR_BITS - 1), a1 = a0, a2 = a0;
    for (int j = 0; j < n; ++j, px += step) {
      const int32_t k = rec[2 + j];
      const uint8_t* p = src + px * 3;
      a0 += p[0] * k, a1 += p[1] * k, a2 += p[2] * k;
    }
    a0 >>= IR_BITS, a1 >>= IR_BITS, a2 >>= IR_BITS;
    uint8_t* q = dst + i * 3;
    q[0] = static_cast<uint8_t>(a0 < 0 ? 0 : (a0 > 255 ? 255 : a0));
    q[1] = static_cast<uint8_t>(a1 < 0 ? 0 : (a1 > 255 ? 255 : a1));
    q[2] = static_cast<uint8_t>(a2 < 0 ? 0 : (a2 > 255 ? 255 : a2));
  }
}

__constant__ double kClipMean[3] = {0.48145466, 0.4578275, 0.40821073};
__constant__ double kClipStd[3] = {0.26862954, 0.26130258, 0.27577711};

__global__ void __launch_bounds__(IR_THREADS) clip_normalize_u8_kernel(const uint8_t* __restrict__ src, int B, int h,
                                                                       int w, int top, int left, int size,
                                                                       float* __restrict__ out) {
  const int64_t total = static_cast<int64_t>(B) * size * size * 3;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * IR_THREADS + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * IR_THREADS) {
    const int c = static_cast<int>(i % 3);
    const int x = static_cast<int>((i / 3) % size);
    const int y = static_cast<int>((i / (3 * size)) % size);
    const int b = static_cast<int>(i / (3 * static_cast<int64_t>(size) * size));
    const uint8_t u = src[((static_cast<int64_t>(b) * h + top + y) * w + left + x) * 3 + c];
    const float q = __fdiv_rn(static_cast<float>(u), 255.0f);
    out[i] = __double2float_rn(__ddiv_rn(__dadd_rn(static_cast<double>(q), -kClipMean[c]), kClipStd[c]));
  }
}

// Fixed-order block tree over IR_THREADS values (one array per sum).
template <typename T, int K>
__device__ __forceinline__ void block_sum(T (&v)[K], T (*sh)[IR_THREADS]) {
#pragma unroll
  for (int k = 0; k < K; ++k) sh[k][threadIdx.x] = v[k];
  __syncthreads();
  for (int s = IR_THREADS / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
#pragma unroll
      for (int k = 0; k < K; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + s];
    }
    __syncthreads();
  }
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = sh[k][0];
}

// One CTA per image: out[b] = {sum wrapped square, sum a, sum a^2, sum a T(a)}.
__global__ void __launch_bounds__(IR_THREADS) pair_stats_u8_kernel(const uint8_t* __restrict__ src, View v,
                                                                   unsigned long long* __restrict__ out) {
  __shared__ unsigned long long sh[4][IR_THREADS];
  const int b = blockIdx.x;
  const int64_t px_img = static_cast<int64_t>(v.th) * v.tw;
  const uint8_t* img = src + static_cast<int64_t>(b) * px_img * 3;
  unsigned long long s[4] = {0, 0, 0, 0};
  for (int64_t e = threadIdx.x; e < px_img * 3; e += IR_THREADS) {
    const int c = static_cast<int>(e % 3);
    const int64_t p = e / 3;
    const int y = static_cast<int>(p / v.tw), x = static_cast<int>(p % v.tw);
    const uint32_t a = img[e], t = img[(v.off + y * v.sy + x * v.sx) * 3 + c];
    const uint32_t d = (a - t) & 255u;
    s[0] += (d * d) & 255u;
    s[1] += a;
    s[2] += a * a;
    s[3] += a * t;
  }
  block_sum(s, sh);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) out[static_cast<int64_t>(b) * 4 + k] = s[k];
  }
}

__device__ __forceinline__ double clipped_degrees(double dot, double na, double nb) {
  double c = dot / (sqrt(na) * sqrt(nb));
  c = c < 0.0 ? 0.0 : (c > 1.0 ? 1.0 : c);   // NaN stays NaN, as in np.clip
  return acos(c) * (180.0 / 3.14159265358979323846);
}

// One CTA per image i: rows v * n + i of feats are its variants.
__global__ void __launch_bounds__(IR_THREADS) feature_angles_kernel(const float* __restrict__ feats, int variants, int n,
                                                                    int dim, float* __restrict__ out) {
  __shared__ double sh[3][IR_THREADS];
  const int i = blockIdx.x;
  const float* f0 = feats + static_cast<int64_t>(i) * dim;
  double total = 0.0;
  for (int vv = 1; vv < variants; ++vv) {
    const float* fv = feats + (static_cast<int64_t>(vv) * n + i) * dim;
    double s[3] = {0.0, 0.0, 0.0};
    for (int c = threadIdx.x; c < dim; c += IR_THREADS) {
      const double a = f0[c], bb = fv[c];
      s[0] += a * bb, s[1] += a * a, s[2] += bb * bb;
    }
    block_sum(s, sh);
    total += clipped_degrees(s[0], s[1], s[2]);
    __syncthreads();
  }
  if (threadIdx.x == 0) out[i] = static_cast<float>(total / (variants - 1));
}

__global__ void __launch_bounds__(IR_THREADS) scaled_cosine_kernel(const float* __restrict__ img,
                                                                   const float* __restrict__ txt, int dim, double scale,
                                                                   float* __restrict__ out) {
  __shared__ double sh[3][IR_THREADS];
  const int i = blockIdx.x;
  const float* a = img + static_cast<int64_t>(i) * dim;
  const float* t = txt + static_cast<int64_t>(i) * dim;
  double s[3] = {0.0, 0.0, 0.0};
  for (int c = threadIdx.x; c < dim; c += IR_THREADS) {
    const double x = a[c], y = t[c];
    s[0] += x * y, s[1] += x * x, s[2] += y * y;
  }
  block_sum(s, sh);
  if (threadIdx.x == 0) out[i] = static_cast<float>(scale * (s[0] / (sqrt(s[1]) * sqrt(s[2]))));
}

int ir_grid(int64_t n) {
  const int64_t g = (n + IR_THREADS - 1) / IR_THREADS;
  return static_cast<int>(g > 132 * 32 ? 132 * 32 : (g < 1 ? 1 : g));
}

bool transform_ok(int h, int w, int transform) {
  if (transform < DDPO_IMAGE_IDENTITY || transform > DDPO_IMAGE_ROT270) return false;
  return h == w || (transform != DDPO_IMAGE_ROT90 && transform != DDPO_IMAGE_ROT270);
}

}  // namespace
}  // namespace ddpo

using namespace ddpo;

extern "C" int ddpo_resample_u8(const uint8_t* src, int batch, int h, int w, int transform, int axis, int n_out,
                                const int32_t* table_host, const int32_t* table_dev, int ksize, uint8_t* dst,
                                void* stream) {
  DDPO_REQUIRE(src && dst && table_host && table_dev && batch > 0 && h > 0 && w > 0 && n_out > 0 && ksize > 0 &&
                   (axis == 0 || axis == 1),
               "resample_u8: bad arguments (batch=%d h=%d w=%d n_out=%d ksize=%d axis=%d)", batch, h, w, n_out, ksize,
               axis);
  DDPO_REQUIRE(transform_ok(h, w, transform),
               "resample_u8: transform %d needs a square image (got %dx%d); non-square rotate is Pillow's affine path",
               transform, h, w);
  const View v = make_view(h, w, transform);
  const int n_in = axis == 0 ? v.tw : v.th;
  for (int o = 0; o < n_out; ++o) {
    const int32_t* rec = table_host + static_cast<int64_t>(o) * (2 + ksize);
    DDPO_REQUIRE(rec[0] >= 0 && rec[1] >= 1 && rec[1] <= ksize && rec[0] + rec[1] <= n_in,
                 "resample_u8: table entry %d (xmin=%d n=%d) outside the %d input samples", o, rec[0], rec[1], n_in);
  }
  resample_u8_kernel<<<ir_grid(static_cast<int64_t>(batch) * (axis == 0 ? v.th : n_out) * (axis == 0 ? n_out : v.tw)),
                       IR_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      src, v, static_cast<int64_t>(h) * w, axis, n_out, table_dev, ksize, batch, dst);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_clip_normalize_u8(const uint8_t* src, int batch, int h, int w, int top, int left, int size,
                                      float* out, void* stream) {
  DDPO_REQUIRE(src && out && batch > 0 && size > 0 && top >= 0 && left >= 0 && top + size <= h && left + size <= w,
               "clip_normalize_u8: bad arguments (%dx%d image, crop %d at (%d, %d))", h, w, size, top, left);
  clip_normalize_u8_kernel<<<ir_grid(static_cast<int64_t>(batch) * size * size * 3), IR_THREADS, 0,
                             static_cast<cudaStream_t>(stream)>>>(src, batch, h, w, top, left, size, out);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_pair_stats_u8(const uint8_t* src, int batch, int h, int w, int transform, uint64_t* out,
                                  void* stream) {
  DDPO_REQUIRE(src && out && batch > 0 && h > 0 && w > 0 &&
                   (transform == DDPO_IMAGE_MIRROR || transform == DDPO_IMAGE_ROT180),
               "pair_stats_u8: bad arguments (h=%d w=%d transform=%d; mirror or 180-degree rotation only)", h, w,
               transform);
  pair_stats_u8_kernel<<<batch, IR_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      src, make_view(h, w, transform), reinterpret_cast<unsigned long long*>(out));
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_feature_angles(const float* feats, int variants, int n, int dim, float* out, void* stream) {
  DDPO_REQUIRE(feats && out && variants >= 2 && n > 0 && dim > 0, "feature_angles: bad arguments (variants=%d n=%d dim=%d)",
               variants, n, dim);
  feature_angles_kernel<<<n, IR_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(feats, variants, n, dim, out);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_scaled_cosine(const float* img, const float* txt, int n, int dim, float logit_scale, float* out,
                                  void* stream) {
  DDPO_REQUIRE(img && txt && out && n > 0 && dim > 0 && std::isfinite(logit_scale),
               "scaled_cosine: bad arguments (n=%d dim=%d)", n, dim);
  // CLIP's logit_scale.exp() is taken in fp32
  scaled_cosine_kernel<<<n, IR_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      img, txt, dim, static_cast<double>(std::exp(logit_scale)), out);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}
