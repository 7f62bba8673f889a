// CLIP image-tower pieces that are not GEMM / attention / LayerNorm shaped (those reuse igemm.cu, attention.cu, norm.cu,
// text.cu): non-overlapping patch extraction (the stride-14 patch convolution becomes one GEMM over flattened patches),
// [CLS | patches] + position embedding, and the L2 normalisation of the image features.
//
// Reference semantics: the aesthetic reward (ddpo/training/callbacks.py:60-95): 3P transformers==4.28.1
// FlaxCLIPModel.get_image_features (FlaxCLIPVisionEmbeddings: Conv(kernel = stride = patch, no bias), class embedding,
// position embedding) followed by x / ||x|| and ddpo/models/laion.py:7-18 AestheticClassifier.
#include "common.cuh"

namespace ddpo {

// img fp32 NHWC [B, S, S, 3] -> out bf16 [B * P * P, ldk]; column k = (ky * patch + kx) * 3 + c, zero padded to ldk
__global__ void __launch_bounds__(256) patchify_bf16_kernel(const float* __restrict__ img, __nv_bfloat16* __restrict__ out,
                                                            int B, int S, int patch, int ldk) {
  const int P = S / patch, K = patch * patch * 3;
  const int64_t total = static_cast<int64_t>(B) * P * P * ldk;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * 256) {
    const int k = static_cast<int>(i % ldk);
    const int64_t row = i / ldk;
    float v = 0.f;
    if (k < K) {
      const int c = k % 3, kx = (k / 3) % patch, ky = k / (3 * patch);
      const int px = static_cast<int>(row % P), py = static_cast<int>((row / P) % P), b = static_cast<int>(row / (P * P));
      v = img[((static_cast<size_t>(b) * S + py * patch + ky) * S + px * patch + kx) * 3 + c];
    }
    out[i] = __float2bfloat16_rn(v);
  }
}

// out[b, 0, :] = cls + pos[0]; out[b, 1 + p, :] = patches[b, p, :] + pos[1 + p]
__global__ void __launch_bounds__(256) vit_tokens_kernel(const float* __restrict__ patches, const float* __restrict__ cls,
                                                         const float* __restrict__ pos, float* __restrict__ out, int B,
                                                         int N, int D4) {
  const int64_t total = static_cast<int64_t>(B) * (N + 1) * D4;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * 256) {
    const int c = static_cast<int>(i % D4);
    const int t = static_cast<int>((i / D4) % (N + 1));
    const int b = static_cast<int>(i / (static_cast<int64_t>(D4) * (N + 1)));
    const float4 a = t == 0 ? reinterpret_cast<const float4*>(cls)[c]
                            : reinterpret_cast<const float4*>(patches)[(static_cast<size_t>(b) * N + t - 1) * D4 + c];
    const float4 p = reinterpret_cast<const float4*>(pos)[static_cast<size_t>(t) * D4 + c];
    reinterpret_cast<float4*>(out)[i] = make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w);
  }
}

// y[r, :] = x[r, :] / ||x[r, :]||_2 ; one warp per row
__global__ void __launch_bounds__(256) l2norm_rows_kernel(const float* __restrict__ x, float* __restrict__ y, int M, int C) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* xr = x + static_cast<size_t>(row) * C;
  float ss = 0.f;
  for (int c = lane; c < C; c += 32) ss += xr[c] * xr[c];
  ss = warp_sum(ss);
  const float inv = 1.0f / sqrtf(ss);
  float* yr = y + static_cast<size_t>(row) * C;
  for (int c = lane; c < C; c += 32) yr[c] = xr[c] * inv;
}

}  // namespace ddpo

using namespace ddpo;

static inline int vgrid(int64_t n) {
  int64_t g = (n + 255) / 256;
  return static_cast<int>(g > 132 * 32 ? 132 * 32 : (g < 1 ? 1 : g));
}

extern "C" int ddpo_patchify_bf16(const float* img_nhwc, void* out_bf16, int batch, int size, int patch, int ldk,
                                  void* stream) {
  DDPO_REQUIRE(img_nhwc && out_bf16 && batch > 0 && patch > 0 && size % patch == 0 && ldk >= patch * patch * 3,
               "patchify_bf16: bad arguments (size=%d patch=%d ldk=%d)", size, patch, ldk);
  const int P = size / patch;
  patchify_bf16_kernel<<<vgrid(static_cast<int64_t>(batch) * P * P * ldk), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      img_nhwc, static_cast<__nv_bfloat16*>(out_bf16), batch, size, patch, ldk);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_vit_tokens(const float* patches, const float* class_embedding, const float* position_embedding,
                               float* out, int batch, int n_patches, int dim, void* stream) {
  DDPO_REQUIRE(patches && class_embedding && position_embedding && out && batch > 0 && n_patches > 0 && dim % 4 == 0,
               "vit_tokens: bad arguments");
  vit_tokens_kernel<<<vgrid(static_cast<int64_t>(batch) * (n_patches + 1) * (dim / 4)), 256, 0,
                      static_cast<cudaStream_t>(stream)>>>(patches, class_embedding, position_embedding, out, batch,
                                                           n_patches, dim / 4);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_l2norm_rows(const float* x, float* y, int m, int c, void* stream) {
  DDPO_REQUIRE(x && y && m > 0 && c > 0, "l2norm_rows: bad arguments");
  l2norm_rows_kernel<<<(m + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, m, c);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}
