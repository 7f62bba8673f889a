// CLIP text-encoder pieces that are not GEMM / attention / (bf16-out) LayerNorm shaped (those reuse igemm.cu,
// attention.cu with the causal flag, norm.cu):
//   * token + position embedding lookup
//   * the MLP activation between fc1 and fc2 (gelu = exact erf form, quick_gelu = x * sigmoid(1.702 x))
//   * the final LayerNorm with fp32 output (the conditioning tensor the U-Net consumes is fp32)
//
// Reference semantics: the reference embeds prompts with 3P transformers==4.28.1 FlaxCLIPTextModel
// (pipeline/policy_gradient.py:185-187 on the host CPU; ddpo/training/diffusion.py:45-51,62-68 inside the RWR step):
// FlaxCLIPTextEmbeddings, FlaxCLIPMLP (ACT2FN[hidden_act]), FlaxCLIPTextTransformer.final_layer_norm.
#include "common.cuh"

namespace ddpo {

// out[m, :] = tok[ids[m], :] + pos[m % L, :]
__global__ void __launch_bounds__(256) embed_tokens_kernel(const int32_t* __restrict__ ids, const float* __restrict__ tok,
                                                           const float* __restrict__ pos, float* __restrict__ out, int M,
                                                           int L, int D4, int vocab) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= static_cast<int64_t>(M) * D4) return;
  const int m = static_cast<int>(i / D4), c = static_cast<int>(i % D4);
  int id = ids[m];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  const float4 a = reinterpret_cast<const float4*>(tok)[static_cast<size_t>(id) * D4 + c];
  const float4 b = reinterpret_cast<const float4*>(pos)[static_cast<size_t>(m % L) * D4 + c];
  reinterpret_cast<float4*>(out)[i] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}

__device__ __forceinline__ float act_f(float x, int act) {
  if (act == 1) return x / (1.0f + expf(-1.702f * x));            // quick_gelu
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));   // gelu (exact)
}

__global__ void __launch_bounds__(256) act_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                       int64_t n4, int act) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * 256) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    reinterpret_cast<uint2*>(y)[i] = make_uint2(pack_bf16(act_f(v.x, act), act_f(v.y, act)),
                                                pack_bf16(act_f(v.z, act), act_f(v.w, act)));
  }
}

// one warp per row; x fp32 [M, C] -> y fp32 [M, C]
__global__ void __launch_bounds__(256) layernorm_f32_kernel(const float* __restrict__ x, const float* __restrict__ scale,
                                                            const float* __restrict__ bias, float* __restrict__ y, int M,
                                                            int C, float eps) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* xr = x + static_cast<size_t>(row) * C;
  float s = 0.f, ss = 0.f;
  for (int c = lane * 4; c < C; c += 128) {
    const float4 v = *reinterpret_cast<const float4*>(xr + c);
    s += (v.x + v.y) + (v.z + v.w);
    ss += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
  }
  s = warp_sum(s), ss = warp_sum(ss);
  const float mean = s / C;
  const float rstd = rsqrtf(fmaxf(0.f, ss / C - mean * mean) + eps);
  float* yr = y + static_cast<size_t>(row) * C;
  for (int c = lane * 4; c < C; c += 128) {
    const float4 v = *reinterpret_cast<const float4*>(xr + c);
    const float4 sc = __ldg(reinterpret_cast<const float4*>(scale + c));
    const float4 bi = __ldg(reinterpret_cast<const float4*>(bias + c));
    *reinterpret_cast<float4*>(yr + c) = make_float4((v.x - mean) * rstd * sc.x + bi.x, (v.y - mean) * rstd * sc.y + bi.y,
                                                     (v.z - mean) * rstd * sc.z + bi.z, (v.w - mean) * rstd * sc.w + bi.w);
  }
}

}  // namespace ddpo

using namespace ddpo;

extern "C" int ddpo_embed_tokens(const int32_t* ids, const float* token_embedding, const float* position_embedding,
                                 float* out, int rows, int seq_len, int dim, int vocab, void* stream) {
  DDPO_REQUIRE(ids && token_embedding && position_embedding && out && rows > 0 && seq_len > 0 && dim % 4 == 0 && vocab > 0,
               "embed_tokens: bad arguments");
  const int64_t n = static_cast<int64_t>(rows) * (dim / 4);
  embed_tokens_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      ids, token_embedding, position_embedding, out, rows, seq_len, dim / 4, vocab);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_act_bf16(const float* x, void* y_bf16, int64_t n, int act, void* stream) {
  DDPO_REQUIRE(x && y_bf16 && n > 0 && n % 4 == 0 && (act == 0 || act == 1), "act_bf16: bad arguments");
  int64_t blocks = (n / 4 + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  act_bf16_kernel<<<static_cast<int>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, static_cast<__nv_bfloat16*>(y_bf16), n / 4, act);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_layernorm_f32(const float* x, const float* scale, const float* bias, float* y, int m, int c, float eps,
                                  void* stream) {
  DDPO_REQUIRE(x && scale && bias && y && m > 0 && c % 4 == 0, "layernorm_f32: bad arguments (m=%d c=%d)", m, c);
  layernorm_f32_kernel<<<(m + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, scale, bias, y, m, c, eps);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}
