// Optimizer step on the flat fp32 parameter / gradient buffers (HBM-bound, one pass).
//
// Restates optax.chain(clip_by_global_norm(max_norm), adamw(lr, b1, b2, eps, wd, mu_dtype=bf16))
// (3P optax==0.1.5; reference pipeline/policy_gradient.py:130-150) fused with
// AccumulatingTrainState.apply_gradients(do_update=True) (ddpo/training/policy_gradient.py:32-43):
//   g~ = grad_acc * grad_scale            (grad_scale = 1 / (n_acc * world_size))
//   g^ = g~ * min(1, max_norm / ||g~||)   (optax: where(norm < max, g, g / norm * max))
//   mu = b1 mu + (1-b1) g^ ; nu = b2 nu + (1-b2) g^2 ; u = mu_hat / (sqrt(nu_hat) + eps) + wd p
//   p -= lr u ; mu stored as bf16 ; grad_acc zeroed.
// The global norm is a two-stage fixed-order reduction (deterministic).
#include "common.cuh"

namespace ddpo {

constexpr int NORM_BLOCKS = 1056;  // 132 SMs (H100 SXM) x 8

__global__ void __launch_bounds__(256) sumsq_partial_kernel(const float* __restrict__ g, int64_t n4, double* __restrict__ part) {
  float acc = 0.f;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(g)[i];
    acc += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
  }
  __shared__ float sm[8];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < 8; ++i) s += sm[i];
    part[blockIdx.x] = s;
  }
}
__global__ void sumsq_final_kernel(const double* __restrict__ part, int nparts, float* __restrict__ out) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < nparts; ++i) s += part[i];
    out[0] = static_cast<float>(s);
  }
}

struct AdamArgs {
  float* p;
  float* g;
  __nv_bfloat16* mu;
  float* nu;
  int64_t n4;
  const float* sumsq;  // of the UNSCALED accumulated gradient
  float grad_scale, max_norm, lr, b1, b2, eps, wd, bc1, bc2;  // bc = 1 - b^t
  float* norm_out;
};

__global__ void __launch_bounds__(256) clip_adamw_kernel(const AdamArgs a) {
  const float norm = a.grad_scale * sqrtf(a.sumsq[0]);
  // optax.clip_by_global_norm: trigger = norm < max ; g = trigger ? g : (g / norm) * max
  const bool no_clip = norm < a.max_norm;
  if (a.norm_out != nullptr && blockIdx.x == 0 && threadIdx.x == 0) a.norm_out[0] = norm;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < a.n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float4 g4 = reinterpret_cast<float4*>(a.g)[i];
    float4 p4 = reinterpret_cast<float4*>(a.p)[i];
    float4 nu4 = reinterpret_cast<float4*>(a.nu)[i];
    uint2 mu2 = reinterpret_cast<uint2*>(a.mu)[i];
    float g[4] = {g4.x, g4.y, g4.z, g4.w}, p[4] = {p4.x, p4.y, p4.z, p4.w}, nu[4] = {nu4.x, nu4.y, nu4.z, nu4.w};
    float mu[4] = {bf16_lo(mu2.x), bf16_hi(mu2.x), bf16_lo(mu2.y), bf16_hi(mu2.y)};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float gj = g[j] * a.grad_scale;
      if (!no_clip) gj = (gj / norm) * a.max_norm;
      mu[j] = (1.0f - a.b1) * gj + a.b1 * mu[j];
      nu[j] = (1.0f - a.b2) * (gj * gj) + a.b2 * nu[j];
      const float u = (mu[j] / a.bc1) / (sqrtf(nu[j] / a.bc2) + a.eps) + a.wd * p[j];
      p[j] = p[j] + (-a.lr) * u;
    }
    reinterpret_cast<float4*>(a.p)[i] = make_float4(p[0], p[1], p[2], p[3]);
    reinterpret_cast<float4*>(a.nu)[i] = make_float4(nu[0], nu[1], nu[2], nu[3]);
    reinterpret_cast<uint2*>(a.mu)[i] = make_uint2(pack_bf16(mu[0], mu[1]), pack_bf16(mu[2], mu[3]));
    reinterpret_cast<float4*>(a.g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

}  // namespace ddpo

using namespace ddpo;

extern "C" int64_t ddpo_optim_workspace_bytes(void) { return NORM_BLOCKS * sizeof(double) + 16; }

// sumsq_out[0] = sum(g^2) (device scalar), deterministic
extern "C" int ddpo_grad_sumsq(const float* g, int64_t n, void* workspace, float* sumsq_out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DDPO_REQUIRE(g && workspace && sumsq_out && n % 4 == 0, "grad_sumsq: bad arguments (n must be a multiple of 4)");
  sumsq_partial_kernel<<<NORM_BLOCKS, 256, 0, stream>>>(g, n / 4, static_cast<double*>(workspace));
  DDPO_LAUNCH_OK();
  sumsq_final_kernel<<<1, 32, 0, stream>>>(static_cast<const double*>(workspace), NORM_BLOCKS, sumsq_out);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_clip_adamw(float* params, float* grad_acc, void* mu_bf16, float* nu, int64_t n,
                               const float* sumsq_dev, float grad_scale, float max_norm, float lr, float b1, float b2,
                               float eps, float weight_decay, int step, float* norm_out, void* stream) {
  DDPO_REQUIRE(params && grad_acc && mu_bf16 && nu && sumsq_dev && n % 4 == 0 && step >= 1, "clip_adamw: bad arguments");
  AdamArgs a;
  a.p = params, a.g = grad_acc, a.mu = static_cast<__nv_bfloat16*>(mu_bf16), a.nu = nu, a.n4 = n / 4;
  a.sumsq = sumsq_dev, a.grad_scale = grad_scale, a.max_norm = max_norm, a.lr = lr, a.b1 = b1, a.b2 = b2;
  a.eps = eps, a.wd = weight_decay;
  a.bc1 = static_cast<float>(1.0 - pow(static_cast<double>(b1), step));
  a.bc2 = static_cast<float>(1.0 - pow(static_cast<double>(b2), step));
  a.norm_out = norm_out;
  clip_adamw_kernel<<<NORM_BLOCKS, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}
