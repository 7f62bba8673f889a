// JAX-compatible threefry2x32 noise, the fused CFG + DDIM step + Gaussian log-prob kernels
// (sample / score / backward) and the PPO clipped-surrogate kernel.
//
// Reference semantics:
//   ddpo/diffusers_patch/scheduling_ddim_flax.py:213-227 (_get_variance), :279-359 (step)
//   ddpo/diffusers_patch/pipeline_flax_stable_diffusion.py:226-235 (CFG, split, step)
//   ddpo/training/policy_gradient.py:103-134 (CFG, score-mode step, PPO loss/info)
//   3P jax==0.4.8 jax/_src/prng.py (threefry_2x32, random_bits) and random.py (normal)
//
// All of these are HBM/latency-bound: one pass over eps_u, eps_c, x (and x_prev), 128-bit
// loads, noise generated in registers, warp-shuffle + fixed-order partial reductions
// (no float atomics -> bit-reproducible log-probs).
#include <string.h>

#include "common.cuh"
#include "prng.cuh"

namespace ddpo {

__global__ void threefry_normal_kernel(const uint32_t* __restrict__ key, float* __restrict__ out, uint32_t n) {
  const uint32_t k0 = key[0], k1 = key[1];
  const uint32_t half = (n + 1) / 2;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < half; i += gridDim.x * blockDim.x) {
    uint32_t hi = i + half;
    u32x2 r = threefry2x32(k0, k1, i, hi < n ? hi : 0u);
    out[i] = bits_to_normal(r.a);
    if (hi < n) out[hi] = bits_to_normal(r.b);
  }
}

// ---------------------------------------------------------------- DDIM step ----
struct DdimCoef {
  float sqrt_at, sqrt_bt, sqrt_aprev, dir, sigma, sd;
};

// prev_sample_mean of scheduling_ddim_flax.py:303-338 for the three prediction types.  `m` is the (guidance-combined)
// model output.  NB the reference's `sample` branch leaves model_output untouched, so the "direction" term is
// dir * m there too (:307-308, :331-333) -- reproduced as written.
template <int PRED>
__device__ __forceinline__ float ddim_mean(const DdimCoef& k, float inv_sqrt_at, float x, float m) {
  if (PRED == DDPO_PRED_EPSILON) {
    const float x0 = (x - k.sqrt_bt * m) * inv_sqrt_at;
    return k.sqrt_aprev * x0 + k.dir * m;
  } else if (PRED == DDPO_PRED_SAMPLE) {
    return k.sqrt_aprev * m + k.dir * m;
  } else {
    const float x0 = k.sqrt_at * x - k.sqrt_bt * m;
    const float e = k.sqrt_at * m + k.sqrt_bt * x;
    return k.sqrt_aprev * x0 + k.dir * e;
  }
}

// d mean / d m
template <int PRED>
__device__ __forceinline__ float ddim_dmean(const DdimCoef& k, float inv_sqrt_at) {
  if (PRED == DDPO_PRED_EPSILON) return k.dir - k.sqrt_aprev * k.sqrt_bt * inv_sqrt_at;
  if (PRED == DDPO_PRED_SAMPLE) return k.sqrt_aprev + k.dir;
  return k.dir * k.sqrt_at - k.sqrt_aprev * k.sqrt_bt;
}

__device__ __forceinline__ DdimCoef ddim_coef(const ddpo_ddim_common& c, int b) {
  const int t = c.timesteps[b * c.timestep_stride];
  const int pt = t - c.step_ratio;
  const float a_t = c.alphas_cumprod[t];
  const float a_prev = pt >= 0 ? c.alphas_cumprod[pt] : c.final_alpha_cumprod;
  const float b_t = 1.0f - a_t;
  const float b_prev = 1.0f - a_prev;
  const float var = __fmul_rn(__fdiv_rn(b_prev, b_t), 1.0f - __fdiv_rn(a_t, a_prev));
  DdimCoef k;
  k.sigma = __fmul_rn(c.eta, sqrtf(var));
  k.sqrt_at = sqrtf(a_t);
  k.sqrt_bt = sqrtf(b_t);
  k.sqrt_aprev = sqrtf(a_prev);
  k.dir = sqrtf(1.0f - a_prev - __fmul_rn(k.sigma, k.sigma));
  k.sd = fmaxf(k.sigma, 1e-6f);
  return k;
}

constexpr int DDIM_THREADS = 256;

// MODE 0: sample (draw noise, write prev_sample, log_prob); MODE 1: score (read prev_sample, log_prob)
template <int MODE, int PRED>
__global__ void __launch_bounds__(DDIM_THREADS) ddim_step_kernel(const ddpo_ddim_common c, const uint32_t* __restrict__ key,
                                                                 float* __restrict__ prev_sample,
                                                                 float* __restrict__ log_prob) {
  const int b = blockIdx.y;
  const int chunk = blockIdx.x;
  const DdimCoef k = ddim_coef(c, b);
  const int n = c.n;
  const int per_chunk = ((n / 4 + DDPO_DDIM_CHUNKS - 1) / DDPO_DDIM_CHUNKS) * 4;
  const int begin = chunk * per_chunk;
  const int end = min(n, begin + per_chunk);
  const size_t base = static_cast<size_t>(b) * n;
  uint32_t k0 = 0, k1 = 0, ntot = 0, half = 0;
  if (MODE == 0) {
    k0 = key[0], k1 = key[1];
    ntot = static_cast<uint32_t>(c.batch) * n;
    half = (ntot + 1) / 2;
  }
  const float g = c.guidance_scale;
  const float inv_sqrt_at = 1.0f / k.sqrt_at;
  float acc = 0.0f;
  for (int i = begin + threadIdx.x * 4; i < end; i += DDIM_THREADS * 4) {
    const float4 eu = *reinterpret_cast<const float4*>(c.eps_uncond + base + i);
    const float4 ec = *reinterpret_cast<const float4*>(c.eps_cond + base + i);
    const float4 x = *reinterpret_cast<const float4*>(c.sample + base + i);
    const float e_u[4] = {eu.x, eu.y, eu.z, eu.w}, e_c[4] = {ec.x, ec.y, ec.z, ec.w}, xs[4] = {x.x, x.y, x.z, x.w};
    float pv[4];
    if (MODE == 1) {
      const float4 p4 = *reinterpret_cast<const float4*>(prev_sample + base + i);
      pv[0] = p4.x, pv[1] = p4.y, pv[2] = p4.z, pv[3] = p4.w;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float eps = e_u[j] + g * (e_c[j] - e_u[j]);
      const float mean = ddim_mean<PRED>(k, inv_sqrt_at, xs[j], eps);
      if (MODE == 0) {
        const uint32_t gi = static_cast<uint32_t>(base) + i + j;
        const float z = bits_to_normal(random_bits_at(k0, k1, gi, half, ntot));
        pv[j] = mean + k.sigma * z;
      }
      const float d = pv[j] - mean;
      acc += d * d;
    }
    if (MODE == 0) *reinterpret_cast<float4*>(prev_sample + base + i) = make_float4(pv[0], pv[1], pv[2], pv[3]);
  }
  __shared__ float warp_part[DDIM_THREADS / 32];
  __shared__ bool is_last;
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = acc;
  __syncthreads();
  float* partials = c.workspace;
  unsigned int* counters = reinterpret_cast<unsigned int*>(c.workspace + c.batch * DDPO_DDIM_CHUNKS);
  if (threadIdx.x == 0) {
    float s = 0.0f;
#pragma unroll
    for (int w = 0; w < DDIM_THREADS / 32; ++w) s += warp_part[w];
    partials[b * DDPO_DDIM_CHUNKS + chunk] = s;
    __threadfence();
    const unsigned int ticket = atomicAdd(&counters[b], 1u);
    is_last = (ticket == DDPO_DDIM_CHUNKS - 1);
    if (is_last) {
      __threadfence();
      float tot = 0.0f;
      for (int q = 0; q < DDPO_DDIM_CHUNKS; ++q) tot += *(volatile float*)&partials[b * DDPO_DDIM_CHUNKS + q];
      // mean over C*H*W of  -(d^2)/(2 sd^2) - log(sd) - log(sqrt(2 pi))
      log_prob[b] = -tot / (2.0f * k.sd * k.sd * static_cast<float>(n)) - logf(k.sd) - 0.91893853320467274178f;
      counters[b] = 0;
    }
  }
}

template <int PRED>
__global__ void __launch_bounds__(DDIM_THREADS) ddim_logprob_bwd_kernel(const ddpo_ddim_common c,
                                                                        const float* __restrict__ prev_sample,
                                                                        const float* __restrict__ dlogp,
                                                                        float* __restrict__ d_eu, float* __restrict__ d_ec) {
  const int b = blockIdx.y;
  const DdimCoef k = ddim_coef(c, b);
  const int n = c.n;
  const size_t base = static_cast<size_t>(b) * n;
  const float g = c.guidance_scale;
  const float inv_sqrt_at = 1.0f / k.sqrt_at;
  // d mean / d eps
  const float c_eps = ddim_dmean<PRED>(k, inv_sqrt_at);
  const float scale = dlogp[b] * c_eps / (k.sd * k.sd * static_cast<float>(n));
  for (int i = (blockIdx.x * DDIM_THREADS + threadIdx.x) * 4; i < n; i += gridDim.x * DDIM_THREADS * 4) {
    const float4 eu = *reinterpret_cast<const float4*>(c.eps_uncond + base + i);
    const float4 ec = *reinterpret_cast<const float4*>(c.eps_cond + base + i);
    const float4 x = *reinterpret_cast<const float4*>(c.sample + base + i);
    const float4 p4 = *reinterpret_cast<const float4*>(prev_sample + base + i);
    const float e_u[4] = {eu.x, eu.y, eu.z, eu.w}, e_c[4] = {ec.x, ec.y, ec.z, ec.w}, xs[4] = {x.x, x.y, x.z, x.w},
                pv[4] = {p4.x, p4.y, p4.z, p4.w};
    float du[4], dc[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float eps = e_u[j] + g * (e_c[j] - e_u[j]);
      const float mean = ddim_mean<PRED>(k, inv_sqrt_at, xs[j], eps);
      const float de = (pv[j] - mean) * scale;
      dc[j] = g * de;
      du[j] = (1.0f - g) * de;
    }
    *reinterpret_cast<float4*>(d_ec + base + i) = make_float4(dc[0], dc[1], dc[2], dc[3]);
    if (d_eu != nullptr) *reinterpret_cast<float4*>(d_eu + base + i) = make_float4(du[0], du[1], du[2], du[3]);
  }
}

// ---------------------------------------------------------------------- PPO ----
__global__ void ppo_loss_kernel(const float* __restrict__ lp, const float* __restrict__ old_lp,
                                const float* __restrict__ adv, int n, int grad_div, float clip,
                                float* __restrict__ info, float* __restrict__ dlogp) {
  __shared__ float s_loss[32], s_kl[32], s_cf[32];
  float loss = 0.f, kl = 0.f, cf = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float a = fminf(fmaxf(adv[i], -10.0f), 10.0f);
    const float d = lp[i] - old_lp[i];
    const float ratio = expf(d);
    const float unclipped = -a * ratio;
    const float clipped = -a * fminf(fmaxf(ratio, 1.0f - clip), 1.0f + clip);
    loss += fmaxf(unclipped, clipped);
    kl += d * d;
    cf += (fabsf(ratio - 1.0f) > clip) ? 1.0f : 0.0f;
    if (dlogp != nullptr) dlogp[i] = (unclipped >= clipped) ? unclipped / static_cast<float>(grad_div) : 0.0f;
  }
  loss = warp_sum(loss), kl = warp_sum(kl), cf = warp_sum(cf);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) s_loss[w] = loss, s_kl[w] = kl, s_cf[w] = cf;
  __syncthreads();
  if (threadIdx.x == 0) {
    float L = 0.f, K = 0.f, C = 0.f;
    for (int i = 0; i < (blockDim.x >> 5); ++i) L += s_loss[i], K += s_kl[i], C += s_cf[i];
    info[0] = 0.5f * K / n;  // approx_kl
    info[1] = C / n;         // clipfrac
    info[2] = L / n;         // loss
  }
}

}  // namespace ddpo

using namespace ddpo;

extern "C" int ddpo_prng_key_host(uint64_t seed, uint32_t out[2]) {
  out[0] = static_cast<uint32_t>(seed >> 32);
  out[1] = static_cast<uint32_t>(seed & 0xFFFFFFFFu);
  return DDPO_OK;
}

extern "C" int ddpo_threefry_split_host(const uint32_t key[2], int num, uint32_t* out) {
  DDPO_REQUIRE(num > 0, "ddpo_threefry_split_host: num must be positive");
  // counts = iota(2*num) split in halves: word0 gets [0,num), word1 gets [num,2num); output = cat(y0, y1)
  for (int i = 0; i < num; ++i) {
    u32x2 r = threefry2x32(key[0], key[1], static_cast<uint32_t>(i), static_cast<uint32_t>(i + num));
    out[i] = r.a;
    out[num + i] = r.b;
  }
  return DDPO_OK;
}

extern "C" int ddpo_threefry_normal(const uint32_t* key_dev, float* out, int64_t n, void* stream) {
  DDPO_REQUIRE(n > 0 && n < (int64_t(1) << 32), "ddpo_threefry_normal: n out of range");
  const int threads = 256;
  int64_t blocks = ((n + 1) / 2 + threads - 1) / threads;
  if (blocks > 132 * 16) blocks = 132 * 16;
  threefry_normal_kernel<<<(int)blocks, threads, 0, static_cast<cudaStream_t>(stream)>>>(key_dev, out, (uint32_t)n);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

static int check_ddim(const ddpo_ddim_common* c) {
  DDPO_REQUIRE(c != nullptr && c->eps_uncond && c->eps_cond && c->sample && c->alphas_cumprod && c->timesteps &&
                   c->workspace,
               "ddim: null pointer in arguments");
  DDPO_REQUIRE(c->batch > 0 && c->n > 0 && c->n % 4 == 0, "ddim: batch=%d n=%d (n must be a multiple of 4)", c->batch,
               c->n);
  DDPO_REQUIRE(c->timestep_stride == 0 || c->timestep_stride == 1, "ddim: timestep_stride must be 0 or 1");
  DDPO_REQUIRE(c->prediction_type >= DDPO_PRED_EPSILON && c->prediction_type <= DDPO_PRED_V,
               "ddim: prediction_type given as %d must be one of epsilon (0), sample (1) or v_prediction (2)",
               c->prediction_type);
  return DDPO_OK;
}

extern "C" int ddpo_ddim_step_sample(const ddpo_ddim_common* c, const uint32_t* key_dev, float* prev_sample,
                                     float* log_prob, void* stream) {
  int rc = check_ddim(c);
  if (rc) return rc;
  DDPO_REQUIRE(key_dev && prev_sample && log_prob, "ddim_step_sample: null output/key");
  dim3 grid(DDPO_DDIM_CHUNKS, c->batch);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (c->prediction_type == DDPO_PRED_EPSILON)
    ddim_step_kernel<0, DDPO_PRED_EPSILON><<<grid, DDIM_THREADS, 0, st>>>(*c, key_dev, prev_sample, log_prob);
  else if (c->prediction_type == DDPO_PRED_SAMPLE)
    ddim_step_kernel<0, DDPO_PRED_SAMPLE><<<grid, DDIM_THREADS, 0, st>>>(*c, key_dev, prev_sample, log_prob);
  else
    ddim_step_kernel<0, DDPO_PRED_V><<<grid, DDIM_THREADS, 0, st>>>(*c, key_dev, prev_sample, log_prob);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_ddim_logprob_fwd(const ddpo_ddim_common* c, const float* prev_sample, float* log_prob,
                                     void* stream) {
  int rc = check_ddim(c);
  if (rc) return rc;
  DDPO_REQUIRE(prev_sample && log_prob, "ddim_logprob_fwd: null pointer");
  dim3 grid(DDPO_DDIM_CHUNKS, c->batch);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* pv = const_cast<float*>(prev_sample);
  if (c->prediction_type == DDPO_PRED_EPSILON)
    ddim_step_kernel<1, DDPO_PRED_EPSILON><<<grid, DDIM_THREADS, 0, st>>>(*c, nullptr, pv, log_prob);
  else if (c->prediction_type == DDPO_PRED_SAMPLE)
    ddim_step_kernel<1, DDPO_PRED_SAMPLE><<<grid, DDIM_THREADS, 0, st>>>(*c, nullptr, pv, log_prob);
  else
    ddim_step_kernel<1, DDPO_PRED_V><<<grid, DDIM_THREADS, 0, st>>>(*c, nullptr, pv, log_prob);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_ddim_logprob_bwd(const ddpo_ddim_common* c, const float* prev_sample, const float* dlogp,
                                     float* d_eps_uncond, float* d_eps_cond, void* stream) {
  int rc = check_ddim(c);
  if (rc) return rc;
  DDPO_REQUIRE(prev_sample && dlogp && d_eps_cond, "ddim_logprob_bwd: null pointer");
  dim3 grid(DDPO_DDIM_CHUNKS, c->batch);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (c->prediction_type == DDPO_PRED_EPSILON)
    ddim_logprob_bwd_kernel<DDPO_PRED_EPSILON><<<grid, DDIM_THREADS, 0, st>>>(*c, prev_sample, dlogp, d_eps_uncond, d_eps_cond);
  else if (c->prediction_type == DDPO_PRED_SAMPLE)
    ddim_logprob_bwd_kernel<DDPO_PRED_SAMPLE><<<grid, DDIM_THREADS, 0, st>>>(*c, prev_sample, dlogp, d_eps_uncond, d_eps_cond);
  else
    ddim_logprob_bwd_kernel<DDPO_PRED_V><<<grid, DDIM_THREADS, 0, st>>>(*c, prev_sample, dlogp, d_eps_uncond, d_eps_cond);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_ppo_loss(const float* log_prob, const float* old_log_prob, const float* advantages, int batch,
                             int micro_batch, float clip_range, float* info3, float* dlogp, void* stream) {
  DDPO_REQUIRE(log_prob && old_log_prob && advantages && info3, "ppo_loss: null pointer");
  DDPO_REQUIRE(batch > 0 && batch <= 65536, "ppo_loss: batch=%d out of range", batch);
  DDPO_REQUIRE(micro_batch > 0 && batch % micro_batch == 0, "ppo_loss: micro_batch must divide batch");
  ppo_loss_kernel<<<1, 256, 0, static_cast<cudaStream_t>(stream)>>>(log_prob, old_log_prob, advantages, batch,
                                                                   micro_batch, clip_range, info3, dlogp);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}
