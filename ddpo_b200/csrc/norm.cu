// GroupNorm(32)+SiLU and LayerNorm, forward and backward (HBM-bound; fp32 statistics).
//
// Replaces flax.linen.GroupNorm / LayerNorm (+ nn.swish) inside the 3P diffusers Flax
// U-Net (FlaxResnetBlock2D norm1/norm2, FlaxTransformer2DModel.norm, conv_norm_out,
// FlaxBasicTransformerBlock norm1..3), reached from the reference at
// pipeline_flax_stable_diffusion.py:219-224 / training/policy_gradient.py:87-102.
// Flax statistics: mean, var = max(0, E[x^2] - E[x]^2), eps = 1e-5 everywhere.
//
// Layout: x fp32 NHWC [B, HW, C] (optionally the channel concat of two tensors: the
// U-Net skip connection is never materialised), y bf16 (the next GEMM's A operand).
//
// Statistics.  The GEMM that PRODUCES x leaves per-(32-row slab, channel) sums and sums of squares of what it writes
// (igemm.cu epilogue); gn_finalize_slabs_kernel folds them, in a fixed order, into one (mean, rstd) pair per
// (sample, group) -- so the forward pass reads x ONCE (algorithmic traffic: 4 B in + 2 B out per element) instead of
// once for the statistics and once more for the normalisation.  Inputs without slab statistics (conv_in's output, the VAE
// decoder, grids with fewer than 32 pixels) go through gn_stats_kernel (per (sample, pixel-chunk) partial sums) and
// gn_finalize_chunks_kernel.  Either way the reduction order depends on (HW, C) only, never on the batch size ->
// batch-invariant, bit-reproducible results.
//
// Apply.  gn_apply_kernel runs on the same (pixel chunk, sample) grid as gn_stats_kernel: a thread owns a channel quad
// (the per-channel affine coefficients in registers) and keeps four independent 16-byte loads of x in flight.
#include "common.cuh"

#include "reduce.cuh"

namespace ddpo {

constexpr int GN_THREADS = 512;
constexpr int GN_GROUPS = 32;

struct GnArgs {
  const float* x0;
  const float* x1;
  int c0, c1, ld0, ld1;
  int hw, chunks, pix_per_chunk;
  const float* scale;
  const float* bias;
  float* partial;  // [B, chunks, 32, 2]
  float eps;
  int silu;
  __nv_bfloat16* y_bf16;   // [B, HW, C] or null
  float* y_f32;            // [B, HW, C] or null
  __nv_bfloat16* raw_bf16;  // [B, HW, C] un-normalised copy or null
  const float* stats0;  // slab statistics of x0 / x1 ([B*HW/32, c, 2]) or null
  const float* stats1;
  float* mr;            // [B, 32, 2] (mean, rstd): written by the finalize kernels, read by every apply / backward kernel
};

__device__ __forceinline__ float2 gn_load2(const GnArgs& a, size_t pix, int c) {
  if (c < a.c0) return *reinterpret_cast<const float2*>(a.x0 + pix * a.ld0 + c);
  return *reinterpret_cast<const float2*>(a.x1 + pix * a.ld1 + (c - a.c0));
}

// grid (chunks, B).  thread -> (row r, channel quad); loops pixels r, r+R, ... with 128-bit loads, 4 pixels in
// flight.  Per-channel partial sums go to shared memory, then one warp per group reduces (rows x channels of
// the group) in a fixed order -> chunk partials.  (A channel quad may straddle two groups: cpg = 10, 30.)
__device__ __forceinline__ float4 gn_load4(const GnArgs& a, size_t pix, int c) {
  if (c < a.c0) return *reinterpret_cast<const float4*>(a.x0 + pix * a.ld0 + c);
  return *reinterpret_cast<const float4*>(a.x1 + pix * a.ld1 + (c - a.c0));
}

__global__ void __launch_bounds__(GN_THREADS) gn_stats_kernel(const GnArgs a) {
  const int C = a.c0 + a.c1, C4 = C >> 2, cpg = C / GN_GROUPS;
  const int cols = C4 < GN_THREADS ? C4 : GN_THREADS;
  const int R = GN_THREADS / cols;
  const int tc = threadIdx.x % cols, tr = threadIdx.x / cols;
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int p_begin = chunk * a.pix_per_chunk;
  const int p_end = min(a.hw, p_begin + a.pix_per_chunk);
  extern __shared__ float sm[];  // [R][C][2]
  const size_t base = static_cast<size_t>(b) * a.hw;
  if (tr < R) {
    for (int c4 = tc; c4 < C4; c4 += cols) {
      const int c = c4 * 4;
      float s[4] = {0.f, 0.f, 0.f, 0.f}, ss[4] = {0.f, 0.f, 0.f, 0.f};
      int p = p_begin + tr;
      for (; p + 3 * R < p_end; p += 4 * R) {
        const float4 v0 = gn_load4(a, base + p, c), v1 = gn_load4(a, base + p + R, c);
        const float4 v2 = gn_load4(a, base + p + 2 * R, c), v3 = gn_load4(a, base + p + 3 * R, c);
        s[0] += (v0.x + v1.x) + (v2.x + v3.x), s[1] += (v0.y + v1.y) + (v2.y + v3.y);
        s[2] += (v0.z + v1.z) + (v2.z + v3.z), s[3] += (v0.w + v1.w) + (v2.w + v3.w);
        ss[0] += (v0.x * v0.x + v1.x * v1.x) + (v2.x * v2.x + v3.x * v3.x);
        ss[1] += (v0.y * v0.y + v1.y * v1.y) + (v2.y * v2.y + v3.y * v3.y);
        ss[2] += (v0.z * v0.z + v1.z * v1.z) + (v2.z * v2.z + v3.z * v3.z);
        ss[3] += (v0.w * v0.w + v1.w * v1.w) + (v2.w * v2.w + v3.w * v3.w);
      }
      for (; p < p_end; p += R) {
        const float4 v = gn_load4(a, base + p, c);
        s[0] += v.x, s[1] += v.y, s[2] += v.z, s[3] += v.w;
        ss[0] += v.x * v.x, ss[1] += v.y * v.y, ss[2] += v.z * v.z, ss[3] += v.w * v.w;
      }
      float* o = sm + (static_cast<size_t>(tr) * C + c) * 2;
#pragma unroll
      for (int j = 0; j < 4; ++j) o[2 * j] = s[j], o[2 * j + 1] = ss[j];
    }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int g = warp; g < GN_GROUPS; g += GN_THREADS / 32) {
    float s = 0.f, ss = 0.f;
    const int n_items = cpg * R;
    for (int i = lane; i < n_items; i += 32) {
      const int c = g * cpg + i % cpg, r = i / cpg;
      s += sm[(static_cast<size_t>(r) * C + c) * 2];
      ss += sm[(static_cast<size_t>(r) * C + c) * 2 + 1];
    }
    s = warp_sum(s), ss = warp_sum(ss);
    if (lane == 0) {
      float* o = a.partial + ((static_cast<size_t>(b) * a.chunks + chunk) * GN_GROUPS + g) * 2;
      o[0] = s, o[1] = ss;
    }
  }
}

// (mean, rstd) of every (sample, group) from the producing GEMMs' slab statistics.  One 256-thread CTA per (sample, group):
// thread t adds items t, t + 256, ... of the (slab, channel-of-group) list in ascending order, then a fixed shuffle tree and
// the eight warp sums in warp order.
constexpr int GNF_THREADS = 256;
__global__ void __launch_bounds__(GNF_THREADS) gn_finalize_slabs_kernel(const GnArgs a, int batch) {
  const int C = a.c0 + a.c1, cpg = C / GN_GROUPS;
  const int b = blockIdx.x / GN_GROUPS, g = blockIdx.x % GN_GROUPS;
  const int nslab = a.hw >> 5;
  const int items = nslab * cpg;
  float s = 0.f, ss = 0.f;
  // eight independent loads per thread in flight (a plain accumulate loop serialises on the load
  // latency), summed in ascending item order
  for (int base = threadIdx.x; base < items; base += GNF_THREADS * 8) {
    float2 v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = base + u * GNF_THREADS;
      v[u] = make_float2(0.f, 0.f);
      if (i < items) {
        const int slab = i / cpg, c = g * cpg + (i - slab * cpg);
        const size_t row = static_cast<size_t>(b) * nslab + slab;
        v[u] = c < a.c0 ? *reinterpret_cast<const float2*>(a.stats0 + (row * a.c0 + c) * 2)
                        : *reinterpret_cast<const float2*>(a.stats1 + (row * a.c1 + (c - a.c0)) * 2);
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) s += v[u].x, ss += v[u].y;
  }
  __shared__ float red[2][GNF_THREADS / 32];
  s = warp_sum(s), ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[0][threadIdx.x >> 5] = s, red[1][threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x == 0) {
    s = ss = 0.f;
#pragma unroll
    for (int w = 0; w < GNF_THREADS / 32; ++w) s += red[0][w], ss += red[1][w];
    const float inv_n = 1.0f / (static_cast<float>(a.hw) * cpg);
    const float mean = s * inv_n;
    const float var = fmaxf(0.f, ss * inv_n - mean * mean);
    a.mr[blockIdx.x * 2] = mean, a.mr[blockIdx.x * 2 + 1] = rsqrtf(var + a.eps);
  }
}

// same from gn_stats_kernel's chunk partials (inputs nobody left slab statistics for): thread per (sample, group).
// The partials are folded in fp64: a sequential fp32 sum of the 512 chunks of a 512^2 VAE group lost up to 512 roundings
// of E[x^2], which E[x^2] - E[x]^2 multiplies by (mean / sigma)^2 -- 6.8x the error of torch fp32 at a 64 sigma offset.
__global__ void gn_finalize_chunks_kernel(const GnArgs a, int batch) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch * GN_GROUPS) return;
  const int b = i / GN_GROUPS, g = i % GN_GROUPS, cpg = (a.c0 + a.c1) / GN_GROUPS;
  double s = 0.0, ss = 0.0;
  for (int ch = 0; ch < a.chunks; ++ch) {
    const float* o = a.partial + ((static_cast<size_t>(b) * a.chunks + ch) * GN_GROUPS + g) * 2;
    s += o[0], ss += o[1];
  }
  const double inv_n = 1.0 / (static_cast<double>(a.hw) * cpg);
  const double mean = s * inv_n;
  const float var = static_cast<float>(fmax(0.0, ss * inv_n - mean * mean));
  a.mr[i * 2] = static_cast<float>(mean), a.mr[i * 2 + 1] = rsqrtf(var + a.eps);
}

// Per-element arithmetic of the apply kernel: the affine part as ONE fused multiply-add y = x * A + B with
// A = rstd * scale, B = bias - mean * A (per thread and channel, computed once), SiLU on one MUFU op when the only
// consumer is the bf16 GEMM operand.  The apply pass was issue- / MUFU-bound with the three-instruction affine and the
// two-MUFU sigmoid.
__device__ __forceinline__ void gn_coef(float mean, float rstd, float scale, float bias, float& A, float& B) {
  A = rstd * scale;
  B = fmaf(-mean, A, bias);
}
template <bool FAST>
__device__ __forceinline__ float gn_act(float x, float A, float B, int silu) {
  const float y = fmaf(x, A, B);
  if (!silu) return y;
  return FAST ? silu_bf16_f(y) : silu_f(y);
}

__global__ void __launch_bounds__(GN_THREADS) gn_apply_kernel(const GnArgs a) {
  const int C = a.c0 + a.c1, C4 = C >> 2, cpg = C / GN_GROUPS;
  const int cols = C4 < GN_THREADS ? C4 : GN_THREADS;
  const int R = GN_THREADS / cols;
  const int tc = threadIdx.x % cols, tr = threadIdx.x / cols;
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int p_begin = chunk * a.pix_per_chunk;
  const int p_end = min(a.hw, p_begin + a.pix_per_chunk);
  __shared__ float s_mean[GN_GROUPS], s_rstd[GN_GROUPS];
  if (threadIdx.x < GN_GROUPS) {
    s_mean[threadIdx.x] = a.mr[(b * GN_GROUPS + threadIdx.x) * 2];
    s_rstd[threadIdx.x] = a.mr[(b * GN_GROUPS + threadIdx.x) * 2 + 1];
  }
  __syncthreads();
  if (tr >= R) return;
  const size_t base = static_cast<size_t>(b) * a.hw;
  for (int c4 = tc; c4 < C4; c4 += cols) {
    const int c = c4 * 4;
    const float4 sc = *reinterpret_cast<const float4*>(a.scale + c);
    const float4 bi = *reinterpret_cast<const float4*>(a.bias + c);
    const float scv[4] = {sc.x, sc.y, sc.z, sc.w}, biv[4] = {bi.x, bi.y, bi.z, bi.w};
    float cA[4], cB[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int g = (c + j) / cpg;
      gn_coef(s_mean[g], s_rstd[g], scv[j], biv[j], cA[j], cB[j]);
    }
    const bool fast = a.y_f32 == nullptr;
    auto emit = [&](size_t pix, const float4& v) {
      const float xv[4] = {v.x, v.y, v.z, v.w};
      float y[4];
      if (fast) {
#pragma unroll
        for (int j = 0; j < 4; ++j) y[j] = gn_act<true>(xv[j], cA[j], cB[j], a.silu);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) y[j] = gn_act<false>(xv[j], cA[j], cB[j], a.silu);
      }
      if (a.y_bf16) *reinterpret_cast<uint2*>(a.y_bf16 + pix * C + c) = make_uint2(pack_bf16(y[0], y[1]), pack_bf16(y[2], y[3]));
      if (a.y_f32) *reinterpret_cast<float4*>(a.y_f32 + pix * C + c) = make_float4(y[0], y[1], y[2], y[3]);
      if (a.raw_bf16)
        *reinterpret_cast<uint2*>(a.raw_bf16 + pix * C + c) = make_uint2(pack_bf16(xv[0], xv[1]), pack_bf16(xv[2], xv[3]));
    };
    int p = p_begin + tr;
    for (; p + 3 * R < p_end; p += 4 * R) {  // four independent 16-byte loads in flight per thread
      const float4 v0 = gn_load4(a, base + p, c), v1 = gn_load4(a, base + p + R, c);
      const float4 v2 = gn_load4(a, base + p + 2 * R, c), v3 = gn_load4(a, base + p + 3 * R, c);
      emit(base + p, v0), emit(base + p + R, v1), emit(base + p + 2 * R, v2), emit(base + p + 3 * R, v3);
    }
    for (; p < p_end; p += R) emit(base + p, gn_load4(a, base + p, c));
  }
}

// ---------------------------------------------------------------- GN backward ----
// y = xhat * scale + bias (then optional SiLU).  Given dy (fp32, w.r.t. the post-activation
// output) computes dx = rstd * (dy' * scale - mean_g(dy' * scale) - xhat * mean_g(dy' * scale * xhat))
// and per-(sample, chunk) partial dscale / dbias (summed in fixed order by gn_param_grad_kernel).
struct GnBwdArgs {
  GnArgs f;
  const void* dy;      // [B, HW, C] gradient w.r.t. GN(+SiLU) output: fp32, or bf16 when dy_bf16
  int dy_bf16;
  float* partial2;     // [B, chunks, 32, 2]: sum(dyh), sum(dyh * xhat)
  float* dx0;          // [B, HW, ld] gradient into x0 (+= if accumulate)
  float* dx1;
  int ldd0, ldd1;
  int accumulate;
  float* dparam_part;  // [B, chunks, 2, C]  partial (dscale, dbias)
};

// four consecutive gradient values at element index `idx` (a multiple of 4).  The element type is a TEMPLATE parameter of
// the kernels: with a run-time branch inside the unrolled load loops the compiler stops batching the row's loads.
template <bool BF16>
__device__ __forceinline__ float4 gn_load_dy4(const void* dy, size_t idx) {
  if (BF16) {
    const uint2 u = *reinterpret_cast<const uint2*>(static_cast<const __nv_bfloat16*>(dy) + idx);
    return make_float4(bf16_lo(u.x), bf16_hi(u.x), bf16_lo(u.y), bf16_hi(u.y));
  }
  return *reinterpret_cast<const float4*>(static_cast<const float*>(dy) + idx);
}

__device__ __forceinline__ float silu_grad_f(float z) {
  const float s = sigmoid_f(z);
  return s * (1.0f + z * (1.0f - s));
}

// pass 1: per-group sums of dyh = dy*act'(z)*scale and dyh*xhat ; also dscale/dbias partials.
// Same thread mapping as the forward (row r, channel quad, 128-bit loads); per-channel partials in shared memory.
template <bool DY_BF16>
__global__ void __launch_bounds__(GN_THREADS) gn_bwd_stats_kernel(const GnBwdArgs a) {
  const GnArgs& f = a.f;
  const int C = f.c0 + f.c1, C4 = C >> 2, cpg = C / GN_GROUPS;
  const int cols = C4 < GN_THREADS ? C4 : GN_THREADS;
  const int R = GN_THREADS / cols;
  const int tc = threadIdx.x % cols, tr = threadIdx.x / cols;
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int p_begin = chunk * f.pix_per_chunk;
  const int p_end = min(f.hw, p_begin + f.pix_per_chunk);
  extern __shared__ float sm[];  // [R][C][4] : a0, a1, dscale, dbias per channel
  __shared__ float s_mean[GN_GROUPS], s_rstd[GN_GROUPS];
  if (threadIdx.x < GN_GROUPS) {
    s_mean[threadIdx.x] = f.mr[(b * GN_GROUPS + threadIdx.x) * 2];
    s_rstd[threadIdx.x] = f.mr[(b * GN_GROUPS + threadIdx.x) * 2 + 1];
  }
  __syncthreads();
  const size_t base = static_cast<size_t>(b) * f.hw;
  if (tr < R) {
    for (int c4 = tc; c4 < C4; c4 += cols) {
      const int c = c4 * 4;
      const float4 sc4 = *reinterpret_cast<const float4*>(f.scale + c);
      const float4 bi4 = *reinterpret_cast<const float4*>(f.bias + c);
      const float sc[4] = {sc4.x, sc4.y, sc4.z, sc4.w}, bi[4] = {bi4.x, bi4.y, bi4.z, bi4.w};
      float mu[4], rs[4], a0[4] = {0, 0, 0, 0}, a1[4] = {0, 0, 0, 0}, ds[4] = {0, 0, 0, 0}, db[4] = {0, 0, 0, 0};
#pragma unroll
      for (int j = 0; j < 4; ++j) mu[j] = s_mean[(c + j) / cpg], rs[j] = s_rstd[(c + j) / cpg];
      for (int p = p_begin + tr; p < p_end; p += R) {
        const size_t pix = base + p;
        const float4 v = gn_load4(f, pix, c);
        const float4 d4 = gn_load_dy4<DY_BF16>(a.dy, pix * C + c);
        const float xv[4] = {v.x, v.y, v.z, v.w};
        float d[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float xh = (xv[j] - mu[j]) * rs[j];
          if (f.silu) d[j] *= silu_grad_f(xh * sc[j] + bi[j]);
          ds[j] += d[j] * xh;
          db[j] += d[j];
          a0[j] += d[j] * sc[j];
          a1[j] += d[j] * sc[j] * xh;
        }
      }
      float* o = sm + (static_cast<size_t>(tr) * C + c) * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) o[4 * j] = a0[j], o[4 * j + 1] = a1[j], o[4 * j + 2] = ds[j], o[4 * j + 3] = db[j];
    }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int g = warp; g < GN_GROUPS; g += GN_THREADS / 32) {
    float s = 0.f, ss = 0.f;
    const int n_items = cpg * R;
    for (int i = lane; i < n_items; i += 32) {
      const int c = g * cpg + i % cpg, r = i / cpg;
      s += sm[(static_cast<size_t>(r) * C + c) * 4];
      ss += sm[(static_cast<size_t>(r) * C + c) * 4 + 1];
    }
    s = warp_sum(s), ss = warp_sum(ss);
    if (lane == 0) {
      float* o = a.partial2 + ((static_cast<size_t>(b) * f.chunks + chunk) * GN_GROUPS + g) * 2;
      o[0] = s, o[1] = ss;
    }
  }
  float* dp = a.dparam_part + (static_cast<size_t>(b) * f.chunks + chunk) * 2 * C;
  for (int c = threadIdx.x; c < C; c += GN_THREADS) {
    float ds = 0.f, db = 0.f;
    for (int r = 0; r < R; ++r) {
      ds += sm[(static_cast<size_t>(r) * C + c) * 4 + 2];
      db += sm[(static_cast<size_t>(r) * C + c) * 4 + 3];
    }
    dp[c] = ds;
    dp[C + c] = db;
  }
}

// pass 2: dx
template <bool DY_BF16>
__global__ void __launch_bounds__(GN_THREADS, 2) gn_bwd_apply_kernel(const GnBwdArgs a) {
  const GnArgs& f = a.f;
  const int C = f.c0 + f.c1, C4 = C >> 2, cpg = C / GN_GROUPS;
  const int cols = C4 < GN_THREADS ? C4 : GN_THREADS;
  const int R = GN_THREADS / cols;
  const int tc = threadIdx.x % cols, tr = threadIdx.x / cols;
  // descending order: the stats pass finished on the last samples / chunks, start with those
  const int b = gridDim.y - 1 - blockIdx.y, chunk = gridDim.x - 1 - blockIdx.x;
  const int p_begin = chunk * f.pix_per_chunk;
  const int p_end = min(f.hw, p_begin + f.pix_per_chunk);
  __shared__ float s_mean[GN_GROUPS], s_rstd[GN_GROUPS], s_m1[GN_GROUPS], s_m2[GN_GROUPS];
  if (threadIdx.x < GN_GROUPS) {
    float p1 = 0.f, p2 = 0.f;
    for (int ch = 0; ch < f.chunks; ++ch) {
      const size_t o = ((static_cast<size_t>(b) * f.chunks + ch) * GN_GROUPS + threadIdx.x) * 2;
      p1 += a.partial2[o], p2 += a.partial2[o + 1];
    }
    const float inv_n = 1.0f / (static_cast<float>(f.hw) * cpg);
    s_mean[threadIdx.x] = f.mr[(b * GN_GROUPS + threadIdx.x) * 2];
    s_rstd[threadIdx.x] = f.mr[(b * GN_GROUPS + threadIdx.x) * 2 + 1];
    s_m1[threadIdx.x] = p1 * inv_n;
    s_m2[threadIdx.x] = p2 * inv_n;
  }
  __syncthreads();
  if (tr >= R) return;
  const size_t base = static_cast<size_t>(b) * f.hw;
  for (int c4 = tc; c4 < C4; c4 += cols) {
    const int c = c4 * 4;
    const float4 sc4 = *reinterpret_cast<const float4*>(f.scale + c);
    const float4 bi4 = *reinterpret_cast<const float4*>(f.bias + c);
    const float sc[4] = {sc4.x, sc4.y, sc4.z, sc4.w}, bi[4] = {bi4.x, bi4.y, bi4.z, bi4.w};
    float mu[4], rs[4], m1[4], m2[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int g = (c + j) / cpg;
      mu[j] = s_mean[g], rs[j] = s_rstd[g], m1[j] = s_m1[g], m2[j] = s_m2[g];
    }
    const bool src0 = c < f.c0;
    auto emit = [&](size_t pix, const float4& v, const float4& d4, const float4& old) {
      const float xv[4] = {v.x, v.y, v.z, v.w};
      float d[4] = {d4.x, d4.y, d4.z, d4.w}, o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xh = (xv[j] - mu[j]) * rs[j];
        if (f.silu) d[j] *= silu_grad_f(xh * sc[j] + bi[j]);
        o[j] = rs[j] * (d[j] * sc[j] - m1[j] - xh * m2[j]);
      }
      float* dst = src0 ? a.dx0 + pix * a.ldd0 + c : a.dx1 + pix * a.ldd1 + (c - f.c0);
      float4 out = make_float4(o[0], o[1], o[2], o[3]);
      if (a.accumulate) out.x += old.x, out.y += old.y, out.z += old.z, out.w += old.w;
      *reinterpret_cast<float4*>(dst) = out;
    };
    auto load_old = [&](size_t pix) {
      if (!a.accumulate) return make_float4(0.f, 0.f, 0.f, 0.f);
      const float* dst = src0 ? a.dx0 + pix * a.ldd0 + c : a.dx1 + pix * a.ldd1 + (c - f.c0);
      return *reinterpret_cast<const float4*>(dst);
    };
    int p = p_begin + tr;
    for (; p + R < p_end; p += 2 * R) {  // two pixels = up to six independent 16-byte loads in flight per thread
      const size_t q0 = base + p, q1 = base + p + R;
      const float4 v0 = gn_load4(f, q0, c), v1 = gn_load4(f, q1, c);
      const float4 d0 = gn_load_dy4<DY_BF16>(a.dy, q0 * C + c);
      const float4 d1 = gn_load_dy4<DY_BF16>(a.dy, q1 * C + c);
      const float4 o0 = load_old(q0), o1 = load_old(q1);
      emit(q0, v0, d0, o0), emit(q1, v1, d1, o1);
    }
    for (; p < p_end; p += R) {
      const size_t q0 = base + p;
      emit(q0, gn_load4(f, q0, c), gn_load_dy4<DY_BF16>(a.dy, q0 * C + c), load_old(q0));
    }
  }
}

// dscale/dbias: partial [rows, 2, C] summed over rows in fixed order into the gradients: reduce_rows_kernel (reduce.cuh)

// ------------------------------------------------------------------ LayerNorm ----
// one warp per row, ROWS rows per warp in flight; the row lives in registers (NC = ceil(C / 128) float4 per lane), so x is
// read once and ROWS * NC independent 16-byte loads per lane are outstanding before the first reduction.
// x fp32 [M, C] -> y bf16 [M, C].  Summation order per row: lane-strided columns in ascending order, then the xor tree.
template <int NC, int ROWS>
__global__ void __launch_bounds__(256) layernorm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ scale,
                                                            const float* __restrict__ bias, __nv_bfloat16* __restrict__ y,
                                                            float* __restrict__ stats, int M, int C, float eps) {
  const int row0 = (blockIdx.x * 8 + (threadIdx.x >> 5)) * ROWS;
  const int lane = threadIdx.x & 31;
  if (row0 >= M) return;
  float4 v[ROWS][NC];
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    const float* xr = x + static_cast<size_t>(row0 + r) * C;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int c = lane * 4 + 128 * i;
      v[r][i] = (c < C && row0 + r < M) ? *reinterpret_cast<const float4*>(xr + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  float4 sc[NC], bi[NC];
#pragma unroll
  for (int i = 0; i < NC; ++i) {
    const int c = lane * 4 + 128 * i;
    if (c < C) {
      sc[i] = __ldg(reinterpret_cast<const float4*>(scale + c));
      bi[i] = __ldg(reinterpret_cast<const float4*>(bias + c));
    }
  }
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    const int row = row0 + r;
    float s = 0.f, ss = 0.f;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      if (lane * 4 + 128 * i < C) {
        const float4 q = v[r][i];
        s += (q.x + q.y) + (q.z + q.w);
        ss += (q.x * q.x + q.y * q.y) + (q.z * q.z + q.w * q.w);
      }
    }
    s = warp_sum(s), ss = warp_sum(ss);
    if (row >= M) continue;   // warp-uniform
    const float mean = s / C;
    const float rstd = rsqrtf(fmaxf(0.f, ss / C - mean * mean) + eps);
    if (stats != nullptr && lane == 0) stats[row * 2] = mean, stats[row * 2 + 1] = rstd;
    __nv_bfloat16* yr = y + static_cast<size_t>(row) * C;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int c = lane * 4 + 128 * i;
      if (c < C) {
        const float4 q = v[r][i];
        uint2 o;
        o.x = pack_bf16((q.x - mean) * rstd * sc[i].x + bi[i].x, (q.y - mean) * rstd * sc[i].y + bi[i].y);
        o.y = pack_bf16((q.z - mean) * rstd * sc[i].z + bi[i].z, (q.w - mean) * rstd * sc[i].w + bi[i].w);
        *reinterpret_cast<uint2*>(yr + c) = o;
      }
    }
  }
}

// backward: dx (+)= rstd * (dy*scale - mean(dy*scale) - xhat * mean(dy*scale*xhat)); per-CTA dscale/dbias partials.
// One warp per row; a lane owns columns lane*4 + 128*i, so its dscale/dbias partial sums live in registers
// (NC = ceil(C/128) column groups); cross-warp reduction through shared memory in fixed order.
constexpr int LN_BWD_ROWS = 64;  // rows per CTA (8 warps x 8 rows)
template <int NC, bool DY_BF16>
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ scale,
                                                            const float* __restrict__ stats, const void* __restrict__ dy,
                                                            float* __restrict__ dx, float* __restrict__ dparam_part,
                                                            int M, int C, int accumulate) {
  extern __shared__ float sm[];  // [8 warps][2][C]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float ds[NC][4], db[NC][4];
  float4 sc[NC];
#pragma unroll
  for (int i = 0; i < NC; ++i) {
    const int c = lane * 4 + 128 * i;
    sc[i] = c < C ? __ldg(reinterpret_cast<const float4*>(scale + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 4; ++j) ds[i][j] = 0.f, db[i][j] = 0.f;
  }
  for (int it = 0; it < LN_BWD_ROWS / 8; ++it) {
    const int row = blockIdx.x * LN_BWD_ROWS + it * 8 + warp;
    if (row >= M) break;
    const float mean = stats[row * 2], rstd = stats[row * 2 + 1];
    const float* xr = x + static_cast<size_t>(row) * C;
    const size_t dr = static_cast<size_t>(row) * C;   // element offset of this row in dy
    float* gr = dx + static_cast<size_t>(row) * C;
    float4 xv[NC], dv[NC], ov[NC];  // the old gradient (accumulate mode) is fetched with x and dy: 3 streams in flight
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int c = lane * 4 + 128 * i;
      ov[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c < C) {
        xv[i] = *reinterpret_cast<const float4*>(xr + c);
        dv[i] = gn_load_dy4<DY_BF16>(dy, dr + c);
        if (accumulate) ov[i] = *reinterpret_cast<const float4*>(gr + c);
      } else {
        xv[i] = make_float4(mean, mean, mean, mean);
        dv[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    float m1 = 0.f, m2 = 0.f;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const float xh[4] = {(xv[i].x - mean) * rstd, (xv[i].y - mean) * rstd, (xv[i].z - mean) * rstd, (xv[i].w - mean) * rstd};
      const float dd[4] = {dv[i].x, dv[i].y, dv[i].z, dv[i].w}, s4[4] = {sc[i].x, sc[i].y, sc[i].z, sc[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        m1 += dd[j] * s4[j];
        m2 += dd[j] * s4[j] * xh[j];
        ds[i][j] += dd[j] * xh[j];
        db[i][j] += dd[j];
      }
    }
    m1 = warp_sum(m1) / C, m2 = warp_sum(m2) / C;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int c = lane * 4 + 128 * i;
      if (c < C) {
        float4 o;
        o.x = rstd * (dv[i].x * sc[i].x - m1 - (xv[i].x - mean) * rstd * m2);
        o.y = rstd * (dv[i].y * sc[i].y - m1 - (xv[i].y - mean) * rstd * m2);
        o.z = rstd * (dv[i].z * sc[i].z - m1 - (xv[i].z - mean) * rstd * m2);
        o.w = rstd * (dv[i].w * sc[i].w - m1 - (xv[i].w - mean) * rstd * m2);
        o.x += ov[i].x, o.y += ov[i].y, o.z += ov[i].z, o.w += ov[i].w;
        *reinterpret_cast<float4*>(gr + c) = o;
      }
    }
  }
  float* my = sm + static_cast<size_t>(warp) * 2 * C;
#pragma unroll
  for (int i = 0; i < NC; ++i) {
    const int c = lane * 4 + 128 * i;
    if (c < C) {
      *reinterpret_cast<float4*>(my + c) = make_float4(ds[i][0], ds[i][1], ds[i][2], ds[i][3]);
      *reinterpret_cast<float4*>(my + C + c) = make_float4(db[i][0], db[i][1], db[i][2], db[i][3]);
    }
  }
  __syncthreads();
  float* dp = dparam_part + static_cast<size_t>(blockIdx.x) * 2 * C;
  for (int c = threadIdx.x; c < C; c += 256) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < 8; ++w) a += sm[(w * 2) * C + c], b += sm[(w * 2 + 1) * C + c];
    dp[c] = a;
    dp[C + c] = b;
  }
}

static int gn_chunking(int hw, int* chunks, int* ppc) {
  // 32 chunks per sample for the U-Net's grids (hw <= 4096); at most 512 pixels per chunk beyond that, so the VAE
  // decoder's 128^2 .. 512^2 levels (2-image chunks) still launch enough CTAs to fill 132 SMs.  The chunking depends
  // on hw only -> reduction order (and the result bits) are independent of the batch size.
  int p = hw / 32;
  if (p > 512) p = 512;
  if (p < 8) p = 8;
  if (p > hw) p = hw;
  *ppc = p;
  *chunks = (hw + p - 1) / p;
  return 0;
}

static int fill_gn(GnArgs& g, const ddpo_groupnorm_args* a) {
  const int C = a->c0 + a->c1;
  DDPO_REQUIRE(a->x0 != nullptr && a->c0 > 0 && C % (2 * GN_GROUPS) == 0 && a->c0 % 2 == 0,
               "groupnorm: channels must be a multiple of 64 and c0 even (c0=%d c1=%d)", a->c0, a->c1);
  DDPO_REQUIRE(a->scale && a->bias && a->workspace, "groupnorm: null scale/bias/workspace");
  g.x0 = a->x0, g.x1 = a->x1, g.c0 = a->c0, g.c1 = a->c1;
  g.ld0 = a->ld0 > 0 ? a->ld0 : a->c0, g.ld1 = a->ld1 > 0 ? a->ld1 : a->c1;
  g.hw = a->hw;
  gn_chunking(a->hw, &g.chunks, &g.pix_per_chunk);
  g.scale = a->scale, g.bias = a->bias, g.eps = a->eps, g.silu = a->silu;
  // workspace: [mr: B*64][forward chunk partials: B*chunks*64][backward partials: B*chunks*64][dscale/dbias partials]
  g.mr = a->workspace;
  g.partial = a->workspace + static_cast<size_t>(a->batch) * GN_GROUPS * 2;
  g.stats0 = a->stats0, g.stats1 = a->stats1;
  g.y_bf16 = static_cast<__nv_bfloat16*>(a->y_bf16), g.y_f32 = a->y_f32;
  g.raw_bf16 = static_cast<__nv_bfloat16*>(a->raw_bf16);
  return DDPO_OK;
}

static size_t gn_stats_smem(int C) {
  const int C4 = C / 4, cols = C4 < GN_THREADS ? C4 : GN_THREADS;
  const int R = GN_THREADS / cols;
  return static_cast<size_t>(R) * C * 2 * sizeof(float);
}

}  // namespace ddpo

using namespace ddpo;

extern "C" int64_t ddpo_groupnorm_workspace_floats(int batch, int hw, int channels) {
  int chunks, ppc;
  gn_chunking(hw, &chunks, &ppc);
  // (mean, rstd) table + fwd partials + bwd partials + dparam partials
  return static_cast<int64_t>(batch) * GN_GROUPS * 2 + static_cast<int64_t>(batch) * chunks * GN_GROUPS * 2 * 2 +
         static_cast<int64_t>(batch) * chunks * 2 * channels;
}

extern "C" int ddpo_groupnorm_fwd(const ddpo_groupnorm_args* a, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  GnArgs g;
  int rc = fill_gn(g, a);
  if (rc) return rc;
  dim3 grid(g.chunks, a->batch);
  const size_t smem = gn_stats_smem(a->c0 + a->c1);
  DDPO_REQUIRE(smem <= 48 * 1024, "groupnorm: too many channels (%d)", a->c0 + a->c1);
  DDPO_REQUIRE(a->c0 % 4 == 0 && g.ld0 % 4 == 0 && g.ld1 % 4 == 0, "groupnorm: channel counts / pitches must be multiples of 4");
  if (!a->stats_only_skip) {
    const bool have_slabs = a->stats0 != nullptr && (a->c1 == 0 || a->stats1 != nullptr) && a->hw % 32 == 0;
    const int n = a->batch * GN_GROUPS;
    if (have_slabs) {
      gn_finalize_slabs_kernel<<<n, GNF_THREADS, 0, stream>>>(g, a->batch);
    } else {
      gn_stats_kernel<<<grid, GN_THREADS, smem, stream>>>(g);
      DDPO_LAUNCH_OK();
      gn_finalize_chunks_kernel<<<(n + 127) / 128, 128, 0, stream>>>(g, a->batch);
    }
    DDPO_LAUNCH_OK();
  }
  if (g.y_bf16 || g.y_f32 || g.raw_bf16) {
    gn_apply_kernel<<<grid, GN_THREADS, 0, stream>>>(g);
    DDPO_LAUNCH_OK();
  }
  return DDPO_OK;
}

extern "C" int ddpo_groupnorm_bwd(const ddpo_groupnorm_args* a, const void* dy, float* dx0, float* dx1, int ldd0,
                                  int ldd1, int accumulate, float* dscale, float* dbias, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  GnBwdArgs b;
  int rc = fill_gn(b.f, a);
  if (rc) return rc;
  const int C = a->c0 + a->c1;
  DDPO_REQUIRE(dy && dx0 && dscale && dbias, "groupnorm_bwd: null pointer");
  b.dy = dy, b.dy_bf16 = a->dy_bf16, b.dx0 = dx0, b.dx1 = dx1, b.ldd0 = ldd0 > 0 ? ldd0 : a->c0, b.ldd1 = ldd1 > 0 ? ldd1 : a->c1;
  b.accumulate = accumulate;
  b.partial2 = b.f.partial + static_cast<size_t>(a->batch) * b.f.chunks * GN_GROUPS * 2;
  b.dparam_part = b.partial2 + static_cast<size_t>(a->batch) * b.f.chunks * GN_GROUPS * 2;
  dim3 grid(b.f.chunks, a->batch);
  const size_t smem = 2 * gn_stats_smem(C);
  static bool attr = false;
  if (!attr) {
    DDPO_CUDA_OK(cudaFuncSetAttribute(gn_bwd_stats_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    DDPO_CUDA_OK(cudaFuncSetAttribute(gn_bwd_stats_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    attr = true;
  }
  DDPO_REQUIRE(smem <= 96 * 1024, "groupnorm_bwd: too many channels (%d)", C);
  DDPO_REQUIRE(b.ldd0 % 4 == 0 && b.ldd1 % 4 == 0, "groupnorm_bwd: gradient pitches must be multiples of 4");
  if (b.dy_bf16) {
    gn_bwd_stats_kernel<true><<<grid, GN_THREADS, smem, stream>>>(b);
    DDPO_LAUNCH_OK();
    gn_bwd_apply_kernel<true><<<grid, GN_THREADS, 0, stream>>>(b);
  } else {
    gn_bwd_stats_kernel<false><<<grid, GN_THREADS, smem, stream>>>(b);
    DDPO_LAUNCH_OK();
    gn_bwd_apply_kernel<false><<<grid, GN_THREADS, 0, stream>>>(b);
  }
  DDPO_LAUNCH_OK();
  launch_reduce_rows(b.dparam_part, 1, a->batch * b.f.chunks, 2 * C, C, dscale, dbias, 1, stream);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_layernorm_fwd(const float* x, const float* scale, const float* bias, void* y_bf16, float* stats,
                                  int m, int c, float eps, void* stream) {
  DDPO_REQUIRE(x && scale && bias && y_bf16 && m > 0 && c % 4 == 0 && c <= 1280,
               "layernorm_fwd: bad arguments (m=%d c=%d; c <= 1280)", m, c);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  __nv_bfloat16* y = static_cast<__nv_bfloat16*>(y_bf16);
  const int nc = (c + 127) / 128;
  if (nc <= 3)
    layernorm_fwd_kernel<3, 4><<<(m + 31) / 32, 256, 0, st>>>(x, scale, bias, y, stats, m, c, eps);
  else if (nc <= 5)
    layernorm_fwd_kernel<5, 2><<<(m + 15) / 16, 256, 0, st>>>(x, scale, bias, y, stats, m, c, eps);
  else
    layernorm_fwd_kernel<10, 1><<<(m + 7) / 8, 256, 0, st>>>(x, scale, bias, y, stats, m, c, eps);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int64_t ddpo_layernorm_bwd_workspace_floats(int m, int c) {
  return static_cast<int64_t>((m + LN_BWD_ROWS - 1) / LN_BWD_ROWS) * 2 * c;
}

extern "C" int ddpo_layernorm_bwd(const float* x, const float* scale, const float* stats, const void* dy, float* dx,
                                  int accumulate, float* dscale, float* dbias, float* workspace, int m, int c, int dy_bf16,
                                  void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DDPO_REQUIRE(x && scale && stats && dy && dx && dscale && dbias && workspace && c % 4 == 0,
               "layernorm_bwd: bad arguments");
  const int ctas = (m + LN_BWD_ROWS - 1) / LN_BWD_ROWS;
  const size_t smem = static_cast<size_t>(8) * 2 * c * sizeof(float);
  DDPO_REQUIRE(c <= 1280 && smem <= 96 * 1024, "layernorm_bwd: C=%d too large (<= 1280)", c);
  static bool attr = false;
  if (!attr) {
    DDPO_CUDA_OK(cudaFuncSetAttribute(layernorm_bwd_kernel<3, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    DDPO_CUDA_OK(cudaFuncSetAttribute(layernorm_bwd_kernel<5, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    DDPO_CUDA_OK(cudaFuncSetAttribute(layernorm_bwd_kernel<10, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    DDPO_CUDA_OK(cudaFuncSetAttribute(layernorm_bwd_kernel<3, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    DDPO_CUDA_OK(cudaFuncSetAttribute(layernorm_bwd_kernel<5, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    DDPO_CUDA_OK(cudaFuncSetAttribute(layernorm_bwd_kernel<10, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    attr = true;
  }
  const int nc = (c + 127) / 128;
#define DDPO_LN_BWD(NC, BF)                                                                                           \
  layernorm_bwd_kernel<NC, BF><<<ctas, 256, smem, stream>>>(x, scale, stats, dy, dx, workspace, m, c, accumulate)
  if (dy_bf16) {
    if (nc <= 3) DDPO_LN_BWD(3, true);
    else if (nc <= 5) DDPO_LN_BWD(5, true);
    else DDPO_LN_BWD(10, true);
  } else {
    if (nc <= 3) DDPO_LN_BWD(3, false);
    else if (nc <= 5) DDPO_LN_BWD(5, false);
    else DDPO_LN_BWD(10, false);
  }
#undef DDPO_LN_BWD
  DDPO_LAUNCH_OK();
  launch_reduce_rows(workspace, 1, ctas, 2 * c, c, dscale, dbias, 1, stream);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}
