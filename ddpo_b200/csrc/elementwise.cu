// Small / memory-bound pieces of the U-Net forward: weight re-layout (fp32 Flax params ->
// bf16 GEMM operands), casts, nearest x2 up-sampling, conv_in (K=36) and conv_out (N=4)
// which are not tensor-core shaped, the sinusoidal timestep embedding and the M=batch
// dense layers of the time-embedding MLP.
//
// Reference: 3P diffusers==0.12.1 FlaxUNet2DConditionModel (conv_in, conv_out, FlaxTimesteps,
// FlaxTimestepEmbedding, FlaxUpsample2D, FlaxResnetBlock2D.time_emb_proj), reached from
// pipeline_flax_stable_diffusion.py:219-224 and training/policy_gradient.py:87-102.
#include "common.cuh"

namespace ddpo {

// -------------------------------------------------------------- weight prep ----
// src fp32 [K, N] (Flax: Dense kernel [in,out]; Conv HWIO flattened to [(tap,cin), cout])
// dst bf16 [N, K] with dst row = perm(n) (+row_offset), leading dim ldk, column offset col_offset.
// perm: GEGLU tile interleave when geglu_half > 0: first `geglu_half*?`... see below.
__global__ void prep_transpose_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int K, int N,
                                      int ldk, int row_offset, int col_offset, int geglu_bn) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.x * 32, n0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int k = k0 + i, n = n0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < K && n < N) ? src[static_cast<size_t>(k) * N + n] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int n = n0 + i, k = k0 + threadIdx.x;
    if (n < N && k < K) {
      int row = n;
      if (geglu_bn > 0) {
        // source columns [0, N/2) = linear, [N/2, N) = gate.  Destination N tile t (geglu_bn rows)
        // holds [geglu_bn/2 linear | geglu_bn/2 gate] of output channels [t*half, (t+1)*half)
        const int half = geglu_bn >> 1, hn = N >> 1;
        const int j = n < hn ? n : n - hn;
        row = (j / half) * geglu_bn + (n < hn ? 0 : half) + (j % half);
      }
      dst[static_cast<size_t>(row + row_offset) * ldk + col_offset + k] = __float2bfloat16_rn(tile[threadIdx.x][i]);
    }
  }
}

// backward-operand layout: dst bf16 [K_in, taps*N] = src[tap][k][n] with the tap index flipped
// (dgrad of a 3x3 conv is a 3x3 conv with the kernel rotated by 180 degrees; for taps==1 it is a cast)
__global__ void prep_dgrad_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int taps, int K,
                                  int N, int64_t total, int ld_dst, int col_offset) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int n = i % N;
  const int64_t r = i / N;
  const int k = r % K, tap = r / K;
  dst[static_cast<size_t>(k) * ld_dst + col_offset + (taps - 1 - tap) * N + n] = __float2bfloat16_rn(src[i]);
}

__global__ void permute_geglu_bias_kernel(const float* __restrict__ src, float* __restrict__ dst, int N, int bn) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const int half = bn >> 1, hn = N >> 1;
  const int j = n < hn ? n : n - hn;
  dst[(j / half) * bn + (n < hn ? 0 : half) + (j % half)] = src[n];
}

// ---------------------------------------------------------------- casts etc ----
__global__ void cast_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, int64_t n4) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    uint2 o;
    o.x = pack_bf16(v.x, v.y), o.y = pack_bf16(v.z, v.w);
    reinterpret_cast<uint2*>(y)[i] = o;
  }
}

// nearest x2 (jax.image.resize "nearest": out[i] = in[i // 2]); x fp32 [B,H,W,C] -> y bf16 [B,2H,2W,C]
__global__ void upsample2x_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, int B, int H, int W,
                                       int C4) {
  const int64_t total = static_cast<int64_t>(B) * H * W * C4;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c4 = i % C4;
    int64_t p = i / C4;
    const int w = p % W;
    p /= W;
    const int h = p % H;
    const int b = p / H;
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    uint2 o;
    o.x = pack_bf16(v.x, v.y), o.y = pack_bf16(v.z, v.w);
    const size_t W2 = 2 * W;
    const size_t base = ((static_cast<size_t>(b) * 2 * H + 2 * h) * W2 + 2 * w) * C4 + c4;
    uint2* yo = reinterpret_cast<uint2*>(y);
    yo[base] = o;
    yo[base + C4] = o;
    yo[base + W2 * C4] = o;
    yo[base + W2 * C4 + C4] = o;
  }
}

// upsample backward: dx[b,h,w,c] (+)= sum of the 2x2 block of dy
__global__ void upsample2x_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int B, int H, int W, int C4,
                                      int accumulate) {
  const int64_t total = static_cast<int64_t>(B) * H * W * C4;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c4 = i % C4;
    int64_t p = i / C4;
    const int w = p % W;
    p /= W;
    const int h = p % H;
    const int b = p / H;
    const size_t W2 = 2 * W;
    const size_t base = ((static_cast<size_t>(b) * 2 * H + 2 * h) * W2 + 2 * w) * C4 + c4;
    const float4* d = reinterpret_cast<const float4*>(dy);
    const float4 a0 = d[base], a1 = d[base + C4], a2 = d[base + W2 * C4], a3 = d[base + W2 * C4 + C4];
    float4 o = make_float4((a0.x + a1.x) + (a2.x + a3.x), (a0.y + a1.y) + (a2.y + a3.y), (a0.z + a1.z) + (a2.z + a3.z),
                           (a0.w + a1.w) + (a2.w + a3.w));
    float4* out = reinterpret_cast<float4*>(dx);
    if (accumulate) {
      const float4 old = out[i];
      o.x += old.x, o.y += old.y, o.z += old.z, o.w += old.w;
    }
    out[i] = o;
  }
}

// ------------------------------------------------------------------ conv_in ----
// x fp32 NCHW [B,Cin,H,W] (Cin <= 8), w fp32 HWIO [3,3,Cin,Cout], y fp32 NHWC [B,H,W,Cout]
constexpr int CI_PIX = 32;
// A thread owns ONE channel quad and walks the CTA's pixels p = grp, grp + R, ... (R = 256 / (Cout / 4) thread groups), so the
// per-channel sums the consuming GroupNorm needs stay in registers: gn_stats (optional) = [slab, Cout, 2] (sum, sum of
// squares) of this CTA's 32 pixels -- exactly one statistics slab, as the igemm epilogues write it -- combined over the
// R groups in ascending order.
__global__ void __launch_bounds__(256) conv_in_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                      const float* __restrict__ bias, float* __restrict__ y, int B, int Cin,
                                                      int H, int W, int Cout, float* __restrict__ gn_stats) {
  __shared__ float patch[CI_PIX][9 * 8];
  __shared__ float part[2][1024];  // [sum | sumsq][grp * Cout + c], R * Cout <= 1024
  const int64_t pix0 = static_cast<int64_t>(blockIdx.x) * CI_PIX;
  const int HW = H * W;
  for (int i = threadIdx.x; i < CI_PIX * 9 * Cin; i += 256) {
    const int p = i / (9 * Cin), r = i % (9 * Cin);
    const int tap = r / Cin, ci = r % Cin;
    const int64_t pix = pix0 + p;
    float v = 0.f;
    if (pix < static_cast<int64_t>(B) * HW) {
      const int b = pix / HW, hw = pix % HW, h = hw / W, ww = hw % W;
      const int yy = h + tap / 3 - 1, xx = ww + tap % 3 - 1;
      if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = x[((static_cast<size_t>(b) * Cin + ci) * H + yy) * W + xx];
    }
    patch[p][r] = v;
  }
  __syncthreads();
  const int K = 9 * Cin;
  const int C4 = Cout >> 2;
  const int R = 256 / C4 < CI_PIX ? 256 / C4 : CI_PIX;   // thread groups (C4 <= 256 checked on the host)
  const int grp = threadIdx.x / C4, c = (threadIdx.x % C4) * 4;
  if (grp < R) {
    const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + c));
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f), ss = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int p = grp; p < CI_PIX; p += R) {
      const int64_t pix = pix0 + p;
      if (pix >= static_cast<int64_t>(B) * HW) break;
      float4 acc = b4;
      for (int k = 0; k < K; ++k) {
        const float a = patch[p][k];
        const float4 wv = __ldg(reinterpret_cast<const float4*>(w + static_cast<size_t>(k) * Cout + c));
        acc.x = fmaf(a, wv.x, acc.x), acc.y = fmaf(a, wv.y, acc.y), acc.z = fmaf(a, wv.z, acc.z),
        acc.w = fmaf(a, wv.w, acc.w);
      }
      *reinterpret_cast<float4*>(y + pix * Cout + c) = acc;
      s.x += acc.x, s.y += acc.y, s.z += acc.z, s.w += acc.w;
      ss.x += acc.x * acc.x, ss.y += acc.y * acc.y, ss.z += acc.z * acc.z, ss.w += acc.w * acc.w;
    }
    if (gn_stats != nullptr) {
      *reinterpret_cast<float4*>(&part[0][grp * Cout + c]) = s;
      *reinterpret_cast<float4*>(&part[1][grp * Cout + c]) = ss;
    }
  }
  if (gn_stats != nullptr) {
    __syncthreads();
    for (int ch = threadIdx.x; ch < Cout; ch += 256) {
      float s = 0.f, ss = 0.f;
      for (int g = 0; g < R; ++g) s += part[0][g * Cout + ch], ss += part[1][g * Cout + ch];
      *reinterpret_cast<float2*>(gn_stats + (static_cast<size_t>(blockIdx.x) * Cout + ch) * 2) = make_float2(s, ss);
    }
  }
}

// ----------------------------------------------------------------- conv_out ----
// x fp32 NHWC [B,H,W,Cin], w fp32 HWIO [3,3,Cin,Cout=4], y fp32 NCHW [B,4,H,W]; one warp per pixel
__global__ void __launch_bounds__(256) conv_out_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                       const float* __restrict__ bias, float* __restrict__ y, int B, int H,
                                                       int W, int Cin) {
  const int64_t pix = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int HW = H * W;
  if (pix >= static_cast<int64_t>(B) * HW) return;
  const int b = pix / HW, hw = pix % HW, h = hw / W, ww = hw % W;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  for (int tap = 0; tap < 9; ++tap) {
    const int yy = h + tap / 3 - 1, xx = ww + tap % 3 - 1;
    if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
    const float* xr = x + ((static_cast<size_t>(b) * H + yy) * W + xx) * Cin;
    const float* wr = w + static_cast<size_t>(tap) * Cin * 4;
    for (int c = lane; c < Cin; c += 32) {
      const float v = xr[c];
      const float4 wv = __ldg(reinterpret_cast<const float4*>(wr + c * 4));
      a0 = fmaf(v, wv.x, a0), a1 = fmaf(v, wv.y, a1), a2 = fmaf(v, wv.z, a2), a3 = fmaf(v, wv.w, a3);
    }
  }
  a0 = warp_sum(a0), a1 = warp_sum(a1), a2 = warp_sum(a2), a3 = warp_sum(a3);
  if (lane == 0) {
    float* yo = y + static_cast<size_t>(b) * 4 * HW + hw;
    yo[0] = a0 + bias[0], yo[HW] = a1 + bias[1], yo[2 * HW] = a2 + bias[2], yo[3 * HW] = a3 + bias[3];
  }
}

// -------------------------------------------------------- timestep embedding ----
// FlaxTimesteps (flip_sin_to_cos=True, freq_shift=0): [cos(t f_i) | sin(t f_i)], f_i = exp(-ln(1e4) i / half)
__global__ void timestep_sincos_kernel(const int32_t* __restrict__ t, int t_stride, float* __restrict__ out, int B,
                                       int dim) {
  const int half = dim >> 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * half) return;
  const int b = i / half, j = i % half;
  const float inc = 9.210340371976184f / static_cast<float>(half);  // ln(10000)/half
  const float f = expf(static_cast<float>(j) * -inc);
  const float a = static_cast<float>(t[b * t_stride]) * f;
  out[b * dim + j] = cosf(a);
  out[b * dim + half + j] = sinf(a);
}

// y[b, n] = act_out( sum_k act_in(x[b,k]) * w[k, n] + bias[n] ), fp32, w in Flax [in,out] layout.
// M = batch is tiny (<= 32): a CTA owns 32 output columns for ALL samples; lane -> column (coalesced
// 128-byte rows of w, each weight read exactly once), warp -> K slice, batch accumulators in registers,
// cross-warp reduction through shared memory in fixed order (deterministic).
constexpr int DS_MAXB = 32;
constexpr int DS_WARPS = 32;  // 1024 threads: warp -> K slice, lane -> output column
template <int BMAX>
__global__ void __launch_bounds__(DS_WARPS * 32) dense_small_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                                    const float* __restrict__ bias, float* __restrict__ y,
                                                                    int B, int K, int N, int silu_in, int silu_out) {
  extern __shared__ float sm[];  // xs[B][K] then red[DS_WARPS][B][32]
  float* xs = sm;
  float* red = sm + static_cast<size_t>(B) * K;
  for (int i = threadIdx.x; i < B * K; i += DS_WARPS * 32) {
    const float v = x[i];
    xs[i] = silu_in ? silu_f(v) : v;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * 32 + lane;
  float acc[BMAX];
#pragma unroll
  for (int b = 0; b < BMAX; ++b) acc[b] = 0.f;
  const int kper = (K + DS_WARPS - 1) / DS_WARPS;
  const int k0 = warp * kper, k1 = min(K, k0 + kper);
  if (n < N) {
    int k = k0;
    for (; k + 7 < k1; k += 8) {
      float wv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) wv[u] = w[static_cast<size_t>(k + u) * N + n];
#pragma unroll
      for (int u = 0; u < 8; ++u)
#pragma unroll
        for (int b = 0; b < BMAX; ++b)
          if (b < B) acc[b] = fmaf(xs[b * K + k + u], wv[u], acc[b]);
    }
    for (; k < k1; ++k) {
      const float wv = w[static_cast<size_t>(k) * N + n];
#pragma unroll
      for (int b = 0; b < BMAX; ++b)
        if (b < B) acc[b] = fmaf(xs[b * K + k], wv, acc[b]);
    }
  }
#pragma unroll
  for (int b = 0; b < BMAX; ++b)
    if (b < B) red[(warp * B + b) * 32 + lane] = acc[b];
  __syncthreads();
  for (int i = threadIdx.x; i < B * 32; i += DS_WARPS * 32) {
    const int b = i >> 5, l = i & 31;
    const int nn = blockIdx.x * 32 + l;
    if (nn >= N) continue;
    float r = bias ? bias[nn] : 0.f;
    for (int wq = 0; wq < DS_WARPS; ++wq) r += red[(wq * B + b) * 32 + l];
    y[static_cast<size_t>(b) * N + nn] = silu_out ? silu_f(r) : r;
  }
}

// Grouped form of dense_small for layers that share the input x (the 22 time-embedding projections of the ResNet
// blocks all read silu(temb)): ONE launch, CTA -> (layer, 32-column block) through a small table of offsets.  Per
// output the arithmetic (K split over warps, fixed-order cross-warp sum) is exactly dense_small_kernel's, so the
// results are bit-identical to the separate launches.
struct DsGroup {
  int64_t w_off, bias_off, y_off;  // in floats, relative to the params / output base pointers
  int32_t n, cta0;                 // output width, first CTA of the group
};
template <int BMAX>
__global__ void __launch_bounds__(DS_WARPS * 32) dense_small_grouped_kernel(const float* __restrict__ x,
                                                                            const float* __restrict__ params,
                                                                            float* __restrict__ ybase,
                                                                            const DsGroup* __restrict__ groups, int n_groups,
                                                                            int B, int B_total, int row0, int K) {
  extern __shared__ float sm[];  // xs[B][K] then red[DS_WARPS][B][32]
  float* xs = sm;
  float* red = sm + static_cast<size_t>(B) * K;
  int g = 0;
  while (g + 1 < n_groups && static_cast<int>(blockIdx.x) >= groups[g + 1].cta0) ++g;
  const DsGroup grp = groups[g];
  const int N = grp.n;
  const int cblock = static_cast<int>(blockIdx.x) - grp.cta0;
  const float* w = params + grp.w_off;
  const float* bias = params + grp.bias_off;
  float* y = ybase + grp.y_off + static_cast<size_t>(row0) * N;   // layer output is [B_total, N]
  (void)B_total;
  for (int i = threadIdx.x; i < B * K; i += DS_WARPS * 32) xs[i] = x[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = cblock * 32 + lane;
  float acc[BMAX];
#pragma unroll
  for (int b = 0; b < BMAX; ++b) acc[b] = 0.f;
  const int kper = (K + DS_WARPS - 1) / DS_WARPS;
  const int k0 = warp * kper, k1 = min(K, k0 + kper);
  if (n < N) {
    int k = k0;
    for (; k + 7 < k1; k += 8) {
      float wv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) wv[u] = w[static_cast<size_t>(k + u) * N + n];
#pragma unroll
      for (int u = 0; u < 8; ++u)
#pragma unroll
        for (int b = 0; b < BMAX; ++b)
          if (b < B) acc[b] = fmaf(xs[b * K + k + u], wv[u], acc[b]);
    }
    for (; k < k1; ++k) {
      const float wv = w[static_cast<size_t>(k) * N + n];
#pragma unroll
      for (int b = 0; b < BMAX; ++b)
        if (b < B) acc[b] = fmaf(xs[b * K + k], wv, acc[b]);
    }
  }
#pragma unroll
  for (int b = 0; b < BMAX; ++b)
    if (b < B) red[(warp * B + b) * 32 + lane] = acc[b];
  __syncthreads();
  for (int i = threadIdx.x; i < B * 32; i += DS_WARPS * 32) {
    const int b = i >> 5, l = i & 31;
    const int nn = cblock * 32 + l;
    if (nn >= N) continue;
    float r = bias[nn];
    for (int wq = 0; wq < DS_WARPS; ++wq) r += red[(wq * B + b) * 32 + l];
    y[static_cast<size_t>(b) * N + nn] = r;
  }
}

static inline int grid_for(int64_t n, int threads) {
  int64_t g = (n + threads - 1) / threads;
  const int64_t cap = 132 * 32;
  return static_cast<int>(g > cap ? cap : (g < 1 ? 1 : g));
}

}  // namespace ddpo

using namespace ddpo;

extern "C" int ddpo_prep_weight(const float* src, void* dst_bf16, int k, int n, int ldk, int row_offset,
                                int col_offset, int geglu_bn, void* stream) {
  DDPO_REQUIRE(src && dst_bf16 && k > 0 && n > 0 && ldk >= k, "prep_weight: bad arguments");
  dim3 grid((k + 31) / 32, (n + 31) / 32), block(32, 8);
  prep_transpose_kernel<<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(
      src, static_cast<__nv_bfloat16*>(dst_bf16), k, n, ldk, row_offset, col_offset, geglu_bn);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_prep_weight_dgrad(const float* src, void* dst_bf16, int taps, int k, int n, int ld_dst, int col_offset,
                                      void* stream) {
  DDPO_REQUIRE(src && dst_bf16 && taps > 0 && k > 0 && n > 0, "prep_weight_dgrad: bad arguments");
  if (ld_dst <= 0) ld_dst = taps * n;
  DDPO_REQUIRE(col_offset >= 0 && col_offset + taps * n <= ld_dst, "prep_weight_dgrad: columns [%d, %d) exceed the row pitch %d",
               col_offset, col_offset + taps * n, ld_dst);
  const int64_t total = static_cast<int64_t>(taps) * k * n;
  prep_dgrad_kernel<<<static_cast<int>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, static_cast<__nv_bfloat16*>(dst_bf16), taps, k, n, total, ld_dst, col_offset);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_permute_geglu_bias(const float* src, float* dst, int n, int bn, void* stream) {
  DDPO_REQUIRE(src && dst && n > 0 && bn > 0 && (n / 2) % (bn / 2) == 0, "permute_geglu_bias: bad arguments");
  permute_geglu_bias_kernel<<<(n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(src, dst, n, bn);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_cast_bf16(const float* x, void* y_bf16, int64_t n, void* stream) {
  DDPO_REQUIRE(x && y_bf16 && n > 0 && n % 4 == 0, "cast_bf16: n must be a positive multiple of 4");
  cast_bf16_kernel<<<grid_for(n / 4, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, static_cast<__nv_bfloat16*>(y_bf16), n / 4);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_upsample2x_bf16(const float* x, void* y_bf16, int batch, int h, int w, int c, void* stream) {
  DDPO_REQUIRE(x && y_bf16 && c % 4 == 0, "upsample2x: bad arguments");
  upsample2x_bf16_kernel<<<grid_for(static_cast<int64_t>(batch) * h * w * (c / 4), 256), 256, 0,
                           static_cast<cudaStream_t>(stream)>>>(x, static_cast<__nv_bfloat16*>(y_bf16), batch, h, w,
                                                                c / 4);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_upsample2x_bwd(const float* dy, float* dx, int batch, int h, int w, int c, int accumulate,
                                   void* stream) {
  DDPO_REQUIRE(dy && dx && c % 4 == 0, "upsample2x_bwd: bad arguments");
  upsample2x_bwd_kernel<<<grid_for(static_cast<int64_t>(batch) * h * w * (c / 4), 256), 256, 0,
                          static_cast<cudaStream_t>(stream)>>>(dy, dx, batch, h, w, c / 4, accumulate);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_conv_in(const float* x_nchw, const float* w_hwio, const float* bias, float* y_nhwc, int batch,
                            int cin, int h, int w, int cout, float* gn_stats, void* stream) {
  DDPO_REQUIRE(x_nchw && w_hwio && bias && y_nhwc && cin > 0 && cin <= 8 && cout % 4 == 0, "conv_in: bad arguments");
  const int64_t pix = static_cast<int64_t>(batch) * h * w;
  DDPO_REQUIRE(cout <= 1024, "conv_in: cout=%d (at most 1024 output channels)", cout);
  conv_in_kernel<<<static_cast<int>((pix + CI_PIX - 1) / CI_PIX), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x_nchw, w_hwio, bias, y_nhwc, batch, cin, h, w, cout, gn_stats);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_conv_out(const float* x_nhwc, const float* w_hwio, const float* bias, float* y_nchw, int batch,
                             int h, int w, int cin, int cout, void* stream) {
  DDPO_REQUIRE(x_nhwc && w_hwio && bias && y_nchw && cout == 4, "conv_out: cout must be 4");
  const int64_t pix = static_cast<int64_t>(batch) * h * w;
  conv_out_kernel<<<static_cast<int>((pix + 7) / 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x_nhwc, w_hwio, bias, y_nchw, batch, h, w, cin);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_timestep_sincos(const int32_t* t, int t_stride, float* out, int batch, int dim, void* stream) {
  DDPO_REQUIRE(t && out && dim % 2 == 0, "timestep_sincos: bad arguments");
  const int n = batch * dim / 2;
  timestep_sincos_kernel<<<(n + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(t, t_stride, out, batch, dim);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_dense_small_grouped(const float* x, const float* params_base, float* y_base, const void* groups_dev,
                                        int n_groups, int total_ctas, int batch, int k, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DDPO_REQUIRE(x && params_base && y_base && groups_dev && n_groups > 0 && total_ctas > 0 && batch > 0 && k > 0,
               "dense_small_grouped: bad arguments");
  static bool attr = false;
  if (!attr) {
    DDPO_CUDA_OK(cudaFuncSetAttribute(dense_small_grouped_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    DDPO_CUDA_OK(cudaFuncSetAttribute(dense_small_grouped_kernel<DS_MAXB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr = true;
  }
  int slab = (200 * 1024) / (4 * k + 4 * DS_WARPS * 32);  // same slab rule as ddpo_dense_small (batch invariance)
  if (slab > DS_MAXB) slab = DS_MAXB;
  DDPO_REQUIRE(slab >= 1, "dense_small_grouped: k=%d too large", k);
  const DsGroup* groups = static_cast<const DsGroup*>(groups_dev);
  for (int b0 = 0; b0 < batch; b0 += slab) {
    const int bb = batch - b0 < slab ? batch - b0 : slab;
    const size_t smem = (static_cast<size_t>(bb) * k + static_cast<size_t>(DS_WARPS) * bb * 32) * sizeof(float);
    const float* xb = x + static_cast<size_t>(b0) * k;
    if (bb <= 8)
      dense_small_grouped_kernel<8><<<total_ctas, DS_WARPS * 32, smem, stream>>>(xb, params_base, y_base, groups, n_groups,
                                                                               bb, batch, b0, k);
    else
      dense_small_grouped_kernel<DS_MAXB><<<total_ctas, DS_WARPS * 32, smem, stream>>>(xb, params_base, y_base, groups,
                                                                                     n_groups, bb, batch, b0, k);
    DDPO_LAUNCH_OK();
  }
  return DDPO_OK;
}

extern "C" int ddpo_dense_small(const float* x, const float* w, const float* bias, float* y, int batch, int k, int n,
                                int silu_in, int silu_out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DDPO_REQUIRE(x && w && y && k > 0 && n > 0 && batch > 0, "dense_small: bad arguments");
  // batches larger than 32 rows are processed in slabs of 32 (same per-row arithmetic -> batch invariant)
  static bool attr = false;
  if (!attr) {
    DDPO_CUDA_OK(cudaFuncSetAttribute(dense_small_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    DDPO_CUDA_OK(cudaFuncSetAttribute(dense_small_kernel<DS_MAXB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr = true;
  }
  int slab = (200 * 1024) / (4 * k + 4 * DS_WARPS * 32);  // rows whose inputs + partials fit in shared memory
  if (slab > DS_MAXB) slab = DS_MAXB;
  DDPO_REQUIRE(slab >= 1, "dense_small: k=%d too large", k);
  for (int b0 = 0; b0 < batch; b0 += slab) {
    const int bb = batch - b0 < slab ? batch - b0 : slab;
    const size_t smem = (static_cast<size_t>(bb) * k + static_cast<size_t>(DS_WARPS) * bb * 32) * sizeof(float);
    const float* xb = x + static_cast<size_t>(b0) * k;
    float* yb = y + static_cast<size_t>(b0) * n;
    if (bb <= 8)
      dense_small_kernel<8><<<(n + 31) / 32, DS_WARPS * 32, smem, stream>>>(xb, w, bias, yb, bb, k, n, silu_in, silu_out);
    else
      dense_small_kernel<DS_MAXB><<<(n + 31) / 32, DS_WARPS * 32, smem, stream>>>(xb, w, bias, yb, bb, k, n, silu_in,
                                                                                 silu_out);
    DDPO_LAUNCH_OK();
  }
  return DDPO_OK;
}
