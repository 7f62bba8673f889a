// Memory-bound pieces of the U-Net backward pass (the hand-written counterpart of what
// `jax.grad(compute_loss)` -- reference ddpo/training/policy_gradient.py:138 -- derives for the
// non-GEMM layers of the 3P Flax U-Net): bias / per-sample column sums fused with the bf16 cast of
// the incoming gradient, GEGLU backward, conv_in / conv_out backward, the M=batch dense layers of
// the time embedding, zero-dilation for the stride-2 conv's data gradient, strided accumulate.
// All reductions are two-stage with fixed order (deterministic).
#include "common.cuh"
#include "reduce.cuh"

namespace ddpo {

// ------------------------------------------------------------ colsum + cast ----
// dy fp32 [M, N] -> optional bf16 copy; partial column sums per row chunk -> part[chunk][N].
// CTA tile = chunk_rows x 128 columns: lane -> float4 column group, warp -> rows w, w+8, ... (4 loads in flight),
// cross-warp reduction through shared memory in fixed order.
constexpr int CS_ROWS = 64;
__global__ void __launch_bounds__(256) colsum_cast_kernel(const float* __restrict__ dy, int ld, __nv_bfloat16* __restrict__ yb,
                                                          float* __restrict__ part, int M, int N, int chunk_rows) {
  __shared__ float4 red[8][32];
  const int chunk = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = (blockIdx.y * 32 + lane) * 4;
  const int r0 = chunk * chunk_rows, r1 = min(M, r0 + chunk_rows);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < N) {
    int r = r0 + warp;
    for (; r + 24 < r1; r += 32) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = *reinterpret_cast<const float4*>(dy + static_cast<size_t>(r + 8 * u) * ld + c);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        acc.x += v[u].x, acc.y += v[u].y, acc.z += v[u].z, acc.w += v[u].w;
        if (yb != nullptr)
          *reinterpret_cast<uint2*>(yb + static_cast<size_t>(r + 8 * u) * N + c) =
              make_uint2(pack_bf16(v[u].x, v[u].y), pack_bf16(v[u].z, v[u].w));
      }
    }
    for (; r < r1; r += 8) {
      const float4 v = *reinterpret_cast<const float4*>(dy + static_cast<size_t>(r) * ld + c);
      acc.x += v.x, acc.y += v.y, acc.z += v.z, acc.w += v.w;
      if (yb != nullptr)
        *reinterpret_cast<uint2*>(yb + static_cast<size_t>(r) * N + c) = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
    }
  }
  if (part == nullptr) return;
  red[warp][lane] = acc;
  __syncthreads();
  if (warp == 0 && c < N) {
    float4 s = red[0][lane];
#pragma unroll
    for (int w = 1; w < 8; ++w) s.x += red[w][lane].x, s.y += red[w][lane].y, s.z += red[w][lane].z, s.w += red[w][lane].w;
    *reinterpret_cast<float4*>(part + static_cast<size_t>(chunk) * N + c) = s;
  }
}
// same for a bf16 input (no copy): partial column sums of x_bf16 [M, N]
__global__ void __launch_bounds__(256) colsum_bf16_kernel(const __nv_bfloat16* __restrict__ x, int ld, float* __restrict__ part,
                                                          int M, int N, int chunk_rows) {
  const int chunk = blockIdx.x;
  const int r0 = chunk * chunk_rows, r1 = min(M, r0 + chunk_rows);
  for (int c = (blockIdx.y * 256 + threadIdx.x) * 2; c < N; c += gridDim.y * 512) {
    float s0 = 0.f, s1 = 0.f;
    for (int r = r0; r < r1; ++r) {
      const uint32_t v = *reinterpret_cast<const uint32_t*>(x + static_cast<size_t>(r) * ld + c);
      s0 += bf16_lo(v), s1 += bf16_hi(v);
    }
    part[static_cast<size_t>(chunk) * N + c] = s0;
    part[static_cast<size_t>(chunk) * N + c + 1] = s1;
  }
}
// second stage (out[g][n] (+)= sum over the chunks of group g, fixed order): reduce_rows_kernel, reduce.cuh

// ------------------------------------------------------------------- GEGLU ----
// pre: bf16 [M, N] tile-interleaved ([bn/2 lin | bn/2 gate] per bn columns, bias included)
// dff: fp32 [M, N/2] gradient w.r.t. lin*gelu(gate);  dpre: bf16 [M, N] in PLAIN order [lin(N/2) | gate(N/2)]
// dff: fp32, or bf16 when dff_bf16 (the bf16 output of the FF down-projection's dgrad GEMM)
__global__ void __launch_bounds__(256) geglu_bwd_kernel(const __nv_bfloat16* __restrict__ pre, const void* __restrict__ dff,
                                                        __nv_bfloat16* __restrict__ dpre, int64_t M, int N, int bn,
                                                        int dff_bf16) {
  // 8 output channels per thread: 16-byte loads of lin / gate, 2 x 16 bytes of dff, two 16-byte stores
  const int half = bn >> 1, hn = N >> 1, groups = hn >> 3;
  const int64_t total = M * groups;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / groups;
    const int j = static_cast<int>(i % groups) * 8;  // output channels j .. j+7 (never straddle a tile: half % 8 == 0)
    const int tile = j / half, pos = j % half;
    const __nv_bfloat16* pr = pre + r * N + tile * bn + pos;
    const uint4 lin8 = *reinterpret_cast<const uint4*>(pr);
    const uint4 gate8 = *reinterpret_cast<const uint4*>(pr + half);
    float dv[8];
    if (dff_bf16) {
      const uint4 d8 = *reinterpret_cast<const uint4*>(static_cast<const __nv_bfloat16*>(dff) + r * hn + j);
      dv[0] = bf16_lo(d8.x), dv[1] = bf16_hi(d8.x), dv[2] = bf16_lo(d8.y), dv[3] = bf16_hi(d8.y);
      dv[4] = bf16_lo(d8.z), dv[5] = bf16_hi(d8.z), dv[6] = bf16_lo(d8.w), dv[7] = bf16_hi(d8.w);
    } else {
      const float4 d0 = *reinterpret_cast<const float4*>(static_cast<const float*>(dff) + r * hn + j);
      const float4 d1 = *reinterpret_cast<const float4*>(static_cast<const float*>(dff) + r * hn + j + 4);
      dv[0] = d0.x, dv[1] = d0.y, dv[2] = d0.z, dv[3] = d0.w, dv[4] = d1.x, dv[5] = d1.y, dv[6] = d1.z, dv[7] = d1.w;
    }
    const uint32_t lw[4] = {lin8.x, lin8.y, lin8.z, lin8.w}, gw[4] = {gate8.x, gate8.y, gate8.z, gate8.w};
    uint32_t ol[4], og[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float l0 = bf16_lo(lw[q]), l1 = bf16_hi(lw[q]), g0 = bf16_lo(gw[q]), g1 = bf16_hi(gw[q]);
      const float e0 = dv[2 * q], e1 = dv[2 * q + 1];
      ol[q] = pack_bf16(e0 * gelu_tanh_f(g0), e1 * gelu_tanh_f(g1));
      og[q] = pack_bf16(e0 * l0 * gelu_tanh_grad_f(g0), e1 * l1 * gelu_tanh_grad_f(g1));
    }
    *reinterpret_cast<uint4*>(dpre + r * N + j) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
    *reinterpret_cast<uint4*>(dpre + r * N + hn + j) = make_uint4(og[0], og[1], og[2], og[3]);
  }
}

// ------------------------------------------------- conv_in / conv_out backward ----
// Both stem convolutions pair a 4-channel NCHW tensor `s` (latents / d_eps) with a C-channel NHWC tensor `g`
// (d conv_in output / conv_out input).  One kernel serves both: thread = channel c of `g`, a CTA walks a contiguous
// pixel range in chunks of STEM_PC pixels whose 9x4 `s` patches are staged in shared memory (zero outside the image):
//   patch[k = tap*4 + n] = s[b, n, y + sign*oy(tap), x + sign*ox(tap)]
//   wgrad:  acc[k] += g[p, c] * patch[k]          -> part[split][...]   (fixed order, reduced in split order)
//   dgrad:  dx[p, c] = sum_k patch[k] * w[k][c]   (conv_out only; w = [tap][C][4] held in 36 registers)
// conv_out (forward y[b,n,q] = bias[n] + sum_{tap,c} x[b,q+off,c] w[tap,c,n]): sign = -1, part index (tap*C + c)*4 + n.
// conv_in  (dw[tap,ci,co] += sum_p lat[b,ci,p+off] dx[p,co]):                 sign = +1, part index (tap*4 + ci)*C + co.
// `g` is read exactly once (coalesced); the old per-tap kernels re-read it 9-36 times.
constexpr int STEM_SPLITS = 256;
constexpr int STEM_PC = 32;
constexpr int COW_SPLITS = STEM_SPLITS, CIW_SPLITS = STEM_SPLITS;
template <bool CONV_OUT>
__global__ void __launch_bounds__(512) stem_bwd_kernel(const float* __restrict__ s, const float* __restrict__ g,
                                                        const float* __restrict__ w, float* __restrict__ dx,
                                                        float* __restrict__ part, int B, int H, int W, int C) {
  __shared__ __align__(16) float patch[STEM_PC][36];
  const int c = threadIdx.x;
  const bool c_ok = c < C;
  const int HW = H * W;
  const int64_t P = static_cast<int64_t>(B) * HW;
  int64_t per = (P + STEM_SPLITS - 1) / STEM_SPLITS;
  per = (per + STEM_PC - 1) / STEM_PC * STEM_PC;
  const int64_t p0 = blockIdx.x * per, p1 = min(P, p0 + per);
  constexpr int sign = CONV_OUT ? -1 : 1;
  float acc[36], wr[36];
#pragma unroll
  for (int k = 0; k < 36; ++k) acc[k] = 0.f, wr[k] = 0.f;
  if (CONV_OUT && c_ok) {
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const float4 wv = __ldg(reinterpret_cast<const float4*>(w + (static_cast<size_t>(tap) * C + c) * 4));
      wr[tap * 4] = wv.x, wr[tap * 4 + 1] = wv.y, wr[tap * 4 + 2] = wv.z, wr[tap * 4 + 3] = wv.w;
    }
  }
  for (int64_t pc = p0; pc < p1; pc += STEM_PC) {
    __syncthreads();
    for (int i = threadIdx.x; i < STEM_PC * 36; i += blockDim.x) {
      const int j = i / 36, k = i % 36, tap = k >> 2, n = k & 3;
      const int64_t p = pc + j;
      float v = 0.f;
      if (p < p1) {
        const int b = p / HW, hw = p % HW, y = hw / W + sign * (tap / 3 - 1), x = hw % W + sign * (tap % 3 - 1);
        if (y >= 0 && y < H && x >= 0 && x < W) v = s[((static_cast<size_t>(b) * 4 + n) * H + y) * W + x];
      }
      patch[j][k] = v;
    }
    __syncthreads();
    if (!c_ok) continue;
    const int np = static_cast<int>(min(static_cast<int64_t>(STEM_PC), p1 - pc));
#pragma unroll 1
    for (int j0 = 0; j0 < np; j0 += 8) {
      float gv[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) gv[j] = (j0 + j < np) ? g[(pc + j0 + j) * C + c] : 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4* pt = reinterpret_cast<const float4*>(patch[j0 + j]);
        float d = 0.f;
#pragma unroll
        for (int q = 0; q < 9; ++q) {
          const float4 pv = pt[q];
          acc[4 * q] += gv[j] * pv.x, acc[4 * q + 1] += gv[j] * pv.y, acc[4 * q + 2] += gv[j] * pv.z,
              acc[4 * q + 3] += gv[j] * pv.w;
          if (CONV_OUT) d += pv.x * wr[4 * q] + pv.y * wr[4 * q + 1] + pv.z * wr[4 * q + 2] + pv.w * wr[4 * q + 3];
        }
        if (CONV_OUT && j0 + j < np) dx[(pc + j0 + j) * C + c] = d;
      }
    }
  }
  if (!c_ok) return;
  float* o = part + static_cast<size_t>(blockIdx.x) * 36 * C;
#pragma unroll
  for (int k = 0; k < 36; ++k) {
    if (CONV_OUT) o[(static_cast<size_t>(k >> 2) * C + c) * 4 + (k & 3)] = acc[k];
    else o[static_cast<size_t>(k) * C + c] = acc[k];
  }
}
__global__ void stem_wgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ dw, int total) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  float s = 0.f;
  for (int q = 0; q < STEM_SPLITS; ++q) s += part[static_cast<size_t>(q) * total + i];
  dw[i] += s;
}
// dbias[n] += sum_{b,p} dy[b,n,p] ; one CTA per output channel, fixed-order block reduction
__global__ void __launch_bounds__(256) conv_out_dbias_kernel(const float* __restrict__ dy, float* __restrict__ dbias, int B,
                                                             int HW) {
  const int n = blockIdx.x;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) {
    const float* d = dy + (static_cast<size_t>(b) * 4 + n) * HW;
    for (int p = threadIdx.x; p < HW; p += 256) acc += d[p];
  }
  __shared__ float sm[8];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < 8; ++i) s += sm[i];
    dbias[n] += s;
  }
}

// ------------------------------------------------------------- dense (M = B) ----
// forward was y = act_out(x' @ w + b), x' = silu_in ? silu(x) : x.
// dpre[b,n] = dy[b,n] * (silu_out ? silu'(pre) : 1) with pre recomputed.
__global__ void dense_small_dpre_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                        const float* __restrict__ bias, const float* __restrict__ dy,
                                        float* __restrict__ dpre, int B, int K, int N, int silu_in, int silu_out) {
  extern __shared__ float xs[];
  const int b = blockIdx.y;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float v = x[static_cast<size_t>(b) * K + k];
    xs[k] = silu_in ? silu_f(v) : v;
  }
  __syncthreads();
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float d = dy[static_cast<size_t>(b) * N + n];
  if (silu_out) {
    float acc = bias ? bias[n] : 0.f;
    for (int k = 0; k < K; ++k) acc = fmaf(xs[k], w[static_cast<size_t>(k) * N + n], acc);
    const float s = sigmoid_f(acc);
    d *= s * (1.0f + acc * (1.0f - s));
  }
  dpre[static_cast<size_t>(b) * N + n] = d;
}
// dw[k,n] += sum_b x'[b,k] dpre[b,n] ; db[n] += sum_b dpre[b,n]
__global__ void dense_small_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dpre,
                                         float* __restrict__ dw, float* __restrict__ db, int B, int K, int N,
                                         int silu_in) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int k = blockIdx.y;
  if (n >= N) return;
  float acc = 0.f, accb = 0.f;
  for (int b = 0; b < B; ++b) {
    float xv = x[static_cast<size_t>(b) * K + k];
    if (silu_in) xv = silu_f(xv);
    const float d = dpre[static_cast<size_t>(b) * N + n];
    acc = fmaf(xv, d, acc);
    accb += d;
  }
  dw[static_cast<size_t>(k) * N + n] += acc;
  if (k == 0 && db != nullptr) db[n] += accb;
}
// dx[b,k] (+)= (silu_in ? silu'(x) : 1) * sum_n dpre[b,n] w[k,n] ; one warp per (b,k)
__global__ void dense_small_dgrad_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                         const float* __restrict__ dpre, float* __restrict__ dx, int B, int K, int N,
                                         int silu_in, int accumulate) {
  const int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  if (k >= K) return;
  float acc = 0.f;
  for (int n = lane; n < N; n += 32) acc = fmaf(dpre[static_cast<size_t>(b) * N + n], w[static_cast<size_t>(k) * N + n], acc);
  acc = warp_sum(acc);
  if (lane == 0) {
    if (silu_in) {
      const float v = x[static_cast<size_t>(b) * K + k];
      const float s = sigmoid_f(v);
      acc *= s * (1.0f + v * (1.0f - s));
    }
    float* o = dx + static_cast<size_t>(b) * K + k;
    *o = accumulate ? *o + acc : acc;
  }
}

// ----------------------------------------------------------------- misc ------
// zero-dilated bf16 copy: y[b,2h,2w,:] = x[b,h,w,:], zeros elsewhere
__global__ void dilate2x_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, int B, int H, int W, int C4) {
  const int64_t total = static_cast<int64_t>(B) * 4 * H * W * C4;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c4 = i % C4;
    int64_t p = i / C4;
    const int w2 = p % (2 * W);
    p /= 2 * W;
    const int h2 = p % (2 * H);
    const int b = p / (2 * H);
    uint2 o = make_uint2(0u, 0u);
    if (((h2 | w2) & 1) == 0) {
      const float4 v = reinterpret_cast<const float4*>(x)[((static_cast<size_t>(b) * H + (h2 >> 1)) * W + (w2 >> 1)) * C4 + c4];
      o.x = pack_bf16(v.x, v.y), o.y = pack_bf16(v.z, v.w);
    }
    reinterpret_cast<uint2*>(y)[i] = o;
  }
}
// dst[r, 0:cols] (+)= src[r, 0:cols]
__global__ void copy2d_kernel(const float* __restrict__ src, int lds, float* __restrict__ dst, int ldd, int64_t rows,
                              int cols4, int accumulate) {
  const int64_t total = rows * cols4;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / cols4;
    const int c = static_cast<int>(i % cols4) * 4;
    float4 v = *reinterpret_cast<const float4*>(src + r * lds + c);
    float4* d = reinterpret_cast<float4*>(dst + r * ldd + c);
    if (accumulate) {
      const float4 o = *d;
      v.x += o.x, v.y += o.y, v.z += o.z, v.w += o.w;
    }
    *d = v;
  }
}

// dst[r, :] = src[index[r], :]: the trajectory buffer's (sample, timestep) rows picked by the epoch's shuffles
// (reference pipeline/policy_gradient.py:385-404,415-423 does this with host advanced indexing + H2D per step)
__global__ void gather_rows_kernel(const float* __restrict__ src, const int64_t* __restrict__ index,
                                   float* __restrict__ dst, int rows, int64_t row4) {
  const int r = blockIdx.y;
  const float4* s = reinterpret_cast<const float4*>(src) + index[r] * row4;
  float4* d = reinterpret_cast<float4*>(dst) + static_cast<int64_t>(r) * row4;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < row4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    d[i] = s[i];
}

static inline int grid_for(int64_t n, int threads) {
  int64_t g = (n + threads - 1) / threads;
  const int64_t cap = 132 * 32;
  return static_cast<int>(g > cap ? cap : (g < 1 ? 1 : g));
}

}  // namespace ddpo

using namespace ddpo;

extern "C" int64_t ddpo_colsum_workspace_floats(int m, int n, int rows_per_group) {
  const int cr = rows_per_group < CS_ROWS ? rows_per_group : CS_ROWS;
  return static_cast<int64_t>((m + cr - 1) / cr) * n;
}

// out[g][n] (+)= sum of rows of group g (groups of rows_per_group consecutive rows; rows_per_group == m: one
// group = bias gradient); optional bf16 copy of dy.
extern "C" int ddpo_colsum_cast(const float* dy, int ld, void* y_bf16, float* out, int rows_per_group, int accumulate,
                                float* workspace, int m, int n, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DDPO_REQUIRE(dy && n % 2 == 0 && m > 0 && rows_per_group > 0, "colsum_cast: bad arguments");
  const int cr = rows_per_group < CS_ROWS ? rows_per_group : CS_ROWS;
  const int chunks = (m + cr - 1) / cr;
  int groups = 1, cpg = chunks;
  if (rows_per_group < m) {
    DDPO_REQUIRE(m % rows_per_group == 0 && rows_per_group % cr == 0, "colsum_cast: rows_per_group=%d does not tile m=%d",
                 rows_per_group, m);
    groups = m / rows_per_group;
    cpg = rows_per_group / cr;
  }
  DDPO_REQUIRE(out == nullptr || workspace != nullptr, "colsum_cast: workspace required");
  DDPO_REQUIRE(n % 4 == 0 && (ld <= 0 || ld % 4 == 0), "colsum_cast: n and ld must be multiples of 4");
  dim3 grid(chunks, (n + 127) / 128);
  colsum_cast_kernel<<<grid, 256, 0, stream>>>(dy, ld > 0 ? ld : n, static_cast<__nv_bfloat16*>(y_bf16),
                                              out ? workspace : nullptr, m, n, cr);
  DDPO_LAUNCH_OK();
  if (out != nullptr) {
    launch_reduce_rows(workspace, groups, cpg, n, n, out, nullptr, accumulate, stream);
    DDPO_LAUNCH_OK();
  }
  return DDPO_OK;
}

extern "C" int ddpo_colsum_bf16(const void* x_bf16, int ld, float* out, int accumulate, float* workspace, int m, int n,
                                void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DDPO_REQUIRE(x_bf16 && out && workspace && n % 2 == 0 && m > 0, "colsum_bf16: bad arguments");
  const int chunks = (m + CS_ROWS - 1) / CS_ROWS;
  dim3 grid(chunks, (n + 511) / 512);
  colsum_bf16_kernel<<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x_bf16), ld > 0 ? ld : n, workspace, m, n,
                                              CS_ROWS);
  DDPO_LAUNCH_OK();
  launch_reduce_rows(workspace, 1, chunks, n, n, out, nullptr, accumulate, stream);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_geglu_bwd(const void* pre_bf16, const void* dff, void* dpre_bf16, int64_t m, int n, int bn,
                              int dff_bf16, void* stream) {
  DDPO_REQUIRE(pre_bf16 && dff && dpre_bf16 && n % bn == 0 && bn % 16 == 0, "geglu_bwd: bad arguments");
  geglu_bwd_kernel<<<grid_for(m * (n / 16), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(pre_bf16), dff, static_cast<__nv_bfloat16*>(dpre_bf16), m, n, bn, dff_bf16);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int64_t ddpo_conv_out_bwd_workspace_floats(int cin) { return static_cast<int64_t>(COW_SPLITS) * 9 * cin * 4; }

extern "C" int ddpo_conv_out_bwd(const float* x_nhwc, const float* w_hwio, const float* dy_nchw, float* dx_nhwc,
                                 float* dw, float* dbias, float* workspace, int batch, int h, int w, int cin,
                                 void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DDPO_REQUIRE(x_nhwc && w_hwio && dy_nchw && dx_nhwc && dw && workspace && cin % 32 == 0 && cin <= 512,
               "conv_out_bwd: bad arguments");
  stem_bwd_kernel<true><<<STEM_SPLITS, cin, 0, stream>>>(dy_nchw, x_nhwc, w_hwio, dx_nhwc, workspace, batch, h, w, cin);
  DDPO_LAUNCH_OK();
  const int total = 9 * cin * 4;
  stem_wgrad_reduce_kernel<<<(total + 255) / 256, 256, 0, stream>>>(workspace, dw, total);
  DDPO_LAUNCH_OK();
  if (dbias != nullptr) {
    conv_out_dbias_kernel<<<4, 256, 0, stream>>>(dy_nchw, dbias, batch, h * w);
    DDPO_LAUNCH_OK();
  }
  return DDPO_OK;
}

extern "C" int64_t ddpo_conv_in_wgrad_workspace_floats(int cin, int cout) {
  return static_cast<int64_t>(CIW_SPLITS) * 9 * cin * cout;
}

extern "C" int ddpo_conv_in_wgrad(const float* lat_nchw, const float* dx_nhwc, float* dw, float* workspace, int batch,
                                  int cin, int h, int w, int cout, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DDPO_REQUIRE(lat_nchw && dx_nhwc && dw && workspace, "conv_in_wgrad: null pointer");
  DDPO_REQUIRE(cin == 4 && cout <= 512, "conv_in_wgrad: needs 4 latent channels and <= 512 output channels");
  stem_bwd_kernel<false><<<STEM_SPLITS, (cout + 31) / 32 * 32, 0, stream>>>(lat_nchw, dx_nhwc, nullptr, nullptr, workspace,
                                                                           batch, h, w, cout);
  DDPO_LAUNCH_OK();
  const int total = 9 * cin * cout;
  stem_wgrad_reduce_kernel<<<(total + 255) / 256, 256, 0, stream>>>(workspace, dw, total);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_dense_small_bwd(const float* x, const float* w, const float* bias, const float* dy, float* dpre_ws,
                                    float* dw, float* db, float* dx, int dx_accumulate, int batch, int k, int n,
                                    int silu_in, int silu_out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DDPO_REQUIRE(x && w && dy && dpre_ws && dw && k * 4 <= 48 * 1024, "dense_small_bwd: bad arguments");
  dim3 g1((n + 127) / 128, batch);
  dense_small_dpre_kernel<<<g1, 128, k * sizeof(float), stream>>>(x, w, bias, dy, dpre_ws, batch, k, n, silu_in, silu_out);
  DDPO_LAUNCH_OK();
  dim3 g2((n + 127) / 128, k);
  dense_small_wgrad_kernel<<<g2, 128, 0, stream>>>(x, dpre_ws, dw, db, batch, k, n, silu_in);
  DDPO_LAUNCH_OK();
  if (dx != nullptr) {
    dim3 g3((k + 7) / 8, batch);
    dense_small_dgrad_kernel<<<g3, 256, 0, stream>>>(x, w, dpre_ws, dx, batch, k, n, silu_in, dx_accumulate);
    DDPO_LAUNCH_OK();
  }
  return DDPO_OK;
}

extern "C" int ddpo_dilate2x_bf16(const float* x, void* y_bf16, int batch, int h, int w, int c, void* stream) {
  DDPO_REQUIRE(x && y_bf16 && c % 4 == 0, "dilate2x: bad arguments");
  dilate2x_bf16_kernel<<<grid_for(static_cast<int64_t>(batch) * 4 * h * w * (c / 4), 256), 256, 0,
                         static_cast<cudaStream_t>(stream)>>>(x, static_cast<__nv_bfloat16*>(y_bf16), batch, h, w, c / 4);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_gather_rows(const float* src, const int64_t* index_dev, float* dst, int rows, int64_t row_floats,
                                void* stream) {
  DDPO_REQUIRE(src && index_dev && dst && rows > 0 && rows <= 65535 && row_floats > 0 && row_floats % 4 == 0,
               "gather_rows: bad arguments (rows=%d row_floats=%lld)", rows, (long long)row_floats);
  const int64_t row4 = row_floats / 4;
  int gx = static_cast<int>((row4 + 255) / 256);
  if (gx > 64) gx = 64;
  gather_rows_kernel<<<dim3(gx, rows), 256, 0, static_cast<cudaStream_t>(stream)>>>(src, index_dev, dst, rows, row4);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int ddpo_copy2d(const float* src, int lds, float* dst, int ldd, int64_t rows, int cols, int accumulate,
                           void* stream) {
  DDPO_REQUIRE(src && dst && cols % 4 == 0 && lds % 4 == 0 && ldd % 4 == 0, "copy2d: bad arguments");
  copy2d_kernel<<<grid_for(rows * (cols / 4), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(src, lds, dst, ldd, rows,
                                                                                                cols / 4, accumulate);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}
