// Low-rank adapters (LoRA) on the attention projections, diffusers' LoRALinearLayer in the Flax layout:
//   y = x W + b + s (x D) U,   W [K, N], D [K, r] (= down.weight^T), U [r, N] (= up.weight^T).
//
// lora_merge: the adapted layer's bf16 GEMM operands bf16(W + s D U), in the forward [N, K] layout of
//   ddpo_prep_weight and / or the dgrad [K, N] layout of ddpo_prep_weight_dgrad (taps = 1), so that every
//   existing forward / backward kernel runs unchanged on the merged weights.  Per element the rank-r sum is formed
//   in fp32 (fma chain over j), s times it is added to W and the result is rounded to bf16 once: with U = 0 the
//   operands are bit-identical to prep_weight's, signed zeros included.  The fp32 value itself (the merged kernel a
//   checkpoint holds) can be written too.
//
// lora_grad: the adapter gradients of G <= 3 adapters that share the input x [M, K] (q/k/v of self-attention share
//   the LayerNorm output, k/v of cross-attention the text context):
//     dU_g += s (x D_g)^T dy_g        dD_g += s x^T (dy_g U_g^T)
//   One launch reads x and every dy_g once.  A cluster of NC CTAs owns a row tile of BM rows at a time; CTA q of the
//   cluster holds columns [q K/NC, (q+1) K/NC) of x and [q N/NC, (q+1) N/NC) of every dy_g in shared memory, forms its
//   partial products of x D and dy U^T over those columns, and the cluster adds the NC partials through distributed
//   shared memory in rank order, so that every CTA holds the full [BM, r] intermediates without them ever reaching
//   HBM.  Each CTA then accumulates its own columns of dD_g / dU_g in shared memory over the row tiles of its cluster.
//   The reduction over M is two-stage and fixed-order: one partial per cluster in the workspace, then a second kernel
//   sums the partials in cluster order and adds s times the sum into the gradient buffer.  No float atomics: two runs
//   are bit-identical.  Arithmetic is fp32 on the CUDA cores (the r-wide products have no tensor-core shape at r = 4).
#include <cooperative_groups.h>

#include <algorithm>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace ddpo {

constexpr int LORA_THREADS = 256;
constexpr int LORA_BM = 16;             // rows per tile
constexpr int LORA_MAX_G = 3;
constexpr int LORA_SMS = 132;           // H100 SXM
constexpr int LORA_SMEM_TWO_PER_SM = 110 * 1024;
constexpr int LORA_SMEM_MAX = 220 * 1024;

// ------------------------------------------------------------------------------------------------ merge ----
__global__ void lora_merge_kernel(const float* __restrict__ W, const float* __restrict__ D, const float* __restrict__ U,
                                  int K, int N, int R, float s, __nv_bfloat16* __restrict__ fwd, int ldk, int row_offset,
                                  __nv_bfloat16* __restrict__ dgrad, int ld_dst, int col_offset,
                                  float* __restrict__ merged) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.x * 32, n0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int k = k0 + i, n = n0 + threadIdx.x;
    float v = 0.f;
    if (k < K && n < N) {
      float acc = 0.f;
      for (int j = 0; j < R; ++j) acc = fmaf(D[static_cast<size_t>(k) * R + j], U[static_cast<size_t>(j) * N + n], acc);
      // a zero low-rank term leaves W as it is (W + 0 would turn a -0.0 kernel element into +0.0)
      const float w = W[static_cast<size_t>(k) * N + n], d = s * acc;
      v = d == 0.f ? w : w + d;
      if (dgrad != nullptr) dgrad[static_cast<size_t>(k) * ld_dst + col_offset + n] = __float2bfloat16_rn(v);
      if (merged != nullptr) merged[static_cast<size_t>(k) * N + n] = v;
    }
    tile[i][threadIdx.x] = v;
  }
  if (fwd == nullptr) return;
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int n = n0 + i, k = k0 + threadIdx.x;
    if (n < N && k < K)
      fwd[static_cast<size_t>(n + row_offset) * ldk + k] = __float2bfloat16_rn(tile[threadIdx.x][i]);
  }
}

// ------------------------------------------------------------------------------------------------- grad ----
struct LoraGradParams {
  const __nv_bfloat16* x;
  const __nv_bfloat16* dy[LORA_MAX_G];
  const float* D[LORA_MAX_G];
  const float* U[LORA_MAX_G];
  float* ws;              // [clusters][G][K*R + R*N] partials
  int ldx, lddy, M, K, N, G, NC;
};

struct LoraSmem {         // offsets in floats into the dynamic shared memory
  int Ds, Us, accD, accU, part, full, scratch, xs, dys, total_bytes;
};

template <int R>
__host__ __device__ inline LoraSmem lora_smem_layout(int Kc, int Nc, int G) {
  LoraSmem L;
  const int S = LORA_THREADS / (2 * G * LORA_BM);     // threads per intermediate row in the first phase
  int o = 0;
  L.Ds = o, o += G * Kc * R;                           // D_g[k0 + k][j]        at Ds[(g Kc + k) R + j]
  L.Us = o, o += G * Nc * R;                           // U_g[j][n0 + n]        at Us[(g Nc + n) R + j]
  L.accD = o, o += G * Kc * R;                         // sum over tiles of x^T (dy U^T)
  L.accU = o, o += G * Nc * R;                         // sum over tiles of dy^T (x D), [n][j]
  L.part = o, o += 2 * G * LORA_BM * R;                // this CTA's partial x D_g (type g) and dy_g U_g^T (type G + g)
  L.full = o, o += 2 * G * LORA_BM * R;                // the cluster's sums
  L.scratch = o, o += S * 2 * G * LORA_BM * R;
  L.xs = o, o += LORA_BM * Kc / 2;                     // bf16 tiles
  L.dys = o, o += G * LORA_BM * Nc / 2;
  L.total_bytes = o * 4;
  return L;
}

__device__ inline void load_tile_bf16(__nv_bfloat16* dst, const __nv_bfloat16* src, int ld, int m0, int M, int cols) {
  const int vec = cols / 8;
  for (int e = threadIdx.x; e < LORA_BM * vec; e += LORA_THREADS) {
    const int i = e / vec, v = e % vec;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (m0 + i < M) val = *reinterpret_cast<const uint4*>(src + static_cast<size_t>(m0 + i) * ld + v * 8);
    *reinterpret_cast<uint4*>(dst + i * cols + v * 8) = val;
  }
}

template <int R>
__global__ void __launch_bounds__(LORA_THREADS) lora_grad_kernel(const LoraGradParams p) {
  extern __shared__ __align__(16) float sm[];
  cg::cluster_group cluster = cg::this_cluster();
  const int NC = p.NC, G = p.G;
  const int q = static_cast<int>(blockIdx.x) % NC;           // rank in the cluster (clusters run along x)
  const int cid = static_cast<int>(blockIdx.x) / NC;
  const int n_clusters = static_cast<int>(gridDim.x) / NC;
  const int Kc = p.K / NC, Nc = p.N / NC, k0 = q * Kc, n0 = q * Nc;
  const LoraSmem L = lora_smem_layout<R>(Kc, Nc, G);
  float* Ds = sm + L.Ds;
  float* Us = sm + L.Us;
  float* accD = sm + L.accD;
  float* accU = sm + L.accU;
  float* part = sm + L.part;
  float* full = sm + L.full;
  float* scratch = sm + L.scratch;
  __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(sm + L.xs);
  __nv_bfloat16* dys = reinterpret_cast<__nv_bfloat16*>(sm + L.dys);
  const int tid = threadIdx.x;

  for (int e = tid; e < G * Kc * R; e += LORA_THREADS) {
    const int g = e / (Kc * R), r = e % (Kc * R);
    Ds[e] = p.D[g][static_cast<size_t>(k0) * R + r];
    accD[e] = 0.f;
  }
  for (int e = tid; e < G * Nc * R; e += LORA_THREADS) {
    const int g = e / (Nc * R), n = (e % (Nc * R)) / R, j = e % R;
    Us[e] = p.U[g][static_cast<size_t>(j) * p.N + n0 + n];
    accU[e] = 0.f;
  }

  const int units = 2 * G * LORA_BM;                          // intermediate rows: (type, i)
  const int S = LORA_THREADS / units;
  const int tiles = (p.M + LORA_BM - 1) / LORA_BM;
  for (int t = cid; t < tiles; t += n_clusters) {
    const int m0 = t * LORA_BM;
    __syncthreads();                                          // previous tile's readers of xs / dys are done
    load_tile_bf16(xs, p.x + k0, p.ldx, m0, p.M, Kc);
    for (int g = 0; g < G; ++g) load_tile_bf16(dys + g * LORA_BM * Nc, p.dy[g] + n0, p.lddy, m0, p.M, Nc);
    __syncthreads();
    // phase 1: partial x D_g over this CTA's x columns, partial dy_g U_g^T over its dy columns (S threads per row,
    // strided over the columns, combined in a fixed order below)
    {
      const int u = tid / S, s = tid % S;
      if (u < units) {
        const int type = u / LORA_BM, i = u % LORA_BM;
        const bool is_x = type < G;
        const int g = is_x ? type : type - G;
        const int len = is_x ? Kc : Nc;
        const __nv_bfloat16* row = is_x ? xs + i * Kc : dys + (g * LORA_BM + i) * Nc;
        const float* w = is_x ? Ds + g * Kc * R : Us + g * Nc * R;
        float acc[R];
#pragma unroll
        for (int j = 0; j < R; ++j) acc[j] = 0.f;
        for (int c = s; c < len; c += S) {
          const float xv = __bfloat162float(row[c]);
          const float4* w4 = reinterpret_cast<const float4*>(w + c * R);
#pragma unroll
          for (int j4 = 0; j4 < R / 4; ++j4) {
            const float4 v = w4[j4];
            acc[4 * j4 + 0] = fmaf(xv, v.x, acc[4 * j4 + 0]);
            acc[4 * j4 + 1] = fmaf(xv, v.y, acc[4 * j4 + 1]);
            acc[4 * j4 + 2] = fmaf(xv, v.z, acc[4 * j4 + 2]);
            acc[4 * j4 + 3] = fmaf(xv, v.w, acc[4 * j4 + 3]);
          }
        }
#pragma unroll
        for (int j = 0; j < R; ++j) scratch[(s * units + u) * R + j] = acc[j];
      }
    }
    __syncthreads();
    for (int e = tid; e < units * R; e += LORA_THREADS) {
      float v = 0.f;
      for (int s = 0; s < S; ++s) v += scratch[s * units * R + e];
      part[e] = v;
    }
    // the cluster's sum of the NC partials, in rank order (identical in every CTA of the cluster)
    if (NC > 1) {
      cluster.sync();
      for (int e = tid; e < units * R; e += LORA_THREADS) {
        float v = 0.f;
        for (int r = 0; r < NC; ++r) v += cluster.map_shared_rank(part, r)[e];
        full[e] = v;
      }
      cluster.sync();                                         // peers may overwrite `part` from here on
    } else {
      __syncthreads();
      for (int e = tid; e < units * R; e += LORA_THREADS) full[e] = part[e];
      __syncthreads();
    }
    // phase 2: dD_g[k] += sum_i x[i][k] (dy_g U_g^T)[i] for this CTA's x columns, dU_g[:, n] += sum_i dy_g[i][n] (x D_g)[i]
    for (int col = tid; col < G * Kc + G * Nc; col += LORA_THREADS) {
      const bool is_x = col < G * Kc;
      const int g = is_x ? col / Kc : (col - G * Kc) / Nc;
      const int c = is_x ? col % Kc : (col - G * Kc) % Nc;
      const float* inter = full + (is_x ? (G + g) : g) * LORA_BM * R;
      float acc[R];
#pragma unroll
      for (int j = 0; j < R; ++j) acc[j] = 0.f;
#pragma unroll 4
      for (int i = 0; i < LORA_BM; ++i) {
        const float v = __bfloat162float(is_x ? xs[i * Kc + c] : dys[(g * LORA_BM + i) * Nc + c]);
        const float4* b4 = reinterpret_cast<const float4*>(inter + i * R);
#pragma unroll
        for (int j4 = 0; j4 < R / 4; ++j4) {
          const float4 b = b4[j4];
          acc[4 * j4 + 0] = fmaf(v, b.x, acc[4 * j4 + 0]);
          acc[4 * j4 + 1] = fmaf(v, b.y, acc[4 * j4 + 1]);
          acc[4 * j4 + 2] = fmaf(v, b.z, acc[4 * j4 + 2]);
          acc[4 * j4 + 3] = fmaf(v, b.w, acc[4 * j4 + 3]);
        }
      }
      float* dst = is_x ? accD + (g * Kc + c) * R : accU + (g * Nc + c) * R;
#pragma unroll
      for (int j = 0; j < R; ++j) dst[j] += acc[j];
    }
  }
  __syncthreads();
  // this cluster's partial: ws[cid][g] = [dD_g (K x R) | dU_g (R x N)], each CTA writing its own columns
  const size_t per_g = static_cast<size_t>(p.K) * R + static_cast<size_t>(R) * p.N;
  float* out = p.ws + static_cast<size_t>(cid) * G * per_g;
  for (int e = tid; e < G * Kc * R; e += LORA_THREADS) {
    const int g = e / (Kc * R), r = e % (Kc * R);
    out[g * per_g + static_cast<size_t>(k0) * R + r] = accD[e];
  }
  for (int e = tid; e < G * Nc * R; e += LORA_THREADS) {
    const int g = e / (Nc * R), j = (e % (Nc * R)) / Nc, n = e % Nc;
    out[g * per_g + static_cast<size_t>(p.K) * R + static_cast<size_t>(j) * p.N + n0 + n] = accU[(g * Nc + n) * R + j];
  }
  if (NC > 1) cluster.sync();                                 // no CTA leaves while a peer may still read its `part`
}

struct LoraOut {
  float* dD[LORA_MAX_G];
  float* dU[LORA_MAX_G];
};

// out += s * sum over clusters of the partials, in cluster order
__global__ void lora_grad_reduce_kernel(const float* __restrict__ ws, int n_clusters, int G, int K, int N, int R, float s,
                                        const LoraOut o) {
  const int64_t per_g = static_cast<int64_t>(K) * R + static_cast<int64_t>(R) * N;
  const int64_t total = G * per_g;
  for (int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float v = 0.f;
    for (int c = 0; c < n_clusters; ++c) v += ws[c * total + e];
    const int g = static_cast<int>(e / per_g);
    const int64_t r = e % per_g;
    float* dst = r < static_cast<int64_t>(K) * R ? o.dD[g] + r : o.dU[g] + (r - static_cast<int64_t>(K) * R);
    *dst += s * v;
  }
}

struct LoraPlan {
  int NC, clusters, smem_bytes;
};

template <int R>
static LoraPlan lora_plan_r(int G, int M, int K, int N) {
  LoraPlan pl{0, 0, 0};
  for (int two = 1; two >= 0 && pl.NC == 0; --two)
    for (int nc = 1; nc <= 8; nc *= 2) {
      if (K % (8 * nc) != 0 || N % (8 * nc) != 0) continue;
      const int bytes = lora_smem_layout<R>(K / nc, N / nc, G).total_bytes;
      if (bytes <= (two ? LORA_SMEM_TWO_PER_SM : LORA_SMEM_MAX)) {
        pl.NC = nc, pl.smem_bytes = bytes;
        const int per_sm = two ? 2 : 1;
        const int tiles = (M + LORA_BM - 1) / LORA_BM;
        pl.clusters = std::max(1, std::min(tiles, LORA_SMS * per_sm / nc));
        break;
      }
    }
  return pl;
}

static LoraPlan lora_plan(int rank, int G, int M, int K, int N) {
  switch (rank) {
    case 4: return lora_plan_r<4>(G, M, K, N);
    case 8: return lora_plan_r<8>(G, M, K, N);
    case 16: return lora_plan_r<16>(G, M, K, N);
    default: return LoraPlan{0, 0, 0};
  }
}

template <int R>
static int launch_lora_grad(const LoraGradParams& p, const LoraPlan& pl, cudaStream_t stream) {
  DDPO_CUDA_OK(cudaFuncSetAttribute(lora_grad_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, pl.smem_bytes));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(pl.NC * pl.clusters, 1, 1);
  cfg.blockDim = dim3(LORA_THREADS, 1, 1);
  cfg.dynamicSmemBytes = pl.smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = pl.NC;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  DDPO_CUDA_OK(cudaLaunchKernelEx(&cfg, lora_grad_kernel<R>, p));
  return DDPO_OK;
}

}  // namespace ddpo

using namespace ddpo;

extern "C" int ddpo_lora_merge(const float* w, int k, int n, const float* down, const float* up, int rank, float scale,
                               void* fwd_bf16, int ldk, int row_offset, void* dgrad_bf16, int ld_dst, int col_offset,
                               float* merged_f32, void* stream) {
  DDPO_REQUIRE(w && down && up && k > 0 && n > 0 && rank > 0 && (fwd_bf16 || dgrad_bf16 || merged_f32),
               "lora_merge: bad arguments");
  if (ldk <= 0) ldk = k;
  if (ld_dst <= 0) ld_dst = n;
  DDPO_REQUIRE(ldk >= k && row_offset >= 0 && col_offset >= 0 && col_offset + n <= ld_dst,
               "lora_merge: bad pitch / offsets (ldk %d, k %d, ld_dst %d, col_offset %d, n %d)", ldk, k, ld_dst,
               col_offset, n);
  dim3 grid((k + 31) / 32, (n + 31) / 32), block(32, 8);
  lora_merge_kernel<<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(
      w, down, up, k, n, rank, scale, static_cast<__nv_bfloat16*>(fwd_bf16), ldk, row_offset,
      static_cast<__nv_bfloat16*>(dgrad_bf16), ld_dst, col_offset, merged_f32);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int64_t ddpo_lora_grad_workspace_floats(int rank, int g, int m, int k, int n) {
  const LoraPlan pl = lora_plan(rank, g, m, k, n);
  if (pl.NC == 0) return -1;
  return static_cast<int64_t>(pl.clusters) * g * (static_cast<int64_t>(k) * rank + static_cast<int64_t>(rank) * n);
}

extern "C" int ddpo_lora_grad(const void* x, int ldx, const void* const* dy, int lddy, const float* const* down,
                              const float* const* up, float* const* d_down, float* const* d_up, int g, int m, int k,
                              int n, int rank, float scale, float* workspace, int64_t workspace_floats, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DDPO_REQUIRE(rank == 4 || rank == 8 || rank == 16, "lora_grad: rank %d (must be 4, 8 or 16)", rank);
  DDPO_REQUIRE(x && dy && down && up && d_down && d_up && workspace && g >= 1 && g <= LORA_MAX_G && m > 0 && k > 0 &&
                   n > 0, "lora_grad: bad arguments");
  DDPO_REQUIRE(ldx >= k && lddy >= n && ldx % 8 == 0 && lddy % 8 == 0 &&
                   reinterpret_cast<uintptr_t>(x) % 16 == 0, "lora_grad: x / dy rows must be 16-byte aligned");
  const LoraPlan pl = lora_plan(rank, g, m, k, n);
  DDPO_REQUIRE(pl.NC > 0, "lora_grad: no tiling for k %d, n %d, %d adapters at rank %d", k, n, g, rank);
  const int64_t need = static_cast<int64_t>(pl.clusters) * g * (static_cast<int64_t>(k) * rank + static_cast<int64_t>(rank) * n);
  DDPO_REQUIRE(workspace_floats >= need, "lora_grad: workspace of %lld floats, need %lld", (long long)workspace_floats,
               (long long)need);
  LoraGradParams p;
  LoraOut o;
  p.x = static_cast<const __nv_bfloat16*>(x);
  for (int i = 0; i < LORA_MAX_G; ++i) {
    const int s = i < g ? i : 0;
    DDPO_REQUIRE(dy[s] && down[s] && up[s] && d_down[s] && d_up[s] && reinterpret_cast<uintptr_t>(dy[s]) % 16 == 0,
                 "lora_grad: adapter %d: missing or misaligned operand", s);
    p.dy[i] = static_cast<const __nv_bfloat16*>(dy[s]);
    p.D[i] = down[s], p.U[i] = up[s];
    o.dD[i] = d_down[s], o.dU[i] = d_up[s];
  }
  p.ws = workspace, p.ldx = ldx, p.lddy = lddy, p.M = m, p.K = k, p.N = n, p.G = g, p.NC = pl.NC;
  int st = DDPO_OK;
  switch (rank) {
    case 4: st = launch_lora_grad<4>(p, pl, stream); break;
    case 8: st = launch_lora_grad<8>(p, pl, stream); break;
    default: st = launch_lora_grad<16>(p, pl, stream); break;
  }
  if (st != DDPO_OK) return st;
  const int64_t total = static_cast<int64_t>(g) * (static_cast<int64_t>(k) * rank + static_cast<int64_t>(rank) * n);
  const int blocks = static_cast<int>(std::min<int64_t>((total + 255) / 256, LORA_SMS * 8));
  lora_grad_reduce_kernel<<<blocks, 256, 0, stream>>>(workspace, pl.clusters, g, k, n, rank, scale, o);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}
