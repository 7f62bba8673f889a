// Fused softmax attention (forward) on wgmma (sm_90a), head dim 64 -- self- and cross-attention of the
// Flax U-Net's BasicTransformerBlock (3P diffusers==0.12.1 attention_flax.py FlaxAttention:
// S = (Q K^T) * d^-0.5, P = softmax(S), O = P V; reached from the reference at
// pipeline_flax_stable_diffusion.py:219-224 / training/policy_gradient.py:87-102).
//
// The [B*h, N, N] score tensor XLA materialises never exists here.  One CTA owns a 128-query
// tile of one (sample, head), two consumer warpgroups of 64 query rows each; K/V stream through a
// 2-stage TMA ring in 128-key blocks (warp 8 is the producer):
//   S_j   = Q K_j^T          wgmma m64n128k16 (both operands K-major in shared memory) -> registers
//   P_j   = exp2((S_j - m) c)   in registers (a quad of threads holds a query row), bf16
//   O     = O * alpha + P_j V_j   wgmma m64n64k16 with A = P from registers, B = V MN-major
// normalised by the row sum at the end.  Keys past nk (TMA zero fill) and, with causal masking, keys
// after the query are masked; key blocks entirely after a causal tile are skipped.
// Fixed reduction order; no atomics.
#include "common.cuh"
#include "wgmma.cuh"

namespace ddpo {

constexpr int AT_THREADS = 288;  // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int AT_BQ = 128, AT_BKV = 128, AT_D = 64;
constexpr int AT_TILE = AT_BQ * AT_D * 2;  // 16 KB: a [128 x 64] bf16 SW128 tile
constexpr int AT_SMEM_Q = 0;
constexpr int AT_SMEM_KV = AT_TILE;                        // 2 stages x (K | V)
constexpr int AT_SMEM_BAR = AT_SMEM_KV + 2 * 2 * AT_TILE;
constexpr int AT_SMEM_TOTAL = AT_SMEM_BAR + 256 + 1024;    // + alignment slack

struct AttnArgs {
  CUtensorMap tmQ, tmK, tmV;
  __nv_bfloat16* out;
  float* lse;  // [B, heads, Nq] or null
  int nq, nk, heads, ldo;
  int causal;         // 1: query i attends keys j <= i (CLIP text encoder); 0: all keys
  float scale_log2e;  // d^-0.5 * log2(e)
  float scale;
};

__global__ void __launch_bounds__(AT_THREADS, 1) attention_fwd_kernel(const __grid_constant__ AttnArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + AT_SMEM_BAR);
  uint64_t* q_full = bars;        // 1
  uint64_t* kv_full = bars + 1;   // [2]
  uint64_t* kv_empty = bars + 3;  // [2] (one arrive per consumer warp)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * AT_BQ, head = blockIdx.y, b = blockIdx.z;
  const int k_end = p.causal ? min(p.nk, q0 + AT_BQ) : p.nk;
  const int nkb = (k_end + AT_BKV - 1) / AT_BKV;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      prefetch_tmap(&p.tmQ);
      prefetch_tmap(&p.tmK);
      prefetch_tmap(&p.tmV);
      mbar_expect_tx(q_full, AT_TILE);
      tma_load_4d(smem + AT_SMEM_Q, &p.tmQ, q_full, 0, head, q0, b);
      for (int j = 0; j < nkb; ++j) {
        const int st = j & 1;
        mbar_wait(&kv_empty[st], ((j >> 1) & 1) ^ 1);
        uint8_t* sK = smem + AT_SMEM_KV + st * 2 * AT_TILE;
        mbar_expect_tx(&kv_full[st], 2 * AT_TILE);
        tma_load_4d(sK, &p.tmK, &kv_full[st], 0, head, j * AT_BKV, b);
        tma_load_4d(sK + AT_TILE, &p.tmV, &kv_full[st], 0, head, j * AT_BKV, b);
      }
    }
    return;
  }

  // ------------------------------------------------------------ consumer warpgroups
  // accumulator fragments: thread holds query rows rq[0] = .. + lane / 4 and rq[1] = rq[0] + 8, columns 8 j + 2 (lane & 3) + {0, 1}
  const int wg = warp >> 2;
  const int t4 = lane & 3;
  int rq[2];
  rq[0] = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  rq[1] = rq[0] + 8;
  int k_lim[2];  // keys [0, k_lim) are visible to the row (causal: j <= i; key 0 is always visible)
#pragma unroll
  for (int h = 0; h < 2; ++h) k_lim[h] = p.causal ? min(p.nk, rq[h] + 1) : p.nk;
  const float c = p.scale_log2e;
  float o[AT_D / 2];
#pragma unroll
  for (int i = 0; i < AT_D / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const uint32_t q_addr = smem_u32(smem + AT_SMEM_Q) + wg * (64 * 128);
  mbar_wait(q_full, 0);
  for (int j = 0; j < nkb; ++j) {
    const int st = j & 1;
    mbar_wait(&kv_full[st], (j >> 1) & 1);
    const uint32_t k_addr = smem_u32(smem + AT_SMEM_KV + st * 2 * AT_TILE), v_addr = k_addr + AT_TILE;
    float s[AT_BKV / 2];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < AT_D / 16; ++k)
      Wgmma<AT_BKV>::ss<0, 0>(s, gmma_desc(q_addr + k * 32, 16, 1024), gmma_desc(k_addr + k * 32, 16, 1024), k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    const int kbase = j * AT_BKV;
    uint32_t pa[AT_BKV / 16][4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int valid = k_lim[h] - kbase;
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < AT_BKV / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (8 * jj + 2 * t4 + e < valid) mx = fmaxf(mx, s[4 * jj + 2 * h + e]);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx);
      const float alpha = ex2_mufu((m_run[h] - m_new) * c);
      const float mc = m_new * c;
      float l_blk = 0.f;
#pragma unroll
      for (int jj = 0; jj < AT_BKV / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * jj + 2 * t4 + e;
          const float pr = col < valid ? ex2_sel<DDPO_EXP_POLY_FWD>(col, s[4 * jj + 2 * h + e] * c - mc) : 0.f;
          s[4 * jj + 2 * h + e] = pr;
          l_blk += pr;
        }
      l_run[h] = l_run[h] * alpha + l_blk;  // this thread's partial row sum (the quad is summed at the end)
      m_run[h] = m_new;
#pragma unroll
      for (int jj = 0; jj < AT_D / 8; ++jj) o[4 * jj + 2 * h] *= alpha, o[4 * jj + 2 * h + 1] *= alpha;
    }
#pragma unroll
    for (int kk = 0; kk < AT_BKV / 16; ++kk) {
      pa[kk][0] = pack_bf16(s[8 * kk + 0], s[8 * kk + 1]);
      pa[kk][1] = pack_bf16(s[8 * kk + 2], s[8 * kk + 3]);
      pa[kk][2] = pack_bf16(s[8 * kk + 4], s[8 * kk + 5]);
      pa[kk][3] = pack_bf16(s[8 * kk + 6], s[8 * kk + 7]);
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < AT_BKV / 16; ++kk)  // B = V: MN-major, 16 keys = 16 rows of 128 B
      Wgmma<AT_D>::rs<1>(o, pa[kk], gmma_desc(v_addr + kk * 16 * 128, 8192, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[st]);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int row = rq[h];
    if (row < p.nq) {
      const float inv = 1.0f / l;
      __nv_bfloat16* out = p.out + (static_cast<size_t>(b) * p.nq + row) * p.ldo + head * AT_D + 2 * t4;
#pragma unroll
      for (int jj = 0; jj < AT_D / 8; ++jj)
        *reinterpret_cast<uint32_t*>(out + 8 * jj) = pack_bf16(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
      if (p.lse != nullptr && t4 == 0)
        p.lse[(static_cast<size_t>(b) * p.heads + head) * p.nq + row] = m_run[h] * p.scale + logf(l);
    }
  }
}

static int make_qkv_map(CUtensorMap* m, const void* base, int heads, int n, int batch, int ld) {
  uint64_t dims[4] = {(uint64_t)AT_D, (uint64_t)heads, (uint64_t)n, (uint64_t)batch};
  uint64_t strides[3] = {(uint64_t)AT_D * 2, (uint64_t)ld * 2, (uint64_t)ld * 2 * n};
  uint32_t box[4] = {(uint32_t)AT_D, 1, (uint32_t)AT_BQ, 1};
  uint32_t es[4] = {1, 1, 1, 1};
  return make_tensor_map(m, base, 2, 4, dims, strides, box, es, 1);
}

}  // namespace ddpo

using namespace ddpo;

extern "C" int ddpo_attention_fwd(const ddpo_attention_args* a, void* stream) {
  DDPO_REQUIRE(a && a->q && a->k && a->v && a->out, "attention_fwd: null pointer");
  DDPO_REQUIRE(a->head_dim == AT_D, "attention_fwd: head_dim must be 64 (got %d)", a->head_dim);
  DDPO_REQUIRE(a->nq > 0 && a->nk > 0 && a->heads > 0 && a->batch > 0, "attention_fwd: bad sizes");
  AttnArgs p;
  memset(&p, 0, sizeof(p));
  int rc;
  if ((rc = make_qkv_map(&p.tmQ, a->q, a->heads, a->nq, a->batch, a->ldq))) return rc;
  if ((rc = make_qkv_map(&p.tmK, a->k, a->heads, a->nk, a->batch, a->ldk))) return rc;
  if ((rc = make_qkv_map(&p.tmV, a->v, a->heads, a->nk, a->batch, a->ldv))) return rc;
  p.out = static_cast<__nv_bfloat16*>(a->out);
  p.lse = a->lse;
  p.nq = a->nq, p.nk = a->nk, p.heads = a->heads, p.ldo = a->ldo;
  p.causal = a->causal != 0;
  DDPO_REQUIRE(!p.causal || a->nq == a->nk, "attention_fwd: causal masking needs nq == nk");
  p.scale = 1.0f / sqrtf(static_cast<float>(AT_D));
  p.scale_log2e = p.scale * 1.4426950408889634f;
  static bool attr = false;
  if (!attr) {
    DDPO_CUDA_OK(cudaFuncSetAttribute(attention_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AT_SMEM_TOTAL));
    attr = true;
  }
  const int n_qtiles = (a->nq + AT_BQ - 1) / AT_BQ;
  dim3 grid(n_qtiles, a->heads, a->batch);
  attention_fwd_kernel<<<grid, AT_THREADS, AT_SMEM_TOTAL, static_cast<cudaStream_t>(stream)>>>(p);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}
