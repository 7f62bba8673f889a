// Fused softmax attention (forward) on wgmma (sm_90a), head dims 40, 64, 80 and 160 -- self- and cross-attention of
// the Flax U-Net's BasicTransformerBlock (3P diffusers==0.12.1 attention_flax.py FlaxAttention:
// S = (Q K^T) * d^-0.5, P = softmax(S), O = P V; reached from the reference at
// pipeline_flax_stable_diffusion.py:219-224 / training/policy_gradient.py:87-102).  SD2 runs d = 64 at every level,
// SD1.x (8 heads) runs d = 40, 80 and 160.
//
// The [B*h, N, N] score tensor XLA materialises never exists here.  One CTA owns a 128-query
// tile of one (sample, head), two consumer warpgroups of 64 query rows each; K/V stream through a
// 2-stage TMA ring in 128-key blocks (warp 8 is the producer).  At d = 80 and 160 the blocks have 64 keys: the wider O
// accumulator leaves no registers for a 128-key score tile under the 168-register cap of a 288-thread CTA, and at
// d = 160 two 128-key stages would not fit in shared memory.
//   S_j   = Q K_j^T          wgmma m64nBKVk16 (both operands K-major in shared memory) -> registers
//   P_j   = exp2((S_j - m) c)   in registers (a quad of threads holds a query row), bf16
//   O     = O * alpha + P_j V_j   wgmma m64n64k16 per 64 columns, A = P from registers, B = V MN-major
// normalised by the row sum at the end.  Keys past nk (TMA zero fill) and, with causal masking, keys
// after the query are masked; key blocks entirely after a causal tile are skipped.
// The head dim is padded in shared memory to whole 64-column SW128 boxes (40 -> 64, 80 -> 128, 160 -> 192): each
// tensor map's innermost extent is the real d, so TMA zero-fills columns [d, 64 * ceil(d / 64)) and the next head's
// data never enters the tile.  The zero columns add nothing to Q K^T and give O columns that are not stored.  Padding
// costs only wgmma work; the softmax (MUFU / issue), which bounds the kernel, is counted per score.
// Fixed reduction order; no atomics.
#include "common.cuh"
#include "wgmma.cuh"

namespace ddpo {

constexpr int AT_THREADS = 288;  // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int AT_BQ = 128;
constexpr int AT_CHUNK = 64;      // head-dim columns per SW128 box (128 B rows)

// Shared-memory plan of head dim D: Q | 2 stages x (K | V), each operand as D_PAD / 64 column chunks of SW128 tiles.
template <int D>
struct AtPlan {
  static constexpr int NCH = (D + AT_CHUNK - 1) / AT_CHUNK;  // 64-column chunks (padded head dim / 64)
  static constexpr int BKV = NCH > 1 ? 64 : 128;             // keys per block (O takes 32 registers per chunk)
  static constexpr int Q_CHUNK = AT_BQ * AT_CHUNK * 2;       // 16 KB: a [128 x 64] bf16 SW128 tile
  static constexpr int KV_CHUNK = BKV * AT_CHUNK * 2;
  static constexpr int STAGE = 2 * NCH * KV_CHUNK;           // K chunks | V chunks
  static constexpr int SMEM_Q = 0;
  static constexpr int SMEM_KV = NCH * Q_CHUNK;
  static constexpr int SMEM_BAR = SMEM_KV + 2 * STAGE;
  static constexpr int SMEM_TOTAL = SMEM_BAR + 256 + 1024;  // + alignment slack
  static_assert(SMEM_TOTAL <= 227 * 1024, "attention_fwd: shared memory plan exceeds 227 KB");
};

struct AttnArgs {
  CUtensorMap tmQ, tmK, tmV;
  __nv_bfloat16* out;
  float* lse;  // [B, heads, Nq] or null
  int nq, nk, heads, ldo;
  int causal;         // 1: query i attends keys j <= i (CLIP text encoder); 0: all keys
  float scale_log2e;  // d^-0.5 * log2(e)
  float scale;
};

template <int D>
__global__ void __launch_bounds__(AT_THREADS, 1) attention_fwd_kernel(const __grid_constant__ AttnArgs p) {
  using P = AtPlan<D>;
  constexpr int NCH = P::NCH, BKV = P::BKV;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + P::SMEM_BAR);
  uint64_t* q_full = bars;        // 1
  uint64_t* kv_full = bars + 1;   // [2]
  uint64_t* kv_empty = bars + 3;  // [2] (one arrive per consumer warp)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * AT_BQ, head = blockIdx.y, b = blockIdx.z;
  const int k_end = p.causal ? min(p.nk, q0 + AT_BQ) : p.nk;
  const int nkb = (k_end + BKV - 1) / BKV;

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
      mbar_expect_tx(q_full, NCH * P::Q_CHUNK);
#pragma unroll
      for (int c = 0; c < NCH; ++c)
        tma_load_4d(smem + P::SMEM_Q + c * P::Q_CHUNK, &p.tmQ, q_full, c * AT_CHUNK, head, q0, b);
      for (int j = 0; j < nkb; ++j) {
        const int st = j & 1;
        mbar_wait(&kv_empty[st], ((j >> 1) & 1) ^ 1);
        uint8_t* sK = smem + P::SMEM_KV + st * P::STAGE;
        mbar_expect_tx(&kv_full[st], P::STAGE);
#pragma unroll
        for (int c = 0; c < NCH; ++c)
          tma_load_4d(sK + c * P::KV_CHUNK, &p.tmK, &kv_full[st], c * AT_CHUNK, head, j * BKV, b);
#pragma unroll
        for (int c = 0; c < NCH; ++c)
          tma_load_4d(sK + (NCH + c) * P::KV_CHUNK, &p.tmV, &kv_full[st], c * AT_CHUNK, head, j * BKV, b);
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
  float o[NCH][AT_CHUNK / 2];  // O columns 64 ch + ..
#pragma unroll
  for (int ch = 0; ch < NCH; ++ch)
#pragma unroll
    for (int i = 0; i < AT_CHUNK / 2; ++i) o[ch][i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const uint32_t q_addr = smem_u32(smem + P::SMEM_Q) + wg * (64 * 128);
  mbar_wait(q_full, 0);
  for (int j = 0; j < nkb; ++j) {
    const int st = j & 1;
    mbar_wait(&kv_full[st], (j >> 1) & 1);
    const uint32_t k_addr = smem_u32(smem + P::SMEM_KV + st * P::STAGE), v_addr = k_addr + NCH * P::KV_CHUNK;
    float s[BKV / 2];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < NCH * AT_CHUNK / 16; ++k)  // 16 head-dim columns per instruction, 4 per 128-byte chunk row
      Wgmma<BKV>::template ss<0, 0>(s, gmma_desc(q_addr + (k / 4) * P::Q_CHUNK + (k % 4) * 32, 16, 1024),
                                    gmma_desc(k_addr + (k / 4) * P::KV_CHUNK + (k % 4) * 32, 16, 1024), k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    const int kbase = j * BKV;
    uint32_t pa[BKV / 16][4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int valid = k_lim[h] - kbase;
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < BKV / 8; ++jj)
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
      for (int jj = 0; jj < BKV / 8; ++jj)
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
      for (int ch = 0; ch < NCH; ++ch)
#pragma unroll
        for (int jj = 0; jj < AT_CHUNK / 8; ++jj) o[ch][4 * jj + 2 * h] *= alpha, o[ch][4 * jj + 2 * h + 1] *= alpha;
    }
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      pa[kk][0] = pack_bf16(s[8 * kk + 0], s[8 * kk + 1]);
      pa[kk][1] = pack_bf16(s[8 * kk + 2], s[8 * kk + 3]);
      pa[kk][2] = pack_bf16(s[8 * kk + 4], s[8 * kk + 5]);
      pa[kk][3] = pack_bf16(s[8 * kk + 6], s[8 * kk + 7]);
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk)  // B = V: MN-major, 16 keys = 16 rows of 128 B
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch)
        Wgmma<AT_CHUNK>::rs<1>(o[ch], pa[kk], gmma_desc(v_addr + ch * P::KV_CHUNK + kk * 16 * 128, 8192, 1024), 1u);
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
      __nv_bfloat16* out = p.out + (static_cast<size_t>(b) * p.nq + row) * p.ldo + head * D + 2 * t4;
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch)
#pragma unroll
        for (int jj = 0; jj < AT_CHUNK / 8; ++jj)  // only the D real columns of the head
          if (D % AT_CHUNK == 0 || ch * AT_CHUNK + 8 * jj + 2 * t4 < D)
            *reinterpret_cast<uint32_t*>(out + ch * AT_CHUNK + 8 * jj) =
                pack_bf16(o[ch][4 * jj + 2 * h] * inv, o[ch][4 * jj + 2 * h + 1] * inv);
      if (p.lse != nullptr && t4 == 0)
        p.lse[(static_cast<size_t>(b) * p.heads + head) * p.nq + row] = m_run[h] * p.scale + logf(l);
    }
  }
}

// [batch, n, ld] bf16 with head h at columns [h d, h d + d): boxes of 64 columns x box_rows rows; columns past d of a
// box are out of the tensor's innermost extent and arrive as zeros
static int make_qkv_map(CUtensorMap* m, const void* base, int d, int heads, int n, int batch, int ld, int box_rows) {
  uint64_t dims[4] = {(uint64_t)d, (uint64_t)heads, (uint64_t)n, (uint64_t)batch};
  uint64_t strides[3] = {(uint64_t)d * 2, (uint64_t)ld * 2, (uint64_t)ld * 2 * n};
  uint32_t box[4] = {(uint32_t)AT_CHUNK, 1, (uint32_t)box_rows, 1};
  uint32_t es[4] = {1, 1, 1, 1};
  return make_tensor_map(m, base, 2, 4, dims, strides, box, es, 1);
}

template <int D>
static int attention_fwd_launch(const ddpo_attention_args* a, cudaStream_t stream) {
  using P = AtPlan<D>;
  AttnArgs p;
  memset(&p, 0, sizeof(p));
  int rc;
  if ((rc = make_qkv_map(&p.tmQ, a->q, D, a->heads, a->nq, a->batch, a->ldq, AT_BQ))) return rc;
  if ((rc = make_qkv_map(&p.tmK, a->k, D, a->heads, a->nk, a->batch, a->ldk, P::BKV))) return rc;
  if ((rc = make_qkv_map(&p.tmV, a->v, D, a->heads, a->nk, a->batch, a->ldv, P::BKV))) return rc;
  p.out = static_cast<__nv_bfloat16*>(a->out);
  p.lse = a->lse;
  p.nq = a->nq, p.nk = a->nk, p.heads = a->heads, p.ldo = a->ldo;
  p.causal = a->causal != 0;
  p.scale = 1.0f / sqrtf(static_cast<float>(D));
  p.scale_log2e = p.scale * 1.4426950408889634f;
  static bool attr = false;
  if (!attr) {
    DDPO_CUDA_OK(cudaFuncSetAttribute(attention_fwd_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, P::SMEM_TOTAL));
    attr = true;
  }
  const int n_qtiles = (a->nq + AT_BQ - 1) / AT_BQ;
  dim3 grid(n_qtiles, a->heads, a->batch);
  attention_fwd_kernel<D><<<grid, AT_THREADS, P::SMEM_TOTAL, stream>>>(p);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

}  // namespace ddpo

using namespace ddpo;

extern "C" int ddpo_attention_fwd(const ddpo_attention_args* a, void* stream) {
  DDPO_REQUIRE(a && a->q && a->k && a->v && a->out, "attention_fwd: null pointer");
  const int d = a->head_dim;
  DDPO_REQUIRE(d == 40 || d == 64 || d == 80 || d == 160, "attention_fwd: head_dim must be 40, 64, 80 or 160 (got %d)", d);
  DDPO_REQUIRE(a->nq > 0 && a->nk > 0 && a->heads > 0 && a->batch > 0, "attention_fwd: bad sizes");
  DDPO_REQUIRE(attention_operands_ok(a->q, a->ldq, a->heads, d) && attention_operands_ok(a->k, a->ldk, a->heads, d) &&
                   attention_operands_ok(a->v, a->ldv, a->heads, d) && attention_operands_ok(a->out, a->ldo, a->heads, d),
               "attention_fwd: q/k/v/out need 16-byte aligned base pointers, pitches that are multiples of 8 elements "
               "and at least heads * head_dim");
  DDPO_REQUIRE(!a->causal || a->nq == a->nk, "attention_fwd: causal masking needs nq == nk");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (d) {
    case 40: return attention_fwd_launch<40>(a, s);
    case 80: return attention_fwd_launch<80>(a, s);
    case 160: return attention_fwd_launch<160>(a, s);
    default: return attention_fwd_launch<64>(a, s);
  }
}
