// Fused softmax attention (forward) on wgmma (sm_90a), head dims 40, 64, 80 and 160 -- self- and cross-attention of
// the Flax U-Net's BasicTransformerBlock (3P diffusers==0.12.1 attention_flax.py FlaxAttention:
// S = (Q K^T) * d^-0.5, P = softmax(S), O = P V; reached from the reference at
// pipeline_flax_stable_diffusion.py:219-224 / training/policy_gradient.py:87-102).  SD2 runs d = 64 at every level,
// SD1.x (8 heads) runs d = 40, 80 and 160.
//
// The [B*h, N, N] score tensor XLA materialises never exists here.  One CTA owns a 128-query tile of one
// (sample, head), two consumer warpgroups of 64 query rows each; K/V stream through a TMA ring of NST stages in 128-key
// blocks (warp 8 is the producer).  At d = 80 and 160 the blocks have 64 keys: the wider O accumulator leaves no
// registers for a 128-key score tile under the 168-register cap of a 288-thread CTA, and at d = 160 a 128-key ring
// would not fit in shared memory.
//   S_j   = Q K_j^T          wgmma m64nBKVk16 (both operands K-major in shared memory) -> registers
//   P_j   = exp2((S_j - m) c)   in registers (a quad of threads holds a query row), bf16
//   O     = O * alpha + P_j V_j   wgmma m64n64k16 per 64 columns, A = P from registers, B = V MN-major
// normalised by the row sum at the end.
// Keys past nk (TMA zero fill) and, with causal masking, keys after the query are masked; key blocks entirely after a
// causal tile are skipped.  Only a block that reaches past nk or the tile's first causal row runs the per-element mask:
// the blocks of 4096-, 1024- and 256-token self-attention are all full.
// The head dim is padded in shared memory to whole 64-column SW128 boxes (40 -> 64, 80 -> 128, 160 -> 192): each
// tensor map's innermost extent is the real d, so TMA zero-fills columns [d, 64 * ceil(d / 64)) and the next head's
// data never enters the tile.  The zero columns add nothing to Q K^T and give O columns that are not stored.  Padding
// costs only wgmma work; the softmax (MUFU / issue), which bounds the kernel, is counted per score.
// Fixed reduction order; no atomics.
#include <type_traits>

#include "common.cuh"
#include "wgmma.cuh"

namespace ddpo {

constexpr int AT_THREADS = 288;  // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int AT_BQ = 128;
constexpr int AT_CHUNK = 64;      // head-dim columns per SW128 box (128 B rows)

// Shared-memory plan of head dim D: Q | NST stages x (K | V), each operand as D_PAD / 64 column chunks of SW128 tiles.
template <int D>
struct AtPlan {
  static constexpr int NCH = (D + AT_CHUNK - 1) / AT_CHUNK;  // 64-column chunks (padded head dim / 64)
  static constexpr int BKV = NCH > 1 ? 64 : 128;             // keys per block (O takes 32 registers per chunk)
  static constexpr int Q_CHUNK = AT_BQ * AT_CHUNK * 2;       // 16 KB: a [128 x 64] bf16 SW128 tile
  static constexpr int KV_CHUNK = BKV * AT_CHUNK * 2;
  static constexpr int STAGE = 2 * NCH * KV_CHUNK;           // K chunks | V chunks
  static constexpr int SMEM_Q = 0;
  static constexpr int SMEM_KV = NCH * Q_CHUNK;
  static constexpr int FIT = (227 * 1024 - 1280 - SMEM_KV) / STAGE;
  static constexpr int NST = FIT < 4 ? FIT : 4;              // 4 stages; 3 at d = 160 (48 KB each)
  static constexpr int SMEM_BAR = SMEM_KV + NST * STAGE;
  static constexpr int SMEM_TOTAL = SMEM_BAR + 256 + 1024;  // + alignment slack
  static_assert(NST >= 2, "attention_fwd: shared memory plan has room for fewer than two K/V stages");
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

// Column col = 8 jj + 2 t4 + e of a score fragment takes the polynomial exponent when col % PERIOD == PERIOD - 1
// (PERIOD = DDPO_EXP_POLY_FWD).  For an even PERIOD that divides 8 this holds only for e = 1 and only on lanes with
// (2 t4 + 1) % PERIOD == PERIOD - 1, so the choice is a per-lane select instead of a divergent branch per element.
static_assert(DDPO_EXP_POLY_FWD == 0 || (DDPO_EXP_POLY_FWD % 2 == 0 && 8 % DDPO_EXP_POLY_FWD == 0),
              "attention_fwd: the polynomial period must be 0, 2, 4 or 8");

// Online softmax of one key block for the thread's two query rows: S -> P as the bf16 A fragments of the P V wgmma (each
// pair is packed as soon as it is computed, so the fp32 scores die early), returns the O rescale per row.
// MASK: keys past nk and, when causal, after the row (rows row0 and row0 + 8) are excluded (the tail block past nk, the
// causal diagonal); key 0 is always visible.
template <int BKV, bool MASK>
__device__ __forceinline__ void softmax_block(const float (&s)[BKV / 2], uint32_t (&pa)[BKV / 16][4], float (&m_run)[2],
                                              float (&l_run)[2], float (&alpha)[2], int row0, int nk, int causal,
                                              int kbase, int t4, bool poly_lane, float c) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int valid = (causal ? min(nk, row0 + 8 * h + 1) : nk) - kbase;
    float mx4[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};  // max is exact: any grouping gives the same value
#pragma unroll
    for (int jj = 0; jj < BKV / 8; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (!MASK || 8 * jj + 2 * t4 + e < valid) mx4[(jj & 1) * 2 + e] = fmaxf(mx4[(jj & 1) * 2 + e], s[4 * jj + 2 * h + e]);
    float mx = fmaxf(fmaxf(mx4[0], mx4[1]), fmaxf(mx4[2], mx4[3]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float m_new = fmaxf(m_run[h], mx);
    alpha[h] = ex2_mufu((m_run[h] - m_new) * c);
    const float mc = m_new * c;
    float l_blk = 0.f;
#pragma unroll
    for (int jj = 0; jj < BKV / 8; ++jj) {
      float pr[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float x = fmaf(s[4 * jj + 2 * h + e], c, -mc);
        pr[e] = ex2_mufu(x);
        if (DDPO_EXP_POLY_FWD > 0 && e == 1) {
          const float pp = ex2_poly(x);
          pr[e] = poly_lane ? pp : pr[e];
        }
        if (MASK && !(8 * jj + 2 * t4 + e < valid)) pr[e] = 0.f;
        l_blk += pr[e];
      }
      pa[jj / 2][2 * (jj & 1) + h] = pack_bf16(pr[0], pr[1]);  // A fragment: rows r, r + 8 x keys 8 jj + 2 t4 + {0, 1}
    }
    l_run[h] = fmaf(l_run[h], alpha[h], l_blk);  // this thread's partial row sum (the quad is summed at the end)
    m_run[h] = m_new;
  }
}

template <int D>
__global__ void __launch_bounds__(AT_THREADS, 1) attention_fwd_kernel(const __grid_constant__ AttnArgs p) {
  using P = AtPlan<D>;
  constexpr int NCH = P::NCH, BKV = P::BKV, NST = P::NST;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + P::SMEM_BAR);
  uint64_t* q_full = bars;              // 1
  uint64_t* kv_full = bars + 1;         // [NST]
  uint64_t* kv_empty = bars + 1 + NST;  // [NST] (one arrive per consumer warp)

  // the warp index through a shuffle: the compiler then treats it, and the role branch, as warp-uniform (no divergent
  // fallback paths around the softmax shuffles)
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * AT_BQ, head = blockIdx.y, b = blockIdx.z;
  const int k_end = p.causal ? min(p.nk, q0 + AT_BQ) : p.nk;
  const int nkb = (k_end + BKV - 1) / BKV;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < NST; ++i) {
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
        const int st = j % NST;
        mbar_wait(&kv_empty[st], ((j / NST) & 1) ^ 1);
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
  // accumulator fragments: thread holds query rows row0 = .. + lane / 4 and row0 + 8, columns 8 j + 2 (lane & 3) + {0, 1}
  const int wg = warp >> 2;
  const int t4 = lane & 3;
  const bool poly_lane = DDPO_EXP_POLY_FWD > 0 && (2 * t4 + 1) % (DDPO_EXP_POLY_FWD > 0 ? DDPO_EXP_POLY_FWD : 1) ==
                                                      DDPO_EXP_POLY_FWD - 1;
  const int row0 = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const float c = p.scale_log2e;
  float o[NCH][AT_CHUNK / 2];  // O columns 64 ch + ..
#pragma unroll
  for (int ch = 0; ch < NCH; ++ch)
#pragma unroll
    for (int i = 0; i < AT_CHUNK / 2; ++i) o[ch][i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const uint32_t q_addr = smem_u32(smem + P::SMEM_Q) + wg * (64 * 128);
  const uint32_t kv_base = smem_u32(smem + P::SMEM_KV);
  float s[BKV / 2];
  uint32_t pa[BKV / 16][4];

  auto issue_s = [&](int st) {
    const uint32_t k_addr = kv_base + st * P::STAGE;
#pragma unroll
    for (int k = 0; k < NCH * AT_CHUNK / 16; ++k)  // 16 head-dim columns per instruction, 4 per 128-byte chunk row
      Wgmma<BKV>::template ss<0, 0>(s, gmma_desc(q_addr + (k / 4) * P::Q_CHUNK + (k % 4) * 32, 16, 1024),
                                    gmma_desc(k_addr + (k / 4) * P::KV_CHUNK + (k % 4) * 32, 16, 1024), k != 0);
    wgmma_commit();
  };
  auto issue_pv = [&](int st) {
    const uint32_t v_addr = kv_base + st * P::STAGE + NCH * P::KV_CHUNK;
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk)  // B = V: MN-major, 16 keys = 16 rows of 128 B
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch)
        Wgmma<AT_CHUNK>::rs<1>(o[ch], pa[kk], gmma_desc(v_addr + ch * P::KV_CHUNK + kk * 16 * 128, 8192, 1024), 1u);
    wgmma_commit();
  };
  // One key block: S_j = Q K_j^T, its softmax into bf16 P_j fragments, O *= alpha, O += P_j V_j.
  auto step = [&](auto masked, int j) {
    const int st = j % NST;
    mbar_wait(&kv_full[st], (j / NST) & 1);
    wgmma_fence();
    issue_s(st);
    wgmma_wait<0>();
    reg_fence(s);
    float alpha[2];
    softmax_block<BKV, decltype(masked)::value>(s, pa, m_run, l_run, alpha, row0, p.nk, p.causal, j * BKV, t4,
                                                   poly_lane, c);
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch)
#pragma unroll
        for (int jj = 0; jj < AT_CHUNK / 8; ++jj) o[ch][4 * jj + 2 * h] *= alpha[h], o[ch][4 * jj + 2 * h + 1] *= alpha[h];
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) reg_fence(o[ch]);
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) reg_fence(pa[kk]);
    wgmma_fence();
    issue_pv(st);
    wgmma_wait<0>();
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) reg_fence(o[ch]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[st]);
  };

  // blocks [0, n_full) lie below nk and, when causal, end at or before the tile's first query row.  The bound is the
  // same for the whole CTA (not per warpgroup) so that the compiler sees uniform control flow around the wgmmas.
  const int full_lim = p.causal ? min(p.nk, q0 + 1) : p.nk;
  const int n_full = min(nkb, full_lim / BKV);
  mbar_wait(q_full, 0);
  for (int j = 0; j < n_full; ++j) step(std::false_type(), j);
  for (int j = n_full; j < nkb; ++j) step(std::true_type(), j);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int row = row0 + 8 * h;
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
