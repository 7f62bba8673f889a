// Attention backward on wgmma (sm_90a, head dims 40, 64, 80 and 160): the hand-written counterpart of what
// `jax.grad(compute_loss)` (reference ddpo/training/policy_gradient.py:138) derives for
// FlaxAttention (3P diffusers attention_flax.py):  P = softmax(Q K^T / sqrt(d)), O = P V.
//
//   delta_i = rowsum(dO_i * O_i)
//   dP = dO V^T ; dS = P * (dP - delta) / sqrt(d)
//   dV = P^T dO ; dK = dS^T Q ; dQ = dS K
//
// Two deterministic kernels (no atomics): `dkdv` owns a 128-key block and streams 64-query
// blocks, accumulating dK/dV in registers; `dq` owns a 128-query block and streams 64-key blocks,
// accumulating dQ in registers.  P is recomputed from the saved log-sum-exp (never stored).
// Each kernel has two consumer warpgroups (64 rows each) and a TMA producer warp (warp 8).  The
// score-shaped tiles (S^T / dP^T in dkdv, S / dP in dq) are wgmma accumulators; P and dS go from
// those registers straight into the A operand of the next wgmma (P^T dO, dS^T Q, dS K), whose B
// operand is the streamed tile read MN-major.
//
// Head dims other than 64 are padded in shared memory to whole 64-column SW128 boxes (40 -> 64, 80 -> 128,
// 160 -> 192) by TMA zero fill, as in the forward (attention.cu); only the d real columns are stored.  A 288-thread
// CTA has at most 168 registers per thread: enough for one 64-column chunk of dK and dV (or of dQ) next to the two
// score-shaped tiles, not for more.  So a CTA of either kernel owns one 64-column chunk of its outputs, and the CTAs of
// the other chunks of the same key (query) block recompute the score tiles over the whole padded head dim.  At d = 64
// and 40 there is one chunk and nothing is recomputed.
#include "common.cuh"
#include "wgmma.cuh"

namespace ddpo {

constexpr int AB_THREADS = 288;      // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int AB_T = 128 * 64 * 2;   // one [128 x 64] bf16 tile
constexpr int AB_H = 64 * 64 * 2;    // one [64 x 64] bf16 tile
constexpr int AB_CHUNK = 64;         // head-dim columns per SW128 tile

// Shared-memory plans of head dim D: every operand is NCH column chunks of [rows x 64] SW128 tiles.
template <int D>
struct AbPlan {
  static constexpr int NCH = (D + AB_CHUNK - 1) / AB_CHUNK;
  // dkdv: K | V (128 keys) | KV_STAGES x (Q | dO) (64 queries) | per-warp LSE / delta slots | barriers
  static constexpr int KV_STAGES = NCH > 2 ? 2 : 3;
  static constexpr int KV_SMEM_K = 0, KV_SMEM_V = NCH * AB_T, KV_SMEM_RING = 2 * NCH * AB_T;
  static constexpr int KV_STAGE = 2 * NCH * AB_H;
  static constexpr int KV_SMEM_STATS = KV_SMEM_RING + KV_STAGES * KV_STAGE;
  static constexpr int KV_SMEM_BAR = KV_SMEM_STATS + 8 * 128 * 4, KV_SMEM_TOTAL = KV_SMEM_BAR + 256 + 1024;
  // dq: Q | dO (128 queries) | DQ_STAGES x (K | V) (64 keys) | barriers
  static constexpr int DQ_STAGES = NCH > 2 ? 2 : 4;
  static constexpr int DQ_SMEM_Q = 0, DQ_SMEM_DO = NCH * AB_T, DQ_SMEM_RING = 2 * NCH * AB_T;
  static constexpr int DQ_STAGE = 2 * NCH * AB_H;
  static constexpr int DQ_SMEM_BAR = DQ_SMEM_RING + DQ_STAGES * DQ_STAGE, DQ_SMEM_TOTAL = DQ_SMEM_BAR + 256 + 1024;
  static_assert(KV_SMEM_TOTAL <= 227 * 1024 && DQ_SMEM_TOTAL <= 227 * 1024, "attention_bwd: shared memory plan exceeds 227 KB");
};

struct AttnBwdArgs {
  CUtensorMap tmQ, tmK, tmV, tmDO;          // 128-row boxes
  CUtensorMap tmQ64, tmK64, tmV64, tmDO64;  // 64-row boxes (the streamed operands)
  const float* lse;    // [B, heads, nq]
  const float* delta;  // [B, heads, nq]
  __nv_bfloat16* dq;
  __nv_bfloat16* dk;
  __nv_bfloat16* dv;
  int nq, nk, heads, lddq, lddk, lddv;
  float scale, scale_log2e;
};

// bf16 A-operand fragments of a 64 x 64 accumulator block (m64n64 layout -> four m64k16 register operands)
__device__ __forceinline__ void acc_to_afrag(const float (&x)[32], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    a[kk][0] = pack_bf16(x[8 * kk + 0], x[8 * kk + 1]);
    a[kk][1] = pack_bf16(x[8 * kk + 2], x[8 * kk + 3]);
    a[kk][2] = pack_bf16(x[8 * kk + 4], x[8 * kk + 5]);
    a[kk][3] = pack_bf16(x[8 * kk + 6], x[8 * kk + 7]);
  }
}

// bf16 store of a 64 x 64 accumulator block: rows row0 / row0 + 8 of this thread, columns 8 j + 2 (lane & 3), of which
// only columns < ncols (the head's real columns in this chunk) are written
__device__ __forceinline__ void store_acc_bf16(const float (&x)[32], __nv_bfloat16* base, size_t ld, int row0, int nrows, int lane,
                                               int ncols) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + 8 * h;
    if (row >= nrows) continue;
    __nv_bfloat16* o = base + static_cast<size_t>(row) * ld + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (ncols >= AB_CHUNK || 8 * j + 2 * (lane & 3) < ncols)
        *reinterpret_cast<uint32_t*>(o + 8 * j) = pack_bf16(x[4 * j + 2 * h], x[4 * j + 2 * h + 1]);
  }
}

// ------------------------------------------------------------------ dK, dV ----
// blockIdx.x = key block * NCH + column chunk
template <int D>
__global__ void __launch_bounds__(AB_THREADS, 1) attention_bwd_dkdv_kernel(const __grid_constant__ AttnBwdArgs p) {
  using P = AbPlan<D>;
  constexpr int NCH = P::NCH, KV_STAGES = P::KV_STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + P::KV_SMEM_BAR);
  uint64_t* kv_full = bars;          // 1
  uint64_t* qdo_full = bars + 1;     // [KV_STAGES]
  uint64_t* qdo_empty = bars + 1 + KV_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = (blockIdx.x / NCH) * 128, chunk = blockIdx.x % NCH, head = blockIdx.y, b = blockIdx.z;
  const int nqb = (p.nq + 63) / 64;
  float* stats = reinterpret_cast<float*>(smem + P::KV_SMEM_STATS) + (warp & 7) * 128;  // this warp's slot

  if (threadIdx.x == 0) {
    mbar_init(kv_full, 1);
    for (int i = 0; i < KV_STAGES; ++i) mbar_init(&qdo_full[i], 1), mbar_init(&qdo_empty[i], 8);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      prefetch_tmap(&p.tmK), prefetch_tmap(&p.tmV), prefetch_tmap(&p.tmQ64), prefetch_tmap(&p.tmDO64);
      mbar_expect_tx(kv_full, 2 * NCH * AB_T);
#pragma unroll
      for (int c = 0; c < NCH; ++c) tma_load_4d(smem + P::KV_SMEM_K + c * AB_T, &p.tmK, kv_full, c * AB_CHUNK, head, k0, b);
#pragma unroll
      for (int c = 0; c < NCH; ++c) tma_load_4d(smem + P::KV_SMEM_V + c * AB_T, &p.tmV, kv_full, c * AB_CHUNK, head, k0, b);
      int st = 0;
      uint32_t ph = 0;
      for (int i = 0; i < nqb; ++i) {
        mbar_wait(&qdo_empty[st], ph ^ 1);
        uint8_t* sQ = smem + P::KV_SMEM_RING + st * P::KV_STAGE;
        mbar_expect_tx(&qdo_full[st], P::KV_STAGE);
#pragma unroll
        for (int c = 0; c < NCH; ++c) tma_load_4d(sQ + c * AB_H, &p.tmQ64, &qdo_full[st], c * AB_CHUNK, head, i * 64, b);
#pragma unroll
        for (int c = 0; c < NCH; ++c)
          tma_load_4d(sQ + (NCH + c) * AB_H, &p.tmDO64, &qdo_full[st], c * AB_CHUNK, head, i * 64, b);
        if (++st == KV_STAGES) st = 0, ph ^= 1;
      }
    }
    return;
  }

  // thread <-> key rows key0 / key0 + 8, query columns 8 j + 2 t4 + {0, 1} of the streamed block
  const int wg = warp >> 2, t4 = lane & 3;
  const int key0 = k0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int keys_left = p.nk - key0;  // this thread's key rows key0 + 8 h are real when 8 h < keys_left
  const size_t stat0 = (static_cast<size_t>(b) * p.heads + head) * p.nq;
  const uint32_t k_addr = smem_u32(smem + P::KV_SMEM_K) + wg * (64 * 128), v_addr = smem_u32(smem + P::KV_SMEM_V) + wg * (64 * 128);
  float dv[32], dk[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dv[i] = 0.f, dk[i] = 0.f;
  mbar_wait(kv_full, 0);
  int st = 0;
  uint32_t ph = 0;
  for (int i = 0; i < nqb; ++i) {
    mbar_wait(&qdo_full[st], ph);
    const uint32_t q_addr = smem_u32(smem + P::KV_SMEM_RING + st * P::KV_STAGE), do_addr = q_addr + NCH * AB_H;
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < NCH * 4; ++k)  // S^T = K Q^T
      Wgmma<64>::ss<0, 0>(s, gmma_desc(k_addr + (k / 4) * AB_T + (k % 4) * 32, 16, 1024),
                          gmma_desc(q_addr + (k / 4) * AB_H + (k % 4) * 32, 16, 1024), k != 0);
#pragma unroll
    for (int k = 0; k < NCH * 4; ++k)  // dP^T = V dO^T
      Wgmma<64>::ss<0, 0>(dp, gmma_desc(v_addr + (k / 4) * AB_T + (k % 4) * 32, 16, 1024),
                          gmma_desc(do_addr + (k / 4) * AB_H + (k % 4) * 32, 16, 1024), k != 0);
    wgmma_commit();
    // log2-domain LSE and scaled delta of the block's 64 queries, two per lane, loaded while the wgmmas run; they go
    // through the warp's shared-memory slot ([lse | delta] x 64) because the 16 query columns each thread needs would
    // take 32 registers for the whole block, which the accumulators and score tiles leave no room for
    float lse_l2[2], delta_s[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int q = i * 64 + 2 * lane + e;
      lse_l2[e] = q < p.nq ? __ldg(p.lse + stat0 + q) * 1.4426950408889634f : 0.f;
      delta_s[e] = q < p.nq ? __ldg(p.delta + stat0 + q) * p.scale : 0.f;
    }
    __syncwarp();  // the previous block's reads of the slot are done
    *reinterpret_cast<float2*>(stats + 2 * lane) = make_float2(lse_l2[0], lse_l2[1]);
    *reinterpret_cast<float2*>(stats + 64 + 2 * lane) = make_float2(delta_s[0], delta_s[1]);
    __syncwarp();
    wgmma_wait<0>();
    const int q_valid = p.nq - i * 64;
    // P, then dS: two passes, so that only one of the two staged rows is read into registers at a time
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 l2 = *reinterpret_cast<const float2*>(stats + 8 * j + 2 * t4);
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * j + 2 * h + e, col = 8 * j + 2 * t4 + e;
          const bool ok = 8 * h < keys_left && col < q_valid;
          s[x] = ok ? ex2_mufu(fmaf(s[x], p.scale_log2e, -(e ? l2.y : l2.x))) : 0.f;
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 ds = *reinterpret_cast<const float2*>(stats + 64 + 8 * j + 2 * t4);
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * j + 2 * h + e;
          dp[x] = s[x] * fmaf(dp[x], p.scale, -(e ? ds.y : ds.x));
        }
    }
    uint32_t pa[4][4], da[4][4];
    acc_to_afrag(s, pa);
    acc_to_afrag(dp, da);
    const uint32_t do_c = do_addr + chunk * AB_H, q_c = q_addr + chunk * AB_H;  // this CTA's 64 columns of dO and Q
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {  // K = 64 query rows, 16 per instruction; B operands MN-major
      Wgmma<64>::rs<1>(dv, pa[kk], gmma_desc(do_c + kk * 2048, 8192, 1024), 1u);
      Wgmma<64>::rs<1>(dk, da[kk], gmma_desc(q_c + kk * 2048, 8192, 1024), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&qdo_empty[st]);
    if (++st == KV_STAGES) st = 0, ph ^= 1;
  }
  const size_t row_base = static_cast<size_t>(b) * p.nk;
  const int col0 = head * D + chunk * AB_CHUNK, ncols = D - chunk * AB_CHUNK;
  store_acc_bf16(dv, p.dv + row_base * p.lddv + col0, p.lddv, key0, p.nk, lane, ncols);
  store_acc_bf16(dk, p.dk + row_base * p.lddk + col0, p.lddk, key0, p.nk, lane, ncols);
}

// ---------------------------------------------------------------------- dQ ----
// blockIdx.x = query block * NCH + column chunk
constexpr int DQ_BKV = 64;

template <int D>
__global__ void __launch_bounds__(AB_THREADS, 1) attention_bwd_dq_kernel(const __grid_constant__ AttnBwdArgs p) {
  using P = AbPlan<D>;
  constexpr int NCH = P::NCH, DQ_STAGES = P::DQ_STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + P::DQ_SMEM_BAR);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;               // [DQ_STAGES]
  uint64_t* kv_empty = bars + 1 + DQ_STAGES;  // [DQ_STAGES]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = (blockIdx.x / NCH) * 128, chunk = blockIdx.x % NCH, head = blockIdx.y, b = blockIdx.z;
  const int nkb = (p.nk + DQ_BKV - 1) / DQ_BKV;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < DQ_STAGES; ++i) mbar_init(&kv_full[i], 1), mbar_init(&kv_empty[i], 8);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      prefetch_tmap(&p.tmQ), prefetch_tmap(&p.tmDO), prefetch_tmap(&p.tmK64), prefetch_tmap(&p.tmV64);
      mbar_expect_tx(q_full, 2 * NCH * AB_T);
#pragma unroll
      for (int c = 0; c < NCH; ++c) tma_load_4d(smem + P::DQ_SMEM_Q + c * AB_T, &p.tmQ, q_full, c * AB_CHUNK, head, q0, b);
#pragma unroll
      for (int c = 0; c < NCH; ++c) tma_load_4d(smem + P::DQ_SMEM_DO + c * AB_T, &p.tmDO, q_full, c * AB_CHUNK, head, q0, b);
      int st = 0;
      uint32_t ph = 0;
      for (int j = 0; j < nkb; ++j) {
        mbar_wait(&kv_empty[st], ph ^ 1);
        uint8_t* sK = smem + P::DQ_SMEM_RING + st * P::DQ_STAGE;
        mbar_expect_tx(&kv_full[st], P::DQ_STAGE);
#pragma unroll
        for (int c = 0; c < NCH; ++c) tma_load_4d(sK + c * AB_H, &p.tmK64, &kv_full[st], c * AB_CHUNK, head, j * DQ_BKV, b);
#pragma unroll
        for (int c = 0; c < NCH; ++c)
          tma_load_4d(sK + (NCH + c) * AB_H, &p.tmV64, &kv_full[st], c * AB_CHUNK, head, j * DQ_BKV, b);
        if (++st == DQ_STAGES) st = 0, ph ^= 1;
      }
    }
    return;
  }

  // thread <-> query rows row0 / row0 + 8, key columns 8 j + 2 t4 + {0, 1} of the streamed block
  const int wg = warp >> 2, t4 = lane & 3;
  const int row0 = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  bool row_ok[2];
  float lse_l2[2], delta_s[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + 8 * h;
    row_ok[h] = row < p.nq;
    const size_t o = (static_cast<size_t>(b) * p.heads + head) * p.nq + row;
    lse_l2[h] = row_ok[h] ? p.lse[o] * 1.4426950408889634f : 0.f;
    delta_s[h] = row_ok[h] ? p.delta[o] * p.scale : 0.f;
  }
  const uint32_t q_addr = smem_u32(smem + P::DQ_SMEM_Q) + wg * (64 * 128), do_addr = smem_u32(smem + P::DQ_SMEM_DO) + wg * (64 * 128);
  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;
  mbar_wait(q_full, 0);
  int st = 0;
  uint32_t ph = 0;
  for (int j = 0; j < nkb; ++j) {
    mbar_wait(&kv_full[st], ph);
    const uint32_t k_addr = smem_u32(smem + P::DQ_SMEM_RING + st * P::DQ_STAGE), v_addr = k_addr + NCH * AB_H;
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < NCH * 4; ++k)  // S = Q K^T
      Wgmma<64>::ss<0, 0>(s, gmma_desc(q_addr + (k / 4) * AB_T + (k % 4) * 32, 16, 1024),
                          gmma_desc(k_addr + (k / 4) * AB_H + (k % 4) * 32, 16, 1024), k != 0);
#pragma unroll
    for (int k = 0; k < NCH * 4; ++k)  // dP = dO V^T
      Wgmma<64>::ss<0, 0>(dp, gmma_desc(do_addr + (k / 4) * AB_T + (k % 4) * 32, 16, 1024),
                          gmma_desc(v_addr + (k / 4) * AB_H + (k % 4) * 32, 16, 1024), k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    const int valid_keys = p.nk - j * DQ_BKV;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * jj + 2 * h + e, col = 8 * jj + 2 * t4 + e;
          const bool ok = row_ok[h] && col < valid_keys;
          const float pr = ok ? ex2_mufu(fmaf(s[x], p.scale_log2e, -lse_l2[h])) : 0.f;
          dp[x] = pr * fmaf(dp[x], p.scale, -delta_s[h]);
        }
    uint32_t da[4][4];
    acc_to_afrag(dp, da);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)  // dQ += dS K: B = this CTA's 64 columns of K, rows of 16 keys (MN-major)
      Wgmma<64>::rs<1>(dq, da[kk], gmma_desc(k_addr + chunk * AB_H + kk * 2048, 8192, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[st]);
    if (++st == DQ_STAGES) st = 0, ph ^= 1;
  }
  store_acc_bf16(dq, p.dq + static_cast<size_t>(b) * p.nq * p.lddq + head * D + chunk * AB_CHUNK, p.lddq, row0, p.nq, lane,
                 D - chunk * AB_CHUNK);
}

__device__ __forceinline__ float dot8_bf16(const uint4 a, const uint4 b4) {
  return bf16_lo(a.x) * bf16_lo(b4.x) + bf16_hi(a.x) * bf16_hi(b4.x) + bf16_lo(a.y) * bf16_lo(b4.y) +
         bf16_hi(a.y) * bf16_hi(b4.y) + bf16_lo(a.z) * bf16_lo(b4.z) + bf16_hi(a.z) * bf16_hi(b4.z) +
         bf16_lo(a.w) * bf16_lo(b4.w) + bf16_hi(a.w) * bf16_hi(b4.w);
}

// delta[b,h,q] = sum_d dO * O ; 8 threads per (row, head), 16-byte loads: thread `sub` sums the 8-column chunks
// sub, sub + 8, .. of the head's D / 8, in that order, then the 8 partial sums are combined by a fixed shuffle tree
template <int D>
__global__ void attention_delta_kernel(const __nv_bfloat16* __restrict__ o, int ldo, const __nv_bfloat16* __restrict__ d_o,
                                       int lddo, float* __restrict__ delta, int B, int nq, int heads) {
  const int64_t gid = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 3;
  const int sub = threadIdx.x & 7;
  const int64_t total = static_cast<int64_t>(B) * nq * heads;
  float acc = 0.f;
  int64_t row = 0;
  int h = 0;
  const bool ok = gid < total;
  if (ok) {
    row = gid / heads;
    h = gid % heads;
    const __nv_bfloat16* orow = o + row * ldo + h * D;
    const __nv_bfloat16* dorow = d_o + row * lddo + h * D;
    if (D / 8 % 8 == 0 || sub < D / 8)
      acc = dot8_bf16(*reinterpret_cast<const uint4*>(orow + sub * 8), *reinterpret_cast<const uint4*>(dorow + sub * 8));
#pragma unroll
    for (int c = sub + 8; c < D / 8; c += 8)
      acc += dot8_bf16(*reinterpret_cast<const uint4*>(orow + c * 8), *reinterpret_cast<const uint4*>(dorow + c * 8));
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  acc += __shfl_xor_sync(0xffffffffu, acc, 4);
  if (ok && sub == 0) {
    const int b = row / nq, qi = row % nq;
    delta[(static_cast<size_t>(b) * heads + h) * nq + qi] = acc;
  }
}

// [batch, n, ld] bf16 with head h at columns [h d, h d + d): boxes of 64 columns x box_rows rows; columns past d of a
// box are out of the tensor's innermost extent and arrive as zeros
static int make_map(CUtensorMap* m, const void* base, int d, int heads, int n, int batch, int ld, int box_rows = 128) {
  uint64_t dims[4] = {(uint64_t)d, (uint64_t)heads, (uint64_t)n, (uint64_t)batch};
  uint64_t strides[3] = {(uint64_t)d * 2, (uint64_t)ld * 2, (uint64_t)ld * 2 * n};
  uint32_t box[4] = {(uint32_t)AB_CHUNK, 1, (uint32_t)box_rows, 1};
  uint32_t es[4] = {1, 1, 1, 1};
  return make_tensor_map(m, base, 2, 4, dims, strides, box, es, 1);
}

template <int D>
static int attention_bwd_launch(const ddpo_attention_bwd_args* a, cudaStream_t stream) {
  using P = AbPlan<D>;
  AttnBwdArgs p;
  memset(&p, 0, sizeof(p));
  int rc;
  if ((rc = make_map(&p.tmQ, a->q, D, a->heads, a->nq, a->batch, a->ldq))) return rc;
  if ((rc = make_map(&p.tmK, a->k, D, a->heads, a->nk, a->batch, a->ldk))) return rc;
  if ((rc = make_map(&p.tmV, a->v, D, a->heads, a->nk, a->batch, a->ldv))) return rc;
  if ((rc = make_map(&p.tmDO, a->dout, D, a->heads, a->nq, a->batch, a->lddo))) return rc;
  if ((rc = make_map(&p.tmQ64, a->q, D, a->heads, a->nq, a->batch, a->ldq, 64))) return rc;
  if ((rc = make_map(&p.tmK64, a->k, D, a->heads, a->nk, a->batch, a->ldk, 64))) return rc;
  if ((rc = make_map(&p.tmV64, a->v, D, a->heads, a->nk, a->batch, a->ldv, 64))) return rc;
  if ((rc = make_map(&p.tmDO64, a->dout, D, a->heads, a->nq, a->batch, a->lddo, 64))) return rc;
  p.lse = a->lse, p.delta = a->delta;
  p.dq = static_cast<__nv_bfloat16*>(a->dq), p.dk = static_cast<__nv_bfloat16*>(a->dk);
  p.dv = static_cast<__nv_bfloat16*>(a->dv);
  p.nq = a->nq, p.nk = a->nk, p.heads = a->heads, p.lddq = a->lddq, p.lddk = a->lddk, p.lddv = a->lddv;
  p.scale = 1.0f / sqrtf(static_cast<float>(D));
  p.scale_log2e = p.scale * 1.4426950408889634f;
  static bool attr = false;
  if (!attr) {
    DDPO_CUDA_OK(cudaFuncSetAttribute(attention_bwd_dkdv_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, P::KV_SMEM_TOTAL));
    DDPO_CUDA_OK(cudaFuncSetAttribute(attention_bwd_dq_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, P::DQ_SMEM_TOTAL));
    attr = true;
  }
  const int64_t items = static_cast<int64_t>(a->batch) * a->nq * a->heads;
  attention_delta_kernel<D><<<static_cast<int>((items * 8 + 255) / 256), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(a->out), a->ldo, static_cast<const __nv_bfloat16*>(a->dout), a->lddo, a->delta,
      a->batch, a->nq, a->heads);
  DDPO_LAUNCH_OK();
  dim3 g1((a->nk + 127) / 128 * P::NCH, a->heads, a->batch);
  attention_bwd_dkdv_kernel<D><<<g1, AB_THREADS, P::KV_SMEM_TOTAL, stream>>>(p);
  DDPO_LAUNCH_OK();
  dim3 g2((a->nq + 127) / 128 * P::NCH, a->heads, a->batch);
  attention_bwd_dq_kernel<D><<<g2, AB_THREADS, P::DQ_SMEM_TOTAL, stream>>>(p);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

}  // namespace ddpo

using namespace ddpo;

extern "C" int ddpo_attention_bwd(const ddpo_attention_bwd_args* a, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DDPO_REQUIRE(a && a->q && a->k && a->v && a->out && a->dout && a->lse && a->delta && a->dq && a->dk && a->dv,
               "attention_bwd: null pointer");
  const int d = a->head_dim;
  DDPO_REQUIRE(d == 40 || d == 64 || d == 80 || d == 160, "attention_bwd: head_dim must be 40, 64, 80 or 160 (got %d)", d);
  DDPO_REQUIRE(a->nq > 0 && a->nk > 0 && a->heads > 0 && a->batch > 0, "attention_bwd: bad sizes");
  const int h = a->heads;
  DDPO_REQUIRE(attention_operands_ok(a->q, a->ldq, h, d) && attention_operands_ok(a->k, a->ldk, h, d) &&
                   attention_operands_ok(a->v, a->ldv, h, d) && attention_operands_ok(a->out, a->ldo, h, d) &&
                   attention_operands_ok(a->dout, a->lddo, h, d) && attention_operands_ok(a->dq, a->lddq, h, d) &&
                   attention_operands_ok(a->dk, a->lddk, h, d) && attention_operands_ok(a->dv, a->lddv, h, d),
               "attention_bwd: q/k/v/out/dout/dq/dk/dv need 16-byte aligned base pointers, pitches that are multiples "
               "of 8 elements and at least heads * head_dim");
  switch (d) {
    case 40: return attention_bwd_launch<40>(a, stream);
    case 80: return attention_bwd_launch<80>(a, stream);
    case 160: return attention_bwd_launch<160>(a, stream);
    default: return attention_bwd_launch<64>(a, stream);
  }
}
