// Implicit-GEMM convolution / linear layer on wgmma (sm_90a).
//
//   out[m, n] = epilogue( sum_{tap, c} A[(b, y*s+dy-p, x*s+dx-p), c] * Wt[n, (tap, c)] )
//
// replaces every dense contraction of the Flax U-Net the reference runs through
// `unet.apply` (reference call sites: pipeline_flax_stable_diffusion.py:219-224,
// training/policy_gradient.py:87-102): nn.Conv 3x3 / 3x3 stride-2 / 1x1 and nn.Dense.
//
// Design:
//  * one CTA per BM x BN output tile (n fastest, so the BM-row activation tile of consecutive CTAs is re-used out
//    of L2); BM (64 or 128) and BN (the N of the wgmma instruction) are template parameters, chosen per launch by
//    `pick_tile` from the shape so that the last wave of tiles is as full as the cost model allows;
//  * the last warp = TMA producer.  The activation operand is fetched straight from the NHWC bf16 tensor with a 4-D
//    tiled tensor map whose box is (64 ch, bw, bh, bb) pixels, bw*bh*bb = BM; the 3x3 taps are the same box shifted by
//    (dx-1, dy-1) and TMA's out-of-bounds zero fill IS the conv padding -> no im2col buffer ever exists.
//    Channel-concatenated inputs (U-Net skip connections) are two tensor maps walked back to back.  Stages of a
//    multi-stage ring are handed over through full / empty mbarriers;
//  * the other warps = BM / 64 consumer warpgroups, 64 rows each: m64nBNk16 bf16 wgmma from shared memory (both
//    operands K-major, 128-byte swizzle), fp32 accumulators in registers, one k-block of wgmma in flight while the
//    next is issued;
//  * epilogue: the accumulators go through shared memory (the drained stage ring) so that every global access of the
//    fused bias / per-sample time-embedding row vector / fp32 residual / GEGLU / slab statistics is coalesced;
//  * K order is fixed and independent of the batch size, of the tile shape and of the position of a row in its
//    tile (each warpgroup runs its own 64 rows over the whole K) -> results are batch-invariant and bit-reproducible
//    whatever (BM, BN) a launch gets (the PPO ratio of an unchanged policy must be exactly 1; reference
//    config/base.py:88 clip 1e-4).
#include "common.cuh"
#include "gemm_model.cuh"
#include "wgmma.cuh"

namespace ddpo {

constexpr int BK = 64;
constexpr int SMEM_PER_SM = 228 * 1024;
constexpr int SMEM_BUDGET = 227 * 1024 - 1024 /*align slack*/ - 256 /*barriers*/;

template <int BM>
constexpr int igemm_consumers() { return BM * 2; }  // one 128-thread warpgroup per 64 rows
template <int BM>
constexpr int igemm_threads() { return igemm_consumers<BM>() + 32; }  // + the TMA producer warp
template <int BM, int BN>
constexpr int igemm_stage_bytes() { return (BM + BN) * BK * 2; }
template <int BM, int BN>
constexpr int igemm_epi_bytes() { return BM * (BN + 4) * 4; }  // fp32 tile, rows padded by 16 B against bank conflicts
// Shared memory one of c co-resident CTAs may use for its ring: the SM's 228 KB less 1 KB the hardware reserves per
// CTA, the alignment slack and the barriers.
constexpr int igemm_smem_budget(int c) { return c == 1 ? SMEM_BUDGET : SMEM_PER_SM / c - 1024 - 1024 - 256; }
// CTAs per SM: the most (at most four consumer warpgroups per SM) that still leave every CTA three operand stages and
// room for the epilogue tile, and whose registers fit (about BN / 2 accumulators + 40 per thread in a 64K register
// file).  Also the __launch_bounds__ occupancy, so ptxas holds the register count to it.
template <int BM, int BN>
constexpr int igemm_ctas_per_sm() {
  for (int c = 256 / BM; c > 1; --c) {
    const int budget = igemm_smem_budget(c);
    if (budget / igemm_stage_bytes<BM, BN>() >= 3 && budget >= igemm_epi_bytes<BM, BN>() &&
        c * igemm_threads<BM>() * (BN / 2 + 40) <= 65536)
      return c;
  }
  return 1;
}
template <int BM, int BN>
constexpr int igemm_stages() {
  const int s = igemm_smem_budget(igemm_ctas_per_sm<BM, BN>()) / igemm_stage_bytes<BM, BN>();
  return s > 8 ? 8 : s;
}

struct IGemmArgs {
  CUtensorMap tmA0, tmA1, tmB;
  int M_total, N_total, stages;
  int taps, kc0, kc1;
  int is_conv, W, H, conv_stride, pad;
  const float* bias;      // [N] or null
  const float* rowvec;    // [B, rowvec_ld] or null: added per sample (time-embedding projection)
  int rows_per_sample, rowvec_ld;
  const float* residual;  // [M, ld_res] fp32 or null
  int ld_res;
  float* out_f32;         // [M, ld_out] or null
  __nv_bfloat16* out_bf16;  // [M, ld_out] or null  (GEGLU: [M, ld_out] with N/2 useful columns)
  int ld_out;
  int geglu;
  int accumulate_out;     // out_f32 += result (used by backward passes that sum two branches)
  float* gn_stats;        // [ceil(M/32), N, 2] or null: per 32-row slab, per column (sum, sum of squares) of the fp32 OUTPUT
                          // values -- the GroupNorm that consumes out_f32 takes its statistics from these instead of
                          // re-reading the tensor (norm.cu gn_finalize_kernel)
  __nv_bfloat16* aux_bf16;  // GEGLU only: pre-activation [M, N] (tile-interleaved, bias included) kept for backward
};

__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ uint2 pack_bf16x4(float4 v) { return make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w)); }

template <int BM, int BN>
__global__ void __launch_bounds__(igemm_threads<BM>(), igemm_ctas_per_sm<BM, BN>())
    igemm_kernel(const __grid_constant__ IGemmArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int CONSUMERS = igemm_consumers<BM>();
  constexpr int A_TILE_BYTES = BM * BK * 2;
  constexpr int SB = igemm_stage_bytes<BM, BN>();
  constexpr int EPI = igemm_epi_bytes<BM, BN>();
  const int stages = p.stages;
  const int main_bytes = stages * SB > EPI ? stages * SB : EPI;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + main_bytes);
  uint64_t* empty_bar = full_bar + stages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_n = p.N_total / BN;
  const int tm = blockIdx.x / tiles_n, tn = blockIdx.x % tiles_n;
  const int m0 = tm * BM, n0 = tn * BN;
  const int kcs = p.kc0 + p.kc1;
  const int kiters = p.taps * kcs;

  if (threadIdx.x == 0) {
    for (int i = 0; i < stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], CONSUMERS / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == CONSUMERS / 32) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0) {
      prefetch_tmap(&p.tmA0);
      prefetch_tmap(&p.tmA1);
      prefetch_tmap(&p.tmB);
      int b0 = 0, h0 = 0, w0 = 0;
      if (p.is_conv) {
        const int HW = p.W * p.H;
        b0 = m0 / HW;
        h0 = (m0 % HW) / p.W;
        w0 = m0 % p.W;  // non-zero only when a pixel row is wider than a tile (W > BM)
      }
      int stage = 0;
      uint32_t phase = 0;
      int kit = 0;
      for (int tap = 0; tap < p.taps; ++tap) {
        const int dy = p.taps == 9 ? tap / 3 : 0, dx = p.taps == 9 ? tap - dy * 3 : 0;
        for (int ch = 0; ch < kcs; ++ch, ++kit) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sA = smem + stage * SB;
          mbar_expect_tx(&full_bar[stage], SB);
          if (p.is_conv) {
            const int cx = w0 * p.conv_stride + dx - p.pad;
            const int cy = h0 * p.conv_stride + dy - p.pad;
            if (ch < p.kc0)
              tma_load_4d(sA, &p.tmA0, &full_bar[stage], ch * BK, cx, cy, b0);
            else
              tma_load_4d(sA, &p.tmA1, &full_bar[stage], (ch - p.kc0) * BK, cx, cy, b0);
          } else {
            tma_load_2d(sA, &p.tmA0, &full_bar[stage], kit * BK, m0);
          }
          tma_load_2d(sA + A_TILE_BYTES, &p.tmB, &full_bar[stage], kit * BK, n0);
          if (++stage == stages) stage = 0, phase ^= 1;
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------- consumers
  const int wg = warp >> 2;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  {
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int kit = 0; kit < kiters; ++kit) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_base = smem_u32(smem + stage * SB) + wg * (64 * 128);
      const uint32_t b_base = smem_u32(smem + stage * SB + A_TILE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        Wgmma<BN>::template ss<0, 0>(acc, gmma_desc(a_base + k * 32, 16, 1024), gmma_desc(b_base + k * 32, 16, 1024),
                                     (kit | k) != 0);
      wgmma_commit();
      wgmma_wait<1>();  // the previous k-block has finished reading its stage
      if (kit > 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == stages) stage = 0, phase ^= 1;
    }
    wgmma_wait<0>();
  }
  named_barrier(1, CONSUMERS);  // every operand stage has been read: the ring becomes the epilogue tile

  // ---------------------------------------------------------------- epilogue
  constexpr int P = BN + 4;
  float* stg = reinterpret_cast<float*>(smem);
  {
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      *reinterpret_cast<float2*>(stg + r0 * P + 8 * j + cq) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(stg + (r0 + 8) * P + 8 * j + cq) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  named_barrier(1, CONSUMERS);
  const int tid = threadIdx.x;
  if (p.geglu) {
    // GEGLU: this N tile is [BN/2 linear | BN/2 gate] columns of the same output channels (host-side row permutation):
    // out = lin * gelu_tanh(gate) -> out_bf16[:, tn*BN/2 + c], pre-activations (training) -> aux[:, n0 + c] / [n0 + BN/2 + c]
    constexpr int HALF = BN / 2, H4 = HALF / 4;
    for (int idx = tid; idx < BM * H4; idx += CONSUMERS) {
      const int r = idx / H4, c = (idx % H4) * 4;
      const int row = m0 + r;
      if (row >= p.M_total) continue;
      const int n = n0 + c;
      const float4 lin = add4(*reinterpret_cast<const float4*>(stg + r * P + c), __ldg(reinterpret_cast<const float4*>(p.bias + n)));
      const float4 gate =
          add4(*reinterpret_cast<const float4*>(stg + r * P + HALF + c), __ldg(reinterpret_cast<const float4*>(p.bias + n + HALF)));
      const float4 f = make_float4(lin.x * gelu_tanh_f(gate.x), lin.y * gelu_tanh_f(gate.y), lin.z * gelu_tanh_f(gate.z),
                                   lin.w * gelu_tanh_f(gate.w));
      *reinterpret_cast<uint2*>(p.out_bf16 + static_cast<size_t>(row) * p.ld_out + tn * HALF + c) = pack_bf16x4(f);
      if (p.aux_bf16 != nullptr) {
        __nv_bfloat16* ax = p.aux_bf16 + static_cast<size_t>(row) * p.N_total + n;
        *reinterpret_cast<uint2*>(ax) = pack_bf16x4(lin);
        *reinterpret_cast<uint2*>(ax + HALF) = pack_bf16x4(gate);
      }
    }
    return;
  }
  constexpr int C4 = BN / 4;
  for (int idx = tid; idx < BM * C4; idx += CONSUMERS) {
    const int r = idx / C4, c = (idx % C4) * 4;
    const int row = m0 + r;
    float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row < p.M_total) {
      const int n = n0 + c;
      f = *reinterpret_cast<const float4*>(stg + r * P + c);
      if (p.bias != nullptr) f = add4(f, __ldg(reinterpret_cast<const float4*>(p.bias + n)));
      if (p.rowvec != nullptr)
        f = add4(f, __ldg(reinterpret_cast<const float4*>(p.rowvec + static_cast<size_t>(row / p.rows_per_sample) * p.rowvec_ld + n)));
      if (p.residual != nullptr) f = add4(f, *reinterpret_cast<const float4*>(p.residual + static_cast<size_t>(row) * p.ld_res + n));
      if (p.out_f32 != nullptr) {
        float4* o = reinterpret_cast<float4*>(p.out_f32 + static_cast<size_t>(row) * p.ld_out + n);
        if (p.accumulate_out) f = add4(f, *o);
        *o = f;
      }
      if (p.out_bf16 != nullptr)
        *reinterpret_cast<uint2*>(p.out_bf16 + static_cast<size_t>(row) * p.ld_out + n) = pack_bf16x4(f);
    }
    if (p.gn_stats != nullptr) *reinterpret_cast<float4*>(stg + r * P + c) = f;  // rows outside the matrix count as zeros
  }
  if (p.gn_stats == nullptr) return;
  named_barrier(1, CONSUMERS);
  // slab statistics: per 32-row slab and column, (sum, sum of squares) over the rows in order -- a function of the 32
  // values only
  for (int idx = tid; idx < (BM / 32) * BN; idx += CONSUMERS) {
    const int s = idx / BN, c = idx % BN;
    const int m_slab = m0 + s * 32;
    if (m_slab >= p.M_total) continue;
    float sum = 0.f, sq = 0.f;
#pragma unroll 8
    for (int r = 0; r < 32; ++r) {
      const float v = stg[(s * 32 + r) * P + c];
      sum += v;
      sq = fmaf(v, v, sq);
    }
    *reinterpret_cast<float2*>(p.gn_stats + (static_cast<size_t>(m_slab >> 5) * p.N_total + n0 + c) * 2) = make_float2(sum, sq);
  }
}

template <int BM, int BN>
static int igemm_launch(IGemmArgs& p, cudaStream_t stream) {
  constexpr int SB = igemm_stage_bytes<BM, BN>();
  constexpr int EPI = igemm_epi_bytes<BM, BN>();
  p.stages = igemm_stages<BM, BN>();
  const size_t smem = (size_t)(p.stages * SB > EPI ? p.stages * SB : EPI) + 256 + 1024;
  static bool attr_set = false;
  if (!attr_set) {
    DDPO_CUDA_OK(cudaFuncSetAttribute(igemm_kernel<BM, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  const int tiles = ((p.M_total + BM - 1) / BM) * (p.N_total / BN);
  igemm_kernel<BM, BN><<<tiles, igemm_threads<BM>(), smem, stream>>>(p);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

struct TileShape {
  int bm, bn, ctas_per_sm, stages;
  int (*launch)(IGemmArgs&, cudaStream_t);
};
template <int BM, int BN>
constexpr TileShape tile_shape() { return {BM, BN, igemm_ctas_per_sm<BM, BN>(), igemm_stages<BM, BN>(), igemm_launch<BM, BN>}; }
// Every instantiated tile, largest first: a tie in the cost model goes to the tile that re-reads its operands least.
// There is no 64 x 256 tile: it fits one CTA per SM, a single warpgroup that cannot keep the tensor cores busy (every
// tile here puts at least two consumer warpgroups on an SM).
constexpr TileShape TILES[] = {tile_shape<128, 256>(), tile_shape<128, 192>(), tile_shape<128, 160>(), tile_shape<128, 128>(),
                               tile_shape<128, 96>(),  tile_shape<64, 192>(),  tile_shape<64, 160>(),  tile_shape<128, 64>(),
                               tile_shape<64, 128>(),  tile_shape<64, 96>(),   tile_shape<128, 32>(),  tile_shape<64, 64>(),
                               tile_shape<64, 32>()};

// GEGLU tiles hold [BN/2 linear | BN/2 gate] and must match the weight permutation (ddpo_prep_weight geglu_bn).
static int geglu_width(int N) {
  for (int w : {256, 192, 128, 64})
    if (N % w == 0) return w;
  return 0;
}

// Cost model of one launch (gemm_model.cuh), in SM clock cycles.
constexpr double EPI_BYTES_PER_ELEM = 8.0;      // epilogue traffic per output element: an fp32 store plus one fp32 read
                                                // (residual, accumulate) or bf16 store, typical of the U-Net's launches
// Makespan = waves x the time of one wave, a wave being K / 16 steps of k16_step_clk plus the epilogue.  The c CTAs
// of a wave share the SM: with c >= 2 one CTA's epilogue overlaps the others' main loops, with c = 1 it does not.
static double tile_makespan(const TileShape& t, int M, int N, int K) {
  const double main_loop = (K / 16) * k16_step_clk(t.bm, t.bn);
  const double epilogue = double(t.bm) * t.bn * EPI_BYTES_PER_ELEM / HBM_BYTES_PER_CLK;
  const double wave = t.ctas_per_sm > 1 ? t.ctas_per_sm * fmax(main_loop, epilogue) : main_loop + epilogue;
  const long long tiles = (long long)((M + t.bm - 1) / t.bm) * (N / t.bn);
  const long long slots = (long long)NUM_SMS * t.ctas_per_sm;
  return double((tiles + slots - 1) / slots) * wave;
}

// The tile of a launch: a function of (M, N, K, GEGLU) alone, so that a layer always runs the same tiles whatever else
// runs.  The K order of an output element does not depend on the tile, so this is a pure scheduling choice: the tile
// with the least modelled makespan.  bm / bn > 0 restrict the choice to tiles of that height / width (tests).
static const TileShape* pick_tile(int M, int N, int K, int geglu, int bm, int bn) {
  const TileShape* best = nullptr;
  double best_time = 0.0;
  for (const TileShape& t : TILES) {
    if ((bm > 0 && t.bm != bm) || (bn > 0 && t.bn != bn) || N % t.bn != 0 || (geglu && bn <= 0 && t.bn != geglu_width(N)))
      continue;
    const double time = tile_makespan(t, M, N, K);
    if (best == nullptr || time < best_time) best = &t, best_time = time;
  }
  return best;
}

}  // namespace ddpo

using namespace ddpo;

extern "C" int ddpo_igemm(const ddpo_igemm_args* a, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DDPO_REQUIRE(a != nullptr, "ddpo_igemm: null args");
  const int cin0 = a->c0, cin1 = a->c1;
  DDPO_REQUIRE(cin0 > 0 && cin0 % BK == 0 && cin1 % BK == 0, "ddpo_igemm: channel counts must be multiples of 64 (c0=%d c1=%d)", cin0, cin1);
  DDPO_REQUIRE(a->taps == 1 || a->taps == 9, "ddpo_igemm: taps must be 1 or 9");
  DDPO_REQUIRE(a->n % 32 == 0, "ddpo_igemm: N=%d must be a multiple of 32", a->n);
  DDPO_REQUIRE(a->out_f32 != nullptr || a->out_bf16 != nullptr, "ddpo_igemm: no output");
  const int ktot = a->taps * (cin0 + cin1);
  const int M_total = a->is_conv ? a->batch * a->w * a->h : a->m;
  const TileShape* tile = pick_tile(M_total, a->n, ktot, a->geglu, a->bm_override, a->bn_override);
  DDPO_REQUIRE(tile != nullptr, "ddpo_igemm: no %d x %d tile for N=%d", a->bm_override, a->bn_override, a->n);
  const int BM = tile->bm, BN = tile->bn;
  if (a->geglu) DDPO_REQUIRE(BN % 64 == 0 && a->out_bf16 != nullptr && a->bias != nullptr, "ddpo_igemm: bad GEGLU config");

  IGemmArgs p;
  memset(&p, 0, sizeof(p));
  if (a->is_conv) {
    // output grid W x H per sample (input grid is stride x larger)
    const int W = a->w, H = a->h, B = a->batch, s = a->conv_stride;
    DDPO_REQUIRE(s == 1 || s == 2, "ddpo_igemm: stride must be 1 or 2");
    DDPO_REQUIRE(W > 0 && H > 0 && (W & (W - 1)) == 0 && (H & (H - 1)) == 0 && W <= 1024,
                 "ddpo_igemm: W,H must be powers of two, W<=1024 (W=%d H=%d)", W, H);
    // a BM-row tile is bb samples x bh rows x bw pixels; rows wider than the tile are cut into W/BM tiles (with
    // stride 2 a 128-pixel box spans 256 input elements, the TMA limit)
    int bw = W < BM ? W : BM, bh = (BM / bw < H) ? BM / bw : H;
    int bb = BM / (bw * bh);
    const int Wi = W * s, Hi = H * s;
    for (int src = 0; src < (cin1 > 0 ? 2 : 1); ++src) {
      const int C = src == 0 ? cin0 : cin1;
      const void* base = src == 0 ? a->a0 : a->a1;
      const int ld = src == 0 ? a->lda0 : a->lda1;  // channel pitch (elements) of a pixel row
      DDPO_REQUIRE(base != nullptr && ld >= C, "ddpo_igemm: bad A source %d", src);
      uint64_t dims[4] = {(uint64_t)C, (uint64_t)Wi, (uint64_t)Hi, (uint64_t)B};
      uint64_t strides[3] = {(uint64_t)ld * 2, (uint64_t)ld * 2 * Wi, (uint64_t)ld * 2 * Wi * Hi};
      uint32_t box[4] = {(uint32_t)BK, (uint32_t)(bw * s), (uint32_t)(bh * s), (uint32_t)bb};
      uint32_t es[4] = {1, (uint32_t)s, (uint32_t)s, 1};
      int rc = make_tensor_map(src == 0 ? &p.tmA0 : &p.tmA1, base, 2, 4, dims, strides, box, es, 1);
      if (rc) return rc;
    }
    if (cin1 == 0) p.tmA1 = p.tmA0;
    p.W = W, p.H = H, p.conv_stride = s, p.pad = (a->taps == 9 && a->conv_pad == 0) ? 1 : 0;
  } else {
    DDPO_REQUIRE(a->taps == 1 && cin1 == 0, "ddpo_igemm: linear mode takes one source, one tap");
    uint64_t dims[2] = {(uint64_t)cin0, (uint64_t)M_total};
    uint64_t strides[1] = {(uint64_t)a->lda0 * 2};
    uint32_t box[2] = {(uint32_t)BK, (uint32_t)BM};
    uint32_t es[2] = {1, 1};
    int rc = make_tensor_map(&p.tmA0, a->a0, 2, 2, dims, strides, box, es, 1);
    if (rc) return rc;
    p.tmA1 = p.tmA0;
    p.W = 1, p.H = 1, p.conv_stride = 1, p.pad = 0;
  }
  {
    uint64_t dims[2] = {(uint64_t)ktot, (uint64_t)a->n};
    uint64_t strides[1] = {(uint64_t)ktot * 2};
    uint32_t box[2] = {(uint32_t)BK, (uint32_t)BN};
    uint32_t es[2] = {1, 1};
    int rc = make_tensor_map(&p.tmB, a->wt, 2, 2, dims, strides, box, es, 1);
    if (rc) return rc;
  }
  p.M_total = M_total, p.N_total = a->n;
  p.taps = a->taps, p.kc0 = cin0 / BK, p.kc1 = cin1 / BK, p.is_conv = a->is_conv;
  p.bias = a->bias, p.rowvec = a->rowvec, p.rows_per_sample = a->rows_per_sample > 0 ? a->rows_per_sample : 1;
  p.rowvec_ld = a->rowvec_ld;
  p.residual = a->residual, p.ld_res = a->ld_res > 0 ? a->ld_res : a->n;
  p.out_f32 = a->out_f32, p.out_bf16 = static_cast<__nv_bfloat16*>(a->out_bf16);
  p.ld_out = a->ld_out > 0 ? a->ld_out : (a->geglu ? a->n / 2 : a->n);
  p.geglu = a->geglu, p.accumulate_out = a->accumulate_out;
  p.aux_bf16 = static_cast<__nv_bfloat16*>(a->aux_bf16);
  p.gn_stats = a->gn_stats;
  // the epilogue moves four columns per access: 16-byte fp32 / 8-byte bf16 vectors
  const auto aligned = [](const void* ptr, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(ptr) & (bytes - 1)) == 0; };
  DDPO_REQUIRE(aligned(a->out_f32, 16) && aligned(a->residual, 16) && aligned(a->bias, 16) && aligned(a->rowvec, 16) &&
                   aligned(a->gn_stats, 8) && aligned(a->out_bf16, 8) && aligned(a->aux_bf16, 8),
               "ddpo_igemm: out_f32 / residual / bias / rowvec must be 16-byte aligned, out_bf16 / aux_bf16 / gn_stats 8-byte aligned");
  DDPO_REQUIRE(p.ld_out % 4 == 0 && p.ld_res % 4 == 0 && (a->rowvec == nullptr || a->rowvec_ld % 4 == 0),
               "ddpo_igemm: ld_out (%d), ld_res (%d) and rowvec_ld (%d) must be multiples of 4", p.ld_out, p.ld_res, a->rowvec_ld);
  if (a->gn_stats != nullptr)
    DDPO_REQUIRE(a->out_f32 != nullptr && !a->geglu && !a->accumulate_out,
                 "ddpo_igemm: gn_stats describes a plain fp32 output (no GEGLU, no accumulate)");
  return tile->launch(p, stream);
}

extern "C" int ddpo_igemm_plan(int m, int n, int k, int geglu, int bm_override, int bn_override, int* plan) {
  DDPO_REQUIRE(plan != nullptr && m > 0 && n > 0 && k > 0, "ddpo_igemm_plan: bad arguments");
  const TileShape* tile = pick_tile(m, n, k, geglu, bm_override, bn_override);
  DDPO_REQUIRE(tile != nullptr, "ddpo_igemm_plan: no %d x %d tile for N=%d", bm_override, bn_override, n);
  plan[0] = tile->bm, plan[1] = tile->bn, plan[2] = tile->ctas_per_sm, plan[3] = tile->stages;
  return DDPO_OK;
}
