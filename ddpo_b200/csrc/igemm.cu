// Implicit-GEMM convolution / linear layer on wgmma (sm_90a).
//
//   out[m, n] = epilogue( sum_{tap, c} A[(b, y*s+dy-p, x*s+dx-p), c] * Wt[n, (tap, c)] )
//
// replaces every dense contraction of the Flax U-Net the reference runs through
// `unet.apply` (reference call sites: pipeline_flax_stable_diffusion.py:219-224,
// training/policy_gradient.py:87-102): nn.Conv 3x3 / 3x3 stride-2 / 1x1 and nn.Dense.
//
// Design:
//  * one CTA per 128 x BN output tile (n fastest, so the 128-row activation tile of consecutive CTAs is re-used out
//    of L2); BN is a template parameter because it is the N of the wgmma instruction;
//  * warp 8 = TMA producer.  The activation operand is fetched straight from the NHWC bf16 tensor with a 4-D tiled
//    tensor map whose box is (64 ch, bw, bh, bb) pixels; the 3x3 taps are the same box shifted by (dx-1, dy-1) and
//    TMA's out-of-bounds zero fill IS the conv padding -> no im2col buffer ever exists.  Channel-concatenated inputs
//    (U-Net skip connections) are two tensor maps walked back to back.  Stages of a multi-stage ring are handed over
//    through full / empty mbarriers;
//  * warps 0-7 = two consumer warpgroups, 64 rows each: m64nBNk16 bf16 wgmma from shared memory (both operands
//    K-major, 128-byte swizzle), fp32 accumulators in registers, one k-block of wgmma in flight while the next is
//    issued;
//  * epilogue: the accumulators go through shared memory (the drained stage ring) so that every global access of the
//    fused bias / per-sample time-embedding row vector / fp32 residual / GEGLU / slab statistics is coalesced;
//  * K order is fixed and independent of the batch size, of the tile width and of the position of a row in its
//    tile -> results are batch-invariant and bit-reproducible (the PPO ratio of an unchanged policy must be exactly 1;
//    reference config/base.py:88 clip 1e-4).
#include "common.cuh"
#include "wgmma.cuh"

namespace ddpo {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_TILE_BYTES = BM * BK * 2;
constexpr int IGEMM_THREADS = 288;  // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int IGEMM_CONSUMERS = 256;
constexpr int SMEM_BUDGET = 227 * 1024 - 1024 /*align slack*/ - 256 /*barriers*/;

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

template <int BN>
constexpr int igemm_stage_bytes() { return A_TILE_BYTES + BN * BK * 2; }
template <int BN>
constexpr int igemm_epi_bytes() { return BM * (BN + 4) * 4; }  // fp32 tile, rows padded by 16 B against bank conflicts

__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ uint2 pack_bf16x4(float4 v) { return make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w)); }

template <int BN>
__global__ void __launch_bounds__(IGEMM_THREADS, BN <= 128 ? 2 : 1) igemm_kernel(const __grid_constant__ IGemmArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int SB = igemm_stage_bytes<BN>();
  constexpr int EPI = igemm_epi_bytes<BN>();
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
      mbar_init(&empty_bar[i], IGEMM_CONSUMERS / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
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
        w0 = m0 % p.W;  // non-zero only when a pixel row is wider than a tile (W > 128)
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
  named_barrier(1, IGEMM_CONSUMERS);  // every operand stage has been read: the ring becomes the epilogue tile

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
  named_barrier(1, IGEMM_CONSUMERS);
  const int tid = threadIdx.x;
  if (p.geglu) {
    // GEGLU: this N tile is [BN/2 linear | BN/2 gate] columns of the same output channels (host-side row permutation):
    // out = lin * gelu_tanh(gate) -> out_bf16[:, tn*BN/2 + c], pre-activations (training) -> aux[:, n0 + c] / [n0 + BN/2 + c]
    constexpr int HALF = BN / 2, H4 = HALF / 4;
    for (int idx = tid; idx < BM * H4; idx += IGEMM_CONSUMERS) {
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
  for (int idx = tid; idx < BM * C4; idx += IGEMM_CONSUMERS) {
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
  named_barrier(1, IGEMM_CONSUMERS);
  // slab statistics: per 32-row slab and column, (sum, sum of squares) over the rows in order -- a function of the 32
  // values only
  for (int idx = tid; idx < (BM / 32) * BN; idx += IGEMM_CONSUMERS) {
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

// Tile width BN (the wgmma N).  The K order of every output element is the same for every width, so the width is a pure
// scheduling choice and depends on N only: 128 where it divides N (two 64 x 128 fp32 accumulator blocks per CTA leave
// room for a deep operand ring), otherwise the widest divisor of N among 160 / 192 / 96 / 64 / 32 (N = 320, 960, ...).
// GEGLU tiles hold [BN/2 linear | BN/2 gate] and must match the weight permutation (ddpo_prep_weight geglu_bn).
static int pick_width(int N, int geglu) {
  if (geglu) {
    for (int w : {256, 192, 128, 64})
      if (N % w == 0) return w;
    return 0;
  }
  for (int w : {128, 160, 192, 96, 64, 32})
    if (N % w == 0) return w;
  return 0;
}

template <int BN>
static int igemm_launch(IGemmArgs& p, cudaStream_t stream) {
  constexpr int SB = igemm_stage_bytes<BN>();
  constexpr int EPI = igemm_epi_bytes<BN>();
  // Three or more stages in half the shared memory: two CTAs per SM, so that one CTA's epilogue overlaps the other's
  // main loop.  Otherwise one CTA with as many stages as fit.
  int stages = (110 * 1024) / SB;
  if (BN > 128 || stages < 3 || stages * SB < EPI) stages = SMEM_BUDGET / SB;
  if (stages > 8) stages = 8;
  DDPO_REQUIRE(stages >= 2, "ddpo_igemm: not enough shared memory for BN=%d", BN);
  p.stages = stages;
  const size_t smem = (size_t)(stages * SB > EPI ? stages * SB : EPI) + 256 + 1024;
  static bool attr_set = false;
  if (!attr_set) {
    DDPO_CUDA_OK(cudaFuncSetAttribute(igemm_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  const int tiles = ((p.M_total + BM - 1) / BM) * (p.N_total / BN);
  igemm_kernel<BN><<<tiles, IGEMM_THREADS, smem, stream>>>(p);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
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
  const int BN = a->bn_override > 0 ? a->bn_override : pick_width(a->n, a->geglu);
  DDPO_REQUIRE(BN == 32 || BN == 64 || BN == 96 || BN == 128 || BN == 160 || BN == 192 || BN == 256,
               "ddpo_igemm: unsupported tile width %d", BN);
  DDPO_REQUIRE(a->n % BN == 0, "ddpo_igemm: no valid BN for N=%d", a->n);
  if (a->geglu) DDPO_REQUIRE(BN % 64 == 0 && a->out_bf16 != nullptr && a->bias != nullptr, "ddpo_igemm: bad GEGLU config");

  IGemmArgs p;
  memset(&p, 0, sizeof(p));
  const int ktot = a->taps * (cin0 + cin1);
  int M_total;
  if (a->is_conv) {
    // output grid W x H per sample (input grid is stride x larger)
    const int W = a->w, H = a->h, B = a->batch, s = a->conv_stride;
    DDPO_REQUIRE(s == 1 || s == 2, "ddpo_igemm: stride must be 1 or 2");
    DDPO_REQUIRE(W > 0 && H > 0 && (W & (W - 1)) == 0 && (H & (H - 1)) == 0 && W <= 1024,
                 "ddpo_igemm: W,H must be powers of two, W<=1024 (W=%d H=%d)", W, H);
    // a 128-row tile is bb samples x bh rows x bw pixels; rows wider than the tile are cut into W/128 tiles (with
    // stride 2 the 128-pixel box spans 256 input elements, the TMA limit)
    int bw = W < BM ? W : BM, bh = (BM / bw < H) ? BM / bw : H;
    int bb = BM / (bw * bh);
    M_total = B * W * H;
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
    M_total = a->m;
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
  switch (BN) {
    case 32: return igemm_launch<32>(p, stream);
    case 64: return igemm_launch<64>(p, stream);
    case 96: return igemm_launch<96>(p, stream);
    case 128: return igemm_launch<128>(p, stream);
    case 160: return igemm_launch<160>(p, stream);
    case 192: return igemm_launch<192>(p, stream);
    default: return igemm_launch<256>(p, stream);
  }
}
