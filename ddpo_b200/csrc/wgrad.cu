// Weight-gradient GEMM on wgmma (sm_90a):  dW[(tap, c_in), c_out] += sum_pixels X[pixel + tap, c_in] * dY[pixel, c_out]
//
// Backward of nn.Conv / nn.Dense of the 3P Flax U-Net w.r.t. their kernels -- the part of
// `jax.grad(compute_loss)` (reference ddpo/training/policy_gradient.py:138) that XLA emits as
// conv_general_dilated / dot_general transposes.  Output is written straight in the Flax
// parameter layout (HWIO == [(tap, c_in), c_out]; Dense [in, out]) and ACCUMULATED into the flat
// fp32 gradient buffer, so `grad_acc += g` (AccumulatingTrainState, :44-47) costs no extra pass.
//
// The reduction (wgmma K) dimension is the pixel index, which is the slow dimension of both NHWC
// operands -> both operands are "MN-major": TMA boxes of [64 pixels x 64 channels] land as
// 128-byte rows (SWIZZLE_128B) and are consumed through transposed wgmma descriptors
// (LBO = 8 KB between 64-channel boxes, SBO = 1 KB between 8-pixel groups).  As in the forward
// kernel the 3x3 taps are shifted boxes with TMA zero fill as padding.
// The rows of dW, (tap, c_in) flattened, are cut into 64-row units (c0 and c1 are multiples of 64).  One CTA = two
// consumer warpgroups, each with a unit of its own (so a CTA may straddle a tap or a source boundary), x BN output
// channels; warp 8 is the TMA producer.  BN = 320 keeps 160 accumulators per thread, more than the 168 registers a
// 288-thread CTA may hold allow: it runs a whole producer warpgroup (384 threads) that hands its registers to the
// consumers (setmaxnreg).  When the unit count is odd, the second warpgroup of the last CTA row has no
// unit: it multiplies a copy of the first one's box and stores nothing.
// Pixels are split into `splits` fixed ranges to fill the machine; partial tiles go to a workspace
// and are summed in split order by a second kernel (deterministic, no atomics).  `pick_wgrad_plan` chooses BN and the
// split count from the shape.
#include "common.cuh"
#include "gemm_model.cuh"
#include "wgmma.cuh"

namespace ddpo {

constexpr int WG_THREADS = 288;                    // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int WG_THREADS_WIDE = 384;               // BN = 320: warps 8-11 are the producer warpgroup
constexpr int WG_BKP = 64;                         // pixels per pipeline stage
constexpr int WG_BOX_BYTES = WG_BKP * 64 * 2;      // [64 pixels x 64 channels] bf16 = 8 KB
constexpr int WG_A_BYTES = 2 * WG_BOX_BYTES;       // the two warpgroups' 64-row units
constexpr int WG_SMEM_BUDGET = 227 * 1024 - 1024 - 256;

struct WgradKArgs {
  CUtensorMap tmX0, tmX1, tmDY;
  int c0, c1, n;              // input channels per source, output channels
  int taps, is_conv, W, H, conv_stride, pad;
  int splits, pblocks_per_split, pblocks;
  int units;                  // 64-row units of dW: taps * (c0 + c1) / 64
  int NT;                     // column tiles of BN
  int stages;
  float* dst;                 // splits == 1: dW (+=) ; else workspace [splits][rows][n]
};

template <int BN>
constexpr int wgrad_threads() { return BN > 256 ? WG_THREADS_WIDE : WG_THREADS; }

template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(N)); }

// BN = 320 runs an m64n256k16 and an m64n64k16 per k16 step, into two accumulator arrays.
template <int BN>
__global__ void __launch_bounds__(wgrad_threads<BN>(), 1) wgrad_kernel(const __grid_constant__ WgradKArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int BN1 = BN > 256 ? 256 : BN, BN2 = BN - BN1;
  constexpr int SB = WG_A_BYTES + BN * 128;
  const int stages = p.stages;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + stages * SB);
  uint64_t* empty_bar = full_bar + stages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // tile -> (split, CTA row of two units, n tile)
  const int MT = (p.units + 1) / 2;
  const int tile = blockIdx.x;
  const int nt = tile % p.NT;
  const int mt = (tile / p.NT) % MT;
  const int s = tile / p.NT / MT;
  const int ncol0 = nt * BN;
  const int pb0 = s * p.pblocks_per_split;
  const int pb1 = min(p.pblocks, pb0 + p.pblocks_per_split);

  if (threadIdx.x == 0) {
    for (int i = 0; i < stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    if constexpr (BN > 256) setmaxnreg_dec<40>();
    if (warp == 8 && lane == 0) {
      prefetch_tmap(&p.tmX0);
      prefetch_tmap(&p.tmX1);
      prefetch_tmap(&p.tmDY);
      const int HW = p.W * p.H;
      const int upt = (p.c0 + p.c1) / 64;  // units per tap
      // each box: its source, first channel within the source and tap offset (the ghost unit reads the first one's)
      const CUtensorMap* tmX[2];
      int ch[2], cx[2], cy[2];
      for (int b = 0; b < 2; ++b) {
        const int u = min(2 * mt + b, p.units - 1);
        const int tap = u / upt, c = (u - tap * upt) * 64;
        const int src = c >= p.c0;
        tmX[b] = src ? &p.tmX1 : &p.tmX0;
        ch[b] = src ? c - p.c0 : c;
        const int dy = p.taps == 9 ? tap / 3 : 0, dx = p.taps == 9 ? tap % 3 : 0;
        cx[b] = dx - p.pad, cy[b] = dy - p.pad;
      }
      int stage = 0;
      uint32_t phase = 0;
      for (int pb = pb0; pb < pb1; ++pb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sA = smem + stage * SB;
        uint8_t* sB = sA + WG_A_BYTES;
        const int row0 = pb * WG_BKP;
        mbar_expect_tx(&full_bar[stage], SB);
        if (p.is_conv) {
          const int b0 = row0 / HW, h0 = (row0 % HW) / p.W;
          for (int b = 0; b < 2; ++b)
            tma_load_4d(sA + b * WG_BOX_BYTES, tmX[b], &full_bar[stage], ch[b], cx[b], h0 * p.conv_stride + cy[b], b0);
        } else {
          for (int b = 0; b < 2; ++b) tma_load_2d(sA + b * WG_BOX_BYTES, tmX[b], &full_bar[stage], ch[b], row0);
        }
        for (int j = 0; j < BN / 64; ++j) tma_load_2d(sB + j * WG_BOX_BYTES, &p.tmDY, &full_bar[stage], ncol0 + j * 64, row0);
        if (++stage == stages) stage = 0, phase ^= 1;
      }
    }
    return;
  }

  if constexpr (BN > 256) setmaxnreg_inc<232>();
  const int wg = warp >> 2;
  float acc[BN1 / 2];
  float acc2[BN2 > 0 ? BN2 / 2 : 1];
#pragma unroll
  for (int i = 0; i < BN1 / 2; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < BN2 / 2; ++i) acc2[i] = 0.f;
  {
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    bool hung = false;
    for (int pb = pb0; pb < pb1; ++pb) {
      if (!mbar_wait_timed(&full_bar[stage], phase)) {
        hung = true;
        break;
      }
      const uint32_t a_base = smem_u32(smem + stage * SB) + wg * WG_BOX_BYTES;
      const uint32_t b_base = smem_u32(smem + stage * SB) + WG_A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < WG_BKP / 16; ++k) {  // 16 pixels = 16 rows of 128 B
        const uint64_t da = gmma_desc(a_base + k * 2048, WG_BOX_BYTES, 1024);
        const uint32_t scale_d = (pb > pb0 || k > 0) ? 1u : 0u;
        Wgmma<BN1>::template ss<1, 1>(acc, da, gmma_desc(b_base + k * 2048, WG_BOX_BYTES, 1024), scale_d);
        if constexpr (BN2 > 0)
          Wgmma<BN2>::template ss<1, 1>(acc2, da, gmma_desc(b_base + (BN1 / 64) * WG_BOX_BYTES + k * 2048, WG_BOX_BYTES, 1024),
                                        scale_d);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (pb > pb0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == stages) stage = 0, phase ^= 1;
    }
    wgmma_wait<0>();
    if (hung) __trap();
  }

  // accumulator fragment: rows r0 and r0 + 8 of the warpgroup's unit, columns 8 j + 2 (lane & 3) + {0, 1}
  const int u = 2 * mt + wg;
  if (u >= p.units) return;
  const size_t rows_total = static_cast<size_t>(p.units) * 64;
  float* base = p.dst + (p.splits > 1 ? static_cast<size_t>(s) * rows_total * p.n : 0) + ncol0 + 2 * (lane & 3);
  const bool acc_old = p.splits == 1;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = u * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    float* d = base + static_cast<size_t>(row) * p.n;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      float2 o = j < BN1 / 8 ? make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1])
                             : make_float2(acc2[4 * (j - BN1 / 8) + 2 * h], acc2[4 * (j - BN1 / 8) + 2 * h + 1]);
      float2* dp = reinterpret_cast<float2*>(d + 8 * j);
      if (acc_old) {
        const float2 old = *dp;
        o.x += old.x, o.y += old.y;
      }
      *dp = o;
    }
  }
}

__global__ void wgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ dw, int64_t n4, int splits,
                                    int accumulate) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float4 acc = accumulate ? reinterpret_cast<const float4*>(dw)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < splits; ++s) {
      const float4 v = reinterpret_cast<const float4*>(part)[static_cast<int64_t>(s) * n4 + i];
      acc.x += v.x, acc.y += v.y, acc.z += v.z, acc.w += v.w;
    }
    reinterpret_cast<float4*>(dw)[i] = acc;
  }
}

// ------------------------------------------------------------------------------------------------ planning ----
constexpr int WG_WIDTHS[] = {320, 256, 192, 128, 64};  // widest first: a tie in the cost model re-reads X least
constexpr int WG_MIN_PBLOCKS_PER_SPLIT = 8;
// Bounds the workspace, which the U-Net keeps for the whole train pass: 14 745 600 floats (59 MB) is the largest one the
// SD2-base train pass needed when splits were sized for two waves of 256-wide tiles (2 splits of the 640 -> 1280 3x3
// convolution at 16x16), so peak memory does not grow.
constexpr int64_t WG_MAX_PARTIAL_FLOATS = 14745600;

template <int BN>
constexpr int wgrad_stages() {
  constexpr int SB = WG_A_BYTES + BN * 128;
  return WG_SMEM_BUDGET / SB < 8 ? WG_SMEM_BUDGET / SB : 8;
}

struct WgradPlan {
  int bn, splits;
};

// Modelled makespan (SM clock cycles, gemm_model.cuh) of a launch of `ctas` CTAs of 128 rows x bn that each run
// `per_cta` pixel blocks (4 k16 steps each), plus, with splits, the partial stores and the reduction over
// `rows` x n floats, at HBM rate.
static double wgrad_makespan(int bn, int splits, int per_cta, long long ctas, long long rows, int n) {
  const double cta = per_cta * 4.0 * k16_step_clk(128, bn) + 128.0 * bn * 8.0 / HBM_BYTES_PER_CLK;
  const double waves = double((ctas + NUM_SMS - 1) / NUM_SMS);
  const double reduce = splits > 1 ? (splits + 2.0) * rows * n * 4.0 / (HBM_BYTES_PER_CLK * NUM_SMS) : 0.0;
  return waves * cta + reduce;
}

// The column-tile width and pixel split count of a weight gradient over m pixels: a function of the shape alone, so a
// layer always sums its pixels in the same order.  Every width that divides n and every split count that keeps at
// least 8 pixel blocks per split and at most WG_MAX_PARTIAL_FLOATS partial floats is a candidate; the one with the
// least modelled makespan wins.  bn / splits > 0 force that width / split count (tests, micro-benchmarks).  {0, 0} when
// nothing fits.
static WgradPlan pick_wgrad_plan(int m, int c0, int c1, int n, int taps, int bn, int splits) {
  const int pb = (m + WG_BKP - 1) / WG_BKP;
  const long long rows = static_cast<long long>(taps) * (c0 + c1);
  const long long mt = (rows / 64 + 1) / 2;
  int max_s = pb / WG_MIN_PBLOCKS_PER_SPLIT;
  while (max_s > 1 && rows * n * max_s > WG_MAX_PARTIAL_FLOATS) --max_s;
  if (max_s < 1) max_s = 1;
  WgradPlan best = {0, 0};
  double best_time = 0.0;
  for (int w : WG_WIDTHS) {
    if (n % w != 0 || (bn > 0 && w != bn)) continue;
    for (int s = splits > 0 ? splits : 1; s <= (splits > 0 ? splits : max_s); ++s) {
      const int per = (pb + s - 1) / s;
      const int used = splits > 0 ? s : (pb + per - 1) / per;  // no empty trailing split
      if (used != s) continue;
      const double t = wgrad_makespan(w, s, per, mt * (n / w) * s, rows, n);
      if (best.bn == 0 || t < best_time) best = {w, s}, best_time = t;
    }
  }
  return best;
}

template <int BN>
static int wgrad_launch(WgradKArgs p, cudaStream_t stream) {
  constexpr int SB = WG_A_BYTES + BN * 128;
  p.NT = p.n / BN;
  p.stages = wgrad_stages<BN>();
  const size_t smem = (size_t)p.stages * SB + 256 + 1024;
  static bool attr = false;
  if (!attr) {
    DDPO_CUDA_OK(cudaFuncSetAttribute(wgrad_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr = true;
  }
  const int tiles = p.splits * ((p.units + 1) / 2) * p.NT;
  wgrad_kernel<BN><<<tiles, wgrad_threads<BN>(), smem, stream>>>(p);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

}  // namespace ddpo

using namespace ddpo;

static int wgrad_pixels(const ddpo_wgrad_args* a) { return a->is_conv ? a->batch * a->h * a->w : a->m; }

static WgradPlan wgrad_plan_of(const ddpo_wgrad_args* a) {
  return pick_wgrad_plan(wgrad_pixels(a), a->c0, a->c1, a->n, a->taps, a->bn_override, a->splits_override);
}

extern "C" int ddpo_wgrad_plan(int m, int c0, int c1, int n, int taps, int bn_override, int splits_override, int* plan) {
  DDPO_REQUIRE(plan != nullptr && m > 0 && c0 > 0 && c0 % 64 == 0 && c1 >= 0 && c1 % 64 == 0 && n > 0 && n % 64 == 0 &&
                   (taps == 1 || taps == 9),
               "ddpo_wgrad_plan: bad shape (m=%d c0=%d c1=%d n=%d taps=%d)", m, c0, c1, n, taps);
  DDPO_REQUIRE(splits_override >= 0 && splits_override <= (m + WG_BKP - 1) / WG_BKP,
               "ddpo_wgrad_plan: %d splits of %d pixels", splits_override, m);
  const WgradPlan w = pick_wgrad_plan(m, c0, c1, n, taps, bn_override, splits_override);
  DDPO_REQUIRE(w.bn != 0, "ddpo_wgrad_plan: no %d-wide tile for N=%d", bn_override, n);
  plan[0] = w.bn, plan[1] = w.splits;
  return DDPO_OK;
}

extern "C" int64_t ddpo_wgrad_workspace_floats(const ddpo_wgrad_args* a) {
  const WgradPlan w = wgrad_plan_of(a);
  return w.splits > 1 ? static_cast<int64_t>(w.splits) * a->taps * (a->c0 + a->c1) * a->n : 0;
}

extern "C" int ddpo_wgrad(const ddpo_wgrad_args* a, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DDPO_REQUIRE(a && a->dy && a->x0 && a->dw, "wgrad: null pointer");
  DDPO_REQUIRE(a->c0 > 0 && a->c0 % 64 == 0 && a->c1 % 64 == 0 && a->n % 64 == 0, "wgrad: channels must be multiples of 64");
  DDPO_REQUIRE(a->taps == 1 || a->taps == 9, "wgrad: taps must be 1 or 9");
  DDPO_REQUIRE((reinterpret_cast<uintptr_t>(a->dw) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->workspace) & 15) == 0,
               "wgrad: dw and workspace must be 16-byte aligned (the split reduction loads and stores float4)");
  const int M = wgrad_pixels(a);
  const int pblocks = (M + WG_BKP - 1) / WG_BKP;
  DDPO_REQUIRE(a->splits_override >= 0 && a->splits_override <= pblocks, "wgrad: %d splits of %d pixels",
               a->splits_override, M);
  const WgradPlan plan = wgrad_plan_of(a);
  DDPO_REQUIRE(plan.bn != 0, "wgrad: no %d-wide tile for N=%d", a->bn_override, a->n);
  const int64_t need = ddpo_wgrad_workspace_floats(a);
  DDPO_REQUIRE(need == 0 || (a->workspace != nullptr && a->workspace_floats >= need),
               "wgrad: workspace too small (%lld < %lld floats)", (long long)a->workspace_floats, (long long)need);
  WgradKArgs p;
  memset(&p, 0, sizeof(p));
  if (a->is_conv) {
    const int W = a->w, H = a->h, B = a->batch, s = a->conv_stride;
    DDPO_REQUIRE((W & (W - 1)) == 0 && (H & (H - 1)) == 0 && W <= 64, "wgrad: W,H powers of two, W <= 64");
    int bw = W, bh = (WG_BKP / W < H) ? WG_BKP / W : H;
    int bb = WG_BKP / (bw * bh);
    const int Wi = W * s, Hi = H * s;
    for (int src = 0; src < (a->c1 > 0 ? 2 : 1); ++src) {
      const int C = src ? a->c1 : a->c0;
      const int ld = src ? (a->ldx1 > 0 ? a->ldx1 : a->c1) : (a->ldx0 > 0 ? a->ldx0 : a->c0);
      uint64_t dims[4] = {(uint64_t)C, (uint64_t)Wi, (uint64_t)Hi, (uint64_t)B};
      uint64_t strides[3] = {(uint64_t)ld * 2, (uint64_t)ld * 2 * Wi, (uint64_t)ld * 2 * Wi * Hi};
      uint32_t box[4] = {64, (uint32_t)(bw * s), (uint32_t)(bh * s), (uint32_t)bb};
      uint32_t es[4] = {1, (uint32_t)s, (uint32_t)s, 1};
      int rc = make_tensor_map(src ? &p.tmX1 : &p.tmX0, src ? a->x1 : a->x0, 2, 4, dims, strides, box, es, 1);
      if (rc) return rc;
    }
    if (a->c1 == 0) p.tmX1 = p.tmX0;
    p.W = W, p.H = H, p.conv_stride = s, p.pad = a->taps == 9 ? 1 : 0;
  } else {
    DDPO_REQUIRE(a->taps == 1 && a->c1 == 0, "wgrad: linear mode takes one source, one tap");
    uint64_t dims[2] = {(uint64_t)a->c0, (uint64_t)M};
    uint64_t strides[1] = {(uint64_t)(a->ldx0 > 0 ? a->ldx0 : a->c0) * 2};
    uint32_t box[2] = {64, (uint32_t)WG_BKP};
    uint32_t es[2] = {1, 1};
    int rc = make_tensor_map(&p.tmX0, a->x0, 2, 2, dims, strides, box, es, 1);
    if (rc) return rc;
    p.tmX1 = p.tmX0;
    p.W = 1, p.H = 1, p.conv_stride = 1;
  }
  {
    uint64_t dims[2] = {(uint64_t)a->n, (uint64_t)M};
    uint64_t strides[1] = {(uint64_t)(a->ldy > 0 ? a->ldy : a->n) * 2};
    uint32_t box[2] = {64, (uint32_t)WG_BKP};
    uint32_t es[2] = {1, 1};
    int rc = make_tensor_map(&p.tmDY, a->dy, 2, 2, dims, strides, box, es, 1);
    if (rc) return rc;
  }
  p.c0 = a->c0, p.c1 = a->c1, p.n = a->n, p.taps = a->taps, p.is_conv = a->is_conv;
  p.pblocks = pblocks, p.splits = plan.splits;
  p.pblocks_per_split = (pblocks + plan.splits - 1) / plan.splits;
  p.units = a->taps * (a->c0 + a->c1) / 64;
  p.dst = plan.splits > 1 ? a->workspace : a->dw;
  int rc = DDPO_OK;
  switch (plan.bn) {
    case 64: rc = wgrad_launch<64>(p, stream); break;
    case 128: rc = wgrad_launch<128>(p, stream); break;
    case 192: rc = wgrad_launch<192>(p, stream); break;
    case 256: rc = wgrad_launch<256>(p, stream); break;
    default: rc = wgrad_launch<320>(p, stream); break;
  }
  if (rc) return rc;
  if (plan.splits > 1) {
    const int64_t n4 = static_cast<int64_t>(a->taps) * (a->c0 + a->c1) * a->n / 4;
    int blocks = static_cast<int>((n4 + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    wgrad_reduce_kernel<<<blocks, 256, 0, stream>>>(a->workspace, a->dw, n4, plan.splits, 1);
    DDPO_LAUNCH_OK();
  }
  return DDPO_OK;
}
