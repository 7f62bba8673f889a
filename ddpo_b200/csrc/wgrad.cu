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
// One CTA = 128 input channels (two consumer warpgroups of 64) x BN output channels; warp 8 is the TMA producer.
// Pixels are split into `splits` fixed ranges to fill the machine; partial tiles go to a workspace
// and are summed in split order by a second kernel (deterministic, no atomics).
#include "common.cuh"
#include "wgmma.cuh"

namespace ddpo {

constexpr int WG_THREADS = 288;                    // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int WG_BKP = 64;                         // pixels per pipeline stage
constexpr int WG_BOX_BYTES = WG_BKP * 64 * 2;      // [64 pixels x 64 channels] bf16 = 8 KB
constexpr int WG_A_BYTES = 2 * WG_BOX_BYTES;       // 128 input channels
constexpr int WG_SMEM_BUDGET = 227 * 1024 - 1024 - 256;

struct WgradKArgs {
  CUtensorMap tmX0, tmX1, tmDY;
  int c0, c1, n;              // input channels per source, output channels
  int taps, is_conv, W, H, conv_stride, pad;
  int splits, pblocks_per_split, pblocks;
  int mt_per_tap0, mt_per_tap1;  // 128-channel blocks per source
  int n_begin, NT;            // this launch: NT column tiles of BN from column n_begin
  int stages;
  float* dst;                 // splits == 1: dW (+=) ; else workspace [splits][rows][n]
  int accumulate;
};

template <int BN>
__global__ void __launch_bounds__(WG_THREADS, 1) wgrad_kernel(const __grid_constant__ WgradKArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int SB = WG_A_BYTES + BN * 128;
  const int stages = p.stages;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + stages * SB);
  uint64_t* empty_bar = full_bar + stages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // tile -> (split, tap, source, channel block, n tile)
  const int mt_per_tap = p.mt_per_tap0 + p.mt_per_tap1;
  const int MT = p.taps * mt_per_tap;
  const int tile = blockIdx.x;
  const int nt = tile % p.NT;
  const int mt = (tile / p.NT) % MT;
  const int s = tile / p.NT / MT;
  const int tap = mt / mt_per_tap;
  const int mb = mt % mt_per_tap;
  const int src = mb >= p.mt_per_tap0;
  const int blk = src ? mb - p.mt_per_tap0 : mb;
  const int ncol0 = p.n_begin + nt * BN;
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

  if (warp == 8) {
    if (lane == 0) {
      prefetch_tmap(&p.tmX0);
      prefetch_tmap(&p.tmX1);
      prefetch_tmap(&p.tmDY);
      const int HW = p.W * p.H;
      int dy = 0, dx = 0;
      if (p.taps == 9) dy = tap / 3, dx = tap - dy * 3;
      const CUtensorMap* tmX = src ? &p.tmX1 : &p.tmX0;
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
          const int cx = dx - p.pad, cy = h0 * p.conv_stride + dy - p.pad;
          tma_load_4d(sA, tmX, &full_bar[stage], blk * 128, cx, cy, b0);
          tma_load_4d(sA + WG_BOX_BYTES, tmX, &full_bar[stage], blk * 128 + 64, cx, cy, b0);
        } else {
          tma_load_2d(sA, tmX, &full_bar[stage], blk * 128, row0);
          tma_load_2d(sA + WG_BOX_BYTES, tmX, &full_bar[stage], blk * 128 + 64, row0);
        }
        for (int j = 0; j < BN / 64; ++j) tma_load_2d(sB + j * WG_BOX_BYTES, &p.tmDY, &full_bar[stage], ncol0 + j * 64, row0);
        if (++stage == stages) stage = 0, phase ^= 1;
      }
    }
    return;
  }

  const int wg = warp >> 2;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  {
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int pb = pb0; pb < pb1; ++pb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_base = smem_u32(smem + stage * SB) + wg * WG_BOX_BYTES;
      const uint32_t b_base = smem_u32(smem + stage * SB) + WG_A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < WG_BKP / 16; ++k)  // 16 pixels = 16 rows of 128 B
        Wgmma<BN>::template ss<1, 1>(acc, gmma_desc(a_base + k * 2048, WG_BOX_BYTES, 1024),
                                     gmma_desc(b_base + k * 2048, WG_BOX_BYTES, 1024), (pb > pb0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
      if (pb > pb0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == stages) stage = 0, phase ^= 1;
    }
    wgmma_wait<0>();
  }

  // accumulator fragment: rows (input channels) r0 and r0 + 8, columns 8 j + 2 (lane & 3) + {0, 1}
  const int cin = p.c0 + p.c1;
  const int csrc = src ? p.c1 : p.c0;
  const size_t rows_total = static_cast<size_t>(p.taps) * cin;
  float* base = p.dst + (p.splits > 1 ? static_cast<size_t>(s) * rows_total * p.n : 0) + ncol0 + 2 * (lane & 3);
  const bool acc_old = p.splits == 1 && p.accumulate;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int ch = blk * 128 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;  // input channel within the source
    if (ch >= csrc) continue;
    float* d = base + (static_cast<size_t>(tap) * cin + (src ? p.c0 : 0) + ch) * p.n;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      float2 o = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
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

}  // namespace ddpo

using namespace ddpo;

static int wgrad_plan(const ddpo_wgrad_args* a, int* splits, int* pblocks) {
  const int m = a->is_conv ? a->batch * a->h * a->w : a->m;
  const int pb = (m + WG_BKP - 1) / WG_BKP;
  const int cin = a->c0 + a->c1;
  const int mt = a->taps * ((a->c0 + 127) / 128 + (a->c1 + 127) / 128);
  const int nt = a->n / 256 + (a->n % 256 != 0);
  const int tiles = mt * nt;
  // fill ~2 waves of CTAs, keep >= 8 pixel blocks per split, bound the workspace
  int s = (2 * num_sms() + tiles - 1) / tiles;
  if (s > pb / 8) s = pb / 8;
  if (s < 1) s = 1;
  const int64_t wsz = static_cast<int64_t>(a->taps) * cin * a->n;
  while (s > 1 && wsz * s > (int64_t(48) << 20)) --s;  // <= 48M floats of partials
  *splits = s;
  *pblocks = pb;
  return 0;
}

template <int BN>
static int wgrad_launch(WgradKArgs p, int n_begin, int nt, cudaStream_t stream) {
  constexpr int SB = WG_A_BYTES + BN * 128;
  p.n_begin = n_begin, p.NT = nt;
  p.stages = WG_SMEM_BUDGET / SB;
  if (p.stages > 8) p.stages = 8;
  const size_t smem = (size_t)p.stages * SB + 256 + 1024;
  static bool attr = false;
  if (!attr) {
    DDPO_CUDA_OK(cudaFuncSetAttribute(wgrad_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr = true;
  }
  const int tiles = p.splits * p.taps * (p.mt_per_tap0 + p.mt_per_tap1) * nt;
  wgrad_kernel<BN><<<tiles, WG_THREADS, smem, stream>>>(p);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}

extern "C" int64_t ddpo_wgrad_workspace_floats(const ddpo_wgrad_args* a) {
  int s, pb;
  wgrad_plan(a, &s, &pb);
  return s > 1 ? static_cast<int64_t>(s) * a->taps * (a->c0 + a->c1) * a->n : 0;
}

extern "C" int ddpo_wgrad(const ddpo_wgrad_args* a, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DDPO_REQUIRE(a && a->dy && a->x0 && a->dw, "wgrad: null pointer");
  DDPO_REQUIRE(a->c0 % 64 == 0 && a->c1 % 64 == 0 && a->n % 64 == 0, "wgrad: channels must be multiples of 64");
  DDPO_REQUIRE(a->taps == 1 || a->taps == 9, "wgrad: taps must be 1 or 9");
  DDPO_REQUIRE((reinterpret_cast<uintptr_t>(a->dw) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->workspace) & 15) == 0,
               "wgrad: dw and workspace must be 16-byte aligned (the split reduction loads and stores float4)");
  WgradKArgs p;
  memset(&p, 0, sizeof(p));
  int splits, pblocks;
  wgrad_plan(a, &splits, &pblocks);
  const int64_t need = ddpo_wgrad_workspace_floats(a);
  DDPO_REQUIRE(need == 0 || (a->workspace != nullptr && a->workspace_floats >= need),
               "wgrad: workspace too small (%lld < %lld floats)", (long long)a->workspace_floats, (long long)need);
  int M;
  if (a->is_conv) {
    const int W = a->w, H = a->h, B = a->batch, s = a->conv_stride;
    DDPO_REQUIRE((W & (W - 1)) == 0 && (H & (H - 1)) == 0 && W <= 64, "wgrad: W,H powers of two, W <= 64");
    M = B * W * H;
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
    M = a->m;
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
  p.pblocks = pblocks, p.splits = splits;
  p.pblocks_per_split = (pblocks + splits - 1) / splits;
  p.mt_per_tap0 = (a->c0 + 127) / 128, p.mt_per_tap1 = (a->c1 + 127) / 128;
  p.dst = splits > 1 ? a->workspace : a->dw;
  p.accumulate = 1;
  // 256-wide column tiles, then one launch for the remainder (64 / 128 / 192 columns)
  const int n_main = a->n / 256 * 256, rem = a->n - n_main;
  int rc = DDPO_OK;
  if (n_main > 0 && (rc = wgrad_launch<256>(p, 0, n_main / 256, stream))) return rc;
  if (rem == 64) rc = wgrad_launch<64>(p, n_main, 1, stream);
  else if (rem == 128) rc = wgrad_launch<128>(p, n_main, 1, stream);
  else if (rem == 192) rc = wgrad_launch<192>(p, n_main, 1, stream);
  if (rc) return rc;
  if (splits > 1) {
    const int64_t n4 = static_cast<int64_t>(a->taps) * (a->c0 + a->c1) * a->n / 4;
    int blocks = static_cast<int>((n4 + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    wgrad_reduce_kernel<<<blocks, 256, 0, stream>>>(a->workspace, a->dw, n4, splits, 1);
    DDPO_LAUNCH_OK();
  }
  return DDPO_OK;
}
