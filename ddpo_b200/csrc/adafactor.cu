// Adafactor update on the flat fp32 parameter / gradient buffers (HBM-bound).
//
// Restates optax.chain(clip_by_global_norm(max_norm), adafactor(lr, weight_decay_rate=wd)) with every other
// adafactor argument at its optax==0.1.5 default (reference pipeline/policy_gradient.py:132-150), fused with
// AccumulatingTrainState.apply_gradients(do_update=True).  Per parameter tensor p with gradient g:
//   g^ = clip_by_global_norm(grad_acc * grad_scale)            (same first stage as clip_adamw)
//   beta = 1 - step^-0.8 ; G = g^^2 + 1e-30
//   factored (ndim >= 2, second-largest dim >= min_dim_size_to_factor; the two largest dims are the last two,
//   so the tensor is taps independent row-major [R, C] matrices):
//     v_row = beta v_row + (1-beta) mean(G, d0) ; v_col = beta v_col + (1-beta) mean(G, d1)   (d1, d0 = argsort[-2:])
//     rcm = mean(v_row) per tap ; u = g^ (v_row / rcm)^-1/2 v_col^-1/2
//   unfactored: v = beta v + (1-beta) G ; u = g^ v^-1/2
//   u /= max(1, rms(u)) ; u *= lr ; u *= sqrt(max(mean(p^2), 1e-6)) ; u += wd p ; p -= u ; grad_acc = 0
// Note that wd is not multiplied by lr (optax's add_decayed_weights comes after the learning-rate scale).
//
// The host planner cuts every tensor into tiles (128 x 128 floats of one tap, or 1-D chunks of 16384 floats).  The
// update is five launches: (a) per tile, partial row / column sums of G and sum p^2 (unfactored tiles update v and
// their sum u^2 here); (b) per tensor-tap, v_row, v_col and rcm; (c) per factored tile, sum u^2; (d) per tensor, the
// block-RMS clip denominator and the parameter scale; (e) per tile, the update and the zeroing of grad_acc.  There
// are no atomics and every reduction order depends on the shapes only, so replicas stay bit-identical.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <numeric>
#include <vector>

#include "common.cuh"

namespace ddpo {
namespace {

constexpr int AF_TR = 128;         // factored tile rows
constexpr int AF_TC = 128;         // factored tile columns: 32 lanes x float4
constexpr int AF_CHUNK = 16384;    // unfactored tile length
constexpr int AF_THREADS = 256;
constexpr int AF_WARPS = AF_THREADS / 32;
constexpr int64_t AF_MAGIC = 0x4144414641435452LL;
constexpr float AF_EPS = 1e-30f;

// The plan is one int64 array: a header, then per tensor, per tile and per tensor-tap records.
enum { H_MAGIC, H_N, H_NTENSORS, H_NTILES, H_NTAPS, H_STATE, H_WS, H_WORDS = 8 };
// kind: 0 unfactored (R = numel, C = 1, taps = 1), 1 factored with v_row over rows (C >= R), 2 factored with v_row
// over columns (R > C).  sa / sb: state offsets of v_row / v_col, or of v and -1.
enum { T_OFFSET, T_NUMEL, T_KIND, T_TAPS, T_R, T_C, T_SA, T_SB, T_TILE0, T_NRT, T_NCT, T_TAP0, T_WORDS = 12 };
// tile: tensor (-1 for a tile that only zeroes trailing padding), tap, rows [r0, r0 + nr), columns [c0, c0 + nc),
// grad_acc padding [zlo, zhi) it zeroes, workspace offset of its TR row + TC column partial sums (-1 if none)
enum { L_TENSOR, L_TAP, L_R0, L_NR, L_C0, L_NC, L_ZLO, L_ZHI, L_PART, L_WORDS = 9 };
enum { P_TENSOR, P_TAP, P_WORDS = 2 };

struct AfArgs {
  float* p;
  float* g;
  float* state;
  float* ws;
  const int64_t* plan;
  const float* sumsq;  // of the UNSCALED accumulated gradient
  float grad_scale, max_norm, lr, wd, beta;
  float* norm_out;
  int ntensors, ntiles, ntaps;
  // workspace layout (floats): [ntensors][2] clip denominator and parameter scale, [ntaps] rcm, [ntiles][2] partial
  // sum p^2 and sum u^2, then the row / column partials of the factored tiles
  int64_t ws_rcm, ws_tile;
};

__device__ __forceinline__ const int64_t* tensor_rec(const AfArgs& a, int64_t t) { return a.plan + H_WORDS + t * T_WORDS; }
__device__ __forceinline__ const int64_t* tile_rec(const AfArgs& a, int64_t i) {
  return a.plan + H_WORDS + static_cast<int64_t>(a.ntensors) * T_WORDS + i * L_WORDS;
}
__device__ __forceinline__ const int64_t* tap_rec(const AfArgs& a, int64_t i) {
  return a.plan + H_WORDS + static_cast<int64_t>(a.ntensors) * T_WORDS + static_cast<int64_t>(a.ntiles) * L_WORDS +
         i * P_WORDS;
}

// optax.clip_by_global_norm, with the same arithmetic as clip_adamw_kernel
struct Clip {
  float scale, norm, max_norm;
  bool no_clip;
  __device__ __forceinline__ float operator()(float g) const {
    const float x = g * scale;
    return no_clip ? x : (x / norm) * max_norm;
  }
};
__device__ __forceinline__ Clip make_clip(const AfArgs& a) {
  Clip c;
  c.norm = a.grad_scale * sqrtf(a.sumsq[0]);
  c.scale = a.grad_scale, c.max_norm = a.max_norm, c.no_clip = c.norm < a.max_norm;
  return c;
}

// Sum over the block in a fixed order (warp tree, then the warps in order); the result is returned to every thread.
__device__ float block_sum(float v, float* sm) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  for (int i = 0; i < AF_WARPS; ++i) s += sm[i];
  return s;
}

__device__ __forceinline__ float sq_eps(float x) { return __fmul_rn(x, x) + AF_EPS; }

// Factored tile geometry shared by (a), (c) and (e): warp w takes rows w, w + 8, ...; lane l takes columns 4l .. 4l+3.
struct FTile {
  int64_t base;  // flat index of element (r0, c0) of the tile
  int64_t C;
  int nr, nc, col4;
  bool active;
};
__device__ __forceinline__ FTile ftile(const int64_t* T, const int64_t* L) {
  FTile f;
  f.C = T[T_C];
  f.base = T[T_OFFSET] + L[L_TAP] * T[T_R] * f.C + L[L_R0] * f.C + L[L_C0];
  f.nr = static_cast<int>(L[L_NR]), f.nc = static_cast<int>(L[L_NC]);
  f.col4 = (threadIdx.x & 31) * 4;
  f.active = f.col4 < f.nc;
  return f;
}

// Row and column factors of a factored tile: u = (g^ * a) * b with a from v_row, b from v_col (optax's order).
struct Factors {
  const float* vr;  // state vector over this tap's rows
  float fc[4];      // this lane's column factors
  float rcm;
  bool row_is_vrow;
};
__device__ __forceinline__ Factors load_factors(const AfArgs& a, const int64_t* T, const int64_t* L, const FTile& f) {
  Factors F;
  const int64_t k = L[L_TAP], R = T[T_R], C = T[T_C];
  F.row_is_vrow = T[T_KIND] == 1;
  F.rcm = a.ws[a.ws_rcm + T[T_TAP0] + k];
  const float* vrow = a.state + T[T_SA] + k * (F.row_is_vrow ? R : C);
  const float* vcol = a.state + T[T_SB] + k * (F.row_is_vrow ? C : R);
  F.vr = (F.row_is_vrow ? vrow : vcol) + L[L_R0];
  const float* vc = (F.row_is_vrow ? vcol : vrow) + L[L_C0];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float v = f.active ? vc[f.col4 + j] : 1.f;
    F.fc[j] = F.row_is_vrow ? rsqrtf(v) : rsqrtf(v / F.rcm);
  }
  return F;
}
__device__ __forceinline__ float row_factor(const Factors& F, int r) {
  const float v = F.vr[r];
  return F.row_is_vrow ? rsqrtf(v / F.rcm) : rsqrtf(v);
}
__device__ __forceinline__ float fact_u(const Factors& F, float gh, float fr, int j) {
  return F.row_is_vrow ? (gh * fr) * F.fc[j] : (gh * F.fc[j]) * fr;
}

// (a) per tile: partial sums of G by row and by column, sum p^2; unfactored tiles also update v and sum u^2
__global__ void __launch_bounds__(AF_THREADS) af_stats_kernel(const AfArgs a) {
  const Clip cl = make_clip(a);
  if (a.norm_out != nullptr && blockIdx.x == 0 && threadIdx.x == 0) a.norm_out[0] = cl.norm;
  const int64_t* L = tile_rec(a, blockIdx.x);
  if (L[L_TENSOR] < 0) return;
  const int64_t* T = tensor_rec(a, L[L_TENSOR]);
  __shared__ float red[AF_WARPS];
  __shared__ float colp[AF_WARPS][AF_TC];
  float* sums = a.ws + a.ws_tile + 2 * static_cast<int64_t>(blockIdx.x);
  float psq = 0.f;
  if (T[T_KIND] == 0) {
    const int64_t base = T[T_OFFSET] + L[L_R0];
    float* v = a.state + T[T_SA] + L[L_R0];
    const int n = static_cast<int>(L[L_NR]);
    float usq = 0.f;
    for (int i = threadIdx.x; i < n; i += AF_THREADS) {
      const float gh = cl(a.g[base + i]), p = a.p[base + i];
      const float vn = a.beta * v[i] + (1.f - a.beta) * sq_eps(gh);
      v[i] = vn;
      const float u = gh * rsqrtf(vn);
      psq += p * p;
      usq += u * u;
    }
    psq = block_sum(psq, red);
    usq = block_sum(usq, red);
    if (threadIdx.x == 0) sums[0] = psq, sums[1] = usq;
    return;
  }
  const FTile f = ftile(T, L);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* part = a.ws + L[L_PART];
  float cs[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 2
  for (int r = warp; r < f.nr; r += AF_WARPS) {
    float rs = 0.f;
    if (f.active) {
      const int64_t e = f.base + r * f.C + f.col4;
      const float4 g4 = *reinterpret_cast<const float4*>(a.g + e);
      const float4 p4 = *reinterpret_cast<const float4*>(a.p + e);
      const float G0 = sq_eps(cl(g4.x)), G1 = sq_eps(cl(g4.y)), G2 = sq_eps(cl(g4.z)), G3 = sq_eps(cl(g4.w));
      cs[0] += G0, cs[1] += G1, cs[2] += G2, cs[3] += G3;
      rs = (G0 + G1) + (G2 + G3);
      psq += (p4.x * p4.x + p4.y * p4.y) + (p4.z * p4.z + p4.w * p4.w);
    }
    rs = warp_sum(rs);
    if (lane == 0) part[r] = rs;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) colp[warp][f.col4 + j] = cs[j];
  __syncthreads();
  if (threadIdx.x < f.nc) {
    float s = 0.f;
    for (int w = 0; w < AF_WARPS; ++w) s += colp[w][threadIdx.x];
    part[AF_TR + threadIdx.x] = s;
  }
  psq = block_sum(psq, red);
  if (threadIdx.x == 0) sums[0] = psq;
}

// (b) per tensor-tap: v_row, v_col (means of G, then the EMA) and rcm = mean(v_row)
__global__ void __launch_bounds__(AF_THREADS) af_factor_kernel(const AfArgs a) {
  const int64_t* P = tap_rec(a, blockIdx.x);
  const int64_t* T = tensor_rec(a, P[P_TENSOR]);
  const int64_t k = P[P_TAP], R = T[T_R], C = T[T_C], nrt = T[T_NRT], nct = T[T_NCT];
  const bool row_is_vrow = T[T_KIND] == 1;
  const int64_t tile0 = T[T_TILE0] + k * nrt * nct;
  float* vrow = a.state + T[T_SA] + k * (row_is_vrow ? R : C);
  float* vcol = a.state + T[T_SB] + k * (row_is_vrow ? C : R);
  float* vr = row_is_vrow ? vrow : vcol;  // over rows
  float* vc = row_is_vrow ? vcol : vrow;  // over columns
  const float fR = static_cast<float>(R), fC = static_cast<float>(C);
  float vrow_sum = 0.f;
  for (int64_t r = threadIdx.x; r < R; r += AF_THREADS) {
    float s = 0.f;
    for (int64_t ct = 0; ct < nct; ++ct) s += a.ws[tile_rec(a, tile0 + (r / AF_TR) * nct + ct)[L_PART] + r % AF_TR];
    const float v = a.beta * vr[r] + (1.f - a.beta) * (s / fC);
    vr[r] = v;
    if (row_is_vrow) vrow_sum += v;
  }
  for (int64_t c = threadIdx.x; c < C; c += AF_THREADS) {
    float s = 0.f;
    for (int64_t rt = 0; rt < nrt; ++rt) s += a.ws[tile_rec(a, tile0 + rt * nct + c / AF_TC)[L_PART] + AF_TR + c % AF_TC];
    const float v = a.beta * vc[c] + (1.f - a.beta) * (s / fR);
    vc[c] = v;
    if (!row_is_vrow) vrow_sum += v;
  }
  __shared__ float red[AF_WARPS];
  const float s = block_sum(vrow_sum, red);
  if (threadIdx.x == 0) a.ws[a.ws_rcm + blockIdx.x] = s / (row_is_vrow ? fR : fC);
}

// (c) per factored tile: sum u^2 (a second read of g: u needs both new factors)
__global__ void __launch_bounds__(AF_THREADS) af_usq_kernel(const AfArgs a) {
  const int64_t* L = tile_rec(a, blockIdx.x);
  if (L[L_TENSOR] < 0) return;
  const int64_t* T = tensor_rec(a, L[L_TENSOR]);
  if (T[T_KIND] == 0) return;
  const Clip cl = make_clip(a);
  const FTile f = ftile(T, L);
  const Factors F = load_factors(a, T, L, f);
  float usq = 0.f;
  if (f.active) {
#pragma unroll 4
    for (int r = threadIdx.x >> 5; r < f.nr; r += AF_WARPS) {
      const float4 g4 = *reinterpret_cast<const float4*>(a.g + f.base + r * f.C + f.col4);
      const float fr = row_factor(F, r);
      const float u0 = fact_u(F, cl(g4.x), fr, 0), u1 = fact_u(F, cl(g4.y), fr, 1);
      const float u2 = fact_u(F, cl(g4.z), fr, 2), u3 = fact_u(F, cl(g4.w), fr, 3);
      usq += (u0 * u0 + u1 * u1) + (u2 * u2 + u3 * u3);
    }
  }
  __shared__ float red[AF_WARPS];
  usq = block_sum(usq, red);
  if (threadIdx.x == 0) a.ws[a.ws_tile + 2 * static_cast<int64_t>(blockIdx.x) + 1] = usq;
}

// (d) per tensor: clip denominator max(1, rms(u)) and parameter scale sqrt(max(mean(p^2), 1e-6))
__global__ void __launch_bounds__(128) af_tensor_kernel(const AfArgs a) {
  const int64_t* T = tensor_rec(a, blockIdx.x);
  const int64_t t0 = T[T_TILE0], nt = T[T_TAPS] * T[T_NRT] * T[T_NCT];
  double ps = 0.0, us = 0.0;
  for (int64_t i = threadIdx.x; i < nt; i += blockDim.x) {
    ps += a.ws[a.ws_tile + 2 * (t0 + i)];
    us += a.ws[a.ws_tile + 2 * (t0 + i) + 1];
  }
  __shared__ double sm[2][128];
  sm[0][threadIdx.x] = ps, sm[1][threadIdx.x] = us;
  __syncthreads();
  if (threadIdx.x == 0) {
    ps = 0.0, us = 0.0;
    for (int i = 0; i < static_cast<int>(blockDim.x); ++i) ps += sm[0][i], us += sm[1][i];
    const double numel = static_cast<double>(T[T_NUMEL]);
    a.ws[2 * blockIdx.x] = static_cast<float>(fmax(1.0, sqrt(us / numel)));
    a.ws[2 * blockIdx.x + 1] = static_cast<float>(sqrt(fmax(ps / numel, 1e-6)));
  }
}

__device__ __forceinline__ float af_step(float p, float u, float denom, float lr, float pscale, float wd) {
  return p - ((((u / denom) * lr) * pscale) + wd * p);
}

// (e) per tile: p -= lr * pscale * u / denom + wd * p ; grad_acc = 0 (its padding too)
__global__ void __launch_bounds__(AF_THREADS) af_apply_kernel(const AfArgs a) {
  const int64_t* L = tile_rec(a, blockIdx.x);
  for (int64_t i = L[L_ZLO] + threadIdx.x; i < L[L_ZHI]; i += AF_THREADS) a.g[i] = 0.f;
  if (L[L_TENSOR] < 0) return;
  const int64_t* T = tensor_rec(a, L[L_TENSOR]);
  const Clip cl = make_clip(a);
  const float denom = a.ws[2 * L[L_TENSOR]], pscale = a.ws[2 * L[L_TENSOR] + 1];
  if (T[T_KIND] == 0) {
    const int64_t base = T[T_OFFSET] + L[L_R0];
    const float* v = a.state + T[T_SA] + L[L_R0];
    const int n = static_cast<int>(L[L_NR]);
    for (int i = threadIdx.x; i < n; i += AF_THREADS) {
      const float u = cl(a.g[base + i]) * rsqrtf(v[i]);
      a.p[base + i] = af_step(a.p[base + i], u, denom, a.lr, pscale, a.wd);
      a.g[base + i] = 0.f;
    }
    return;
  }
  const FTile f = ftile(T, L);
  if (!f.active) return;
  const Factors F = load_factors(a, T, L, f);
#pragma unroll 4
  for (int r = threadIdx.x >> 5; r < f.nr; r += AF_WARPS) {
    const int64_t e = f.base + r * f.C + f.col4;
    const float4 g4 = *reinterpret_cast<const float4*>(a.g + e);
    float4 p4 = *reinterpret_cast<const float4*>(a.p + e);
    const float fr = row_factor(F, r);
    p4.x = af_step(p4.x, fact_u(F, cl(g4.x), fr, 0), denom, a.lr, pscale, a.wd);
    p4.y = af_step(p4.y, fact_u(F, cl(g4.y), fr, 1), denom, a.lr, pscale, a.wd);
    p4.z = af_step(p4.z, fact_u(F, cl(g4.z), fr, 2), denom, a.lr, pscale, a.wd);
    p4.w = af_step(p4.w, fact_u(F, cl(g4.w), fr, 3), denom, a.lr, pscale, a.wd);
    *reinterpret_cast<float4*>(a.p + e) = p4;
    *reinterpret_cast<float4*>(a.g + e) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

}  // namespace
}  // namespace ddpo

using namespace ddpo;

// Host planner: the only place that decides which tensors are factored (optax's _factored_dims).
extern "C" int ddpo_adafactor_plan(int ntensors, const int64_t* offsets, const int32_t* ndims, const int64_t* dims,
                                   int64_t n, int min_dim_size_to_factor, int64_t* plan, int64_t plan_words,
                                   int64_t* sizes, int64_t* tensor_info) {
  DDPO_REQUIRE(ntensors >= 1 && offsets && ndims && dims && sizes && n >= 0 && n % 4 == 0 && min_dim_size_to_factor >= 1,
               "adafactor_plan: bad arguments");
  std::vector<int64_t> tens(static_cast<size_t>(ntensors) * T_WORDS), tiles, taps;
  int64_t state = 0, nparts = 0, prev_end = 0, di = 0;
  for (int t = 0; t < ntensors; ++t) {
    const int nd = ndims[t];
    DDPO_REQUIRE(nd >= 1 && nd <= 8, "adafactor_plan: tensor %d has %d dims", t, nd);
    const int64_t* s = dims + di;
    di += nd;
    int64_t numel = 1;
    for (int d = 0; d < nd; ++d) {
      DDPO_REQUIRE(s[d] >= 1 && s[d] <= (1LL << 31) - 1, "adafactor_plan: tensor %d has a bad dim", t);
      numel *= s[d];
      DDPO_REQUIRE(numel <= n, "adafactor_plan: tensor %d is larger than the buffer", t);
    }
    const int64_t off = offsets[t];
    DDPO_REQUIRE(off >= prev_end && off + numel <= n, "adafactor_plan: tensor %d at offset %lld overlaps or leaves the buffer",
                 t, static_cast<long long>(off));
    // optax: d1, d0 = argsort(shape)[-2:] (numpy's sort is stable for these short shapes)
    int kind = 0;
    if (nd >= 2) {
      std::vector<int> idx(nd);
      std::iota(idx.begin(), idx.end(), 0);
      std::stable_sort(idx.begin(), idx.end(), [&](int x, int y) { return s[x] < s[y]; });
      const int d1 = idx[nd - 2], d0 = idx[nd - 1];
      if (s[d1] >= min_dim_size_to_factor) {
        DDPO_REQUIRE((d1 == nd - 2 && d0 == nd - 1) || (d1 == nd - 1 && d0 == nd - 2),
                     "adafactor_plan: tensor %d: its two largest dims are not the last two", t);
        kind = d0 == nd - 1 ? 1 : 2;
      }
    }
    int64_t* T = tens.data() + static_cast<size_t>(t) * T_WORDS;
    const int64_t R = kind ? s[nd - 2] : numel, C = kind ? s[nd - 1] : 1, ntap = numel / (R * C);
    if (kind) DDPO_REQUIRE(C % 4 == 0 && off % 4 == 0, "adafactor_plan: factored tensor %d needs 4-float aligned rows", t);
    const int64_t nrt = kind ? (R + AF_TR - 1) / AF_TR : (numel + AF_CHUNK - 1) / AF_CHUNK;
    const int64_t nct = kind ? (C + AF_TC - 1) / AF_TC : 1;
    T[T_OFFSET] = off, T[T_NUMEL] = numel, T[T_KIND] = kind, T[T_TAPS] = ntap, T[T_R] = R, T[T_C] = C;
    T[T_TILE0] = static_cast<int64_t>(tiles.size() / L_WORDS), T[T_NRT] = nrt, T[T_NCT] = nct;
    T[T_TAP0] = kind ? static_cast<int64_t>(taps.size() / P_WORDS) : -1;
    if (kind) {
      const int64_t lrow = kind == 1 ? R : C, lcol = kind == 1 ? C : R;
      T[T_SA] = state, T[T_SB] = state + ntap * lrow;
      state += ntap * (lrow + lcol);
    } else {
      T[T_SA] = state, T[T_SB] = -1;
      state += numel;
    }
    bool first = true;
    for (int64_t k = 0; k < ntap; ++k) {
      if (kind) taps.insert(taps.end(), {t, k});
      for (int64_t rt = 0; rt < nrt; ++rt)
        for (int64_t ct = 0; ct < nct; ++ct) {
          const int64_t r0 = rt * (kind ? AF_TR : AF_CHUNK), c0 = ct * AF_TC;
          const int64_t nr = std::min<int64_t>(kind ? AF_TR : AF_CHUNK, R - r0), nc = kind ? std::min<int64_t>(AF_TC, C - c0) : 1;
          const int64_t part = kind ? nparts++ : -1;
          tiles.insert(tiles.end(), {t, k, r0, nr, kind ? c0 : 0, nc, first ? prev_end : 0, first ? off : 0, part});
          first = false;
        }
    }
    prev_end = off + numel;
  }
  if (prev_end < n) tiles.insert(tiles.end(), {-1, 0, 0, 0, 0, 0, prev_end, n, -1});
  const int64_t ntiles = static_cast<int64_t>(tiles.size() / L_WORDS), ntaps = static_cast<int64_t>(taps.size() / P_WORDS);
  DDPO_REQUIRE(ntiles < (1LL << 31) - 1, "adafactor_plan: too many tiles");
  const int64_t ws_tile = 2LL * ntensors + ntaps, ws_part = ws_tile + 2 * ntiles;
  for (int64_t i = 0; i < ntiles; ++i)
    if (tiles[i * L_WORDS + L_PART] >= 0) tiles[i * L_WORDS + L_PART] = ws_part + tiles[i * L_WORDS + L_PART] * (AF_TR + AF_TC);
  const int64_t ws = ws_part + nparts * (AF_TR + AF_TC);
  const int64_t words = H_WORDS + static_cast<int64_t>(tens.size() + tiles.size() + taps.size());
  DDPO_REQUIRE(plan == nullptr || plan_words >= words, "adafactor_plan: plan needs %lld words", static_cast<long long>(words));
  sizes[0] = words, sizes[1] = state, sizes[2] = ws;
  if (tensor_info != nullptr)
    for (int t = 0; t < ntensors; ++t) {
      const int64_t* T = tens.data() + static_cast<size_t>(t) * T_WORDS;
      tensor_info[3 * t] = T[T_KIND], tensor_info[3 * t + 1] = T[T_SA], tensor_info[3 * t + 2] = T[T_SB];
    }
  if (plan != nullptr) {
    const int64_t head[H_WORDS] = {AF_MAGIC, n, ntensors, ntiles, ntaps, state, ws, 0};
    int64_t* o = std::copy(head, head + H_WORDS, plan);
    o = std::copy(tens.begin(), tens.end(), o);
    o = std::copy(tiles.begin(), tiles.end(), o);
    std::copy(taps.begin(), taps.end(), o);
  }
  return DDPO_OK;
}

extern "C" int ddpo_clip_adafactor(float* params, float* grad_acc, float* state, int64_t state_floats, int64_t n,
                                   const int64_t* plan_host, const int64_t* plan_dev, float* workspace,
                                   int64_t workspace_floats, const float* sumsq_dev, float grad_scale, float max_norm,
                                   float lr, float weight_decay, int step, float* norm_out, void* stream) {
  DDPO_REQUIRE(params && grad_acc && state && plan_host && plan_dev && workspace && sumsq_dev && n % 4 == 0 && step >= 1,
               "clip_adafactor: bad arguments");
  DDPO_REQUIRE(reinterpret_cast<uintptr_t>(params) % 16 == 0 && reinterpret_cast<uintptr_t>(grad_acc) % 16 == 0 &&
                   reinterpret_cast<uintptr_t>(state) % 4 == 0 && reinterpret_cast<uintptr_t>(workspace) % 4 == 0 &&
                   reinterpret_cast<uintptr_t>(plan_dev) % 8 == 0,
               "clip_adafactor: params and grad_acc must be 16-byte aligned");
  DDPO_REQUIRE(plan_host[H_MAGIC] == AF_MAGIC, "clip_adafactor: not an adafactor plan");
  DDPO_REQUIRE(plan_host[H_N] == n, "clip_adafactor: the plan is for %lld floats, the buffer has %lld",
               static_cast<long long>(plan_host[H_N]), static_cast<long long>(n));
  DDPO_REQUIRE(state_floats >= plan_host[H_STATE] && workspace_floats >= plan_host[H_WS],
               "clip_adafactor: state needs %lld floats and workspace %lld", static_cast<long long>(plan_host[H_STATE]),
               static_cast<long long>(plan_host[H_WS]));
  AfArgs a;
  a.p = params, a.g = grad_acc, a.state = state, a.ws = workspace, a.plan = plan_dev, a.sumsq = sumsq_dev;
  a.grad_scale = grad_scale, a.max_norm = max_norm, a.lr = lr, a.wd = weight_decay;
  a.beta = 1.0f - static_cast<float>(pow(static_cast<double>(step), -0.8));  // optax _decay_rate_pow(count) at count + 1 = step
  a.norm_out = norm_out;
  a.ntensors = static_cast<int>(plan_host[H_NTENSORS]), a.ntiles = static_cast<int>(plan_host[H_NTILES]);
  a.ntaps = static_cast<int>(plan_host[H_NTAPS]);
  a.ws_rcm = 2LL * a.ntensors, a.ws_tile = a.ws_rcm + a.ntaps;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  af_stats_kernel<<<a.ntiles, AF_THREADS, 0, s>>>(a);
  DDPO_LAUNCH_OK();
  if (a.ntaps > 0) {
    af_factor_kernel<<<a.ntaps, AF_THREADS, 0, s>>>(a);
    DDPO_LAUNCH_OK();
    af_usq_kernel<<<a.ntiles, AF_THREADS, 0, s>>>(a);
    DDPO_LAUNCH_OK();
  }
  af_tensor_kernel<<<a.ntensors, 128, 0, s>>>(a);
  DDPO_LAUNCH_OK();
  af_apply_kernel<<<a.ntiles, AF_THREADS, 0, s>>>(a);
  DDPO_LAUNCH_OK();
  return DDPO_OK;
}
