// Shared device/host helpers for libddpo_b200 (sm_90a only).
// PTX wrappers for mbarrier, TMA (cp.async.bulk.tensor) and wgmma (fence / commit / wait,
// shared-memory matrix descriptors), status handling.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ddpo_b200.h"

namespace ddpo {

// ---------------------------------------------------------------- status ----
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);
#define DDPO_CUDA_OK(expr)                                        \
  do {                                                            \
    cudaError_t _e = (expr);                                      \
    if (_e != cudaSuccess) return ::ddpo::cuda_fail(_e, #expr);   \
  } while (0)
#define DDPO_REQUIRE(cond, ...)                                   \
  do {                                                            \
    if (!(cond)) {                                                \
      ::ddpo::set_error(__VA_ARGS__);                             \
      return DDPO_ERR_INVALID;                                    \
    }                                                             \
  } while (0)
#define DDPO_LAUNCH_OK() DDPO_CUDA_OK(cudaGetLastError())

int num_sms();

// Encode a (<=5-D) bf16/f32 tiled tensor map through the driver entry point
// (resolved lazily with cudaGetDriverEntryPoint so the library has no link-time
// dependency on libcuda and loads on a CPU-only box).
int make_tensor_map(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes /* rank-1 entries, dims 1.. */, const uint32_t* box,
                    const uint32_t* elem_strides, int swizzle_128b);

// An attention operand or output: bf16 [batch, n, ld] with head h at columns [h d, h d + d).  TMA and the 16-byte loads
// of the attention kernels need a 16-byte aligned base and a row pitch of whole 16-byte units.
inline bool attention_operands_ok(const void* base, int ld, int heads, int d) {
  return (reinterpret_cast<uintptr_t>(base) & 15) == 0 && ld % 8 == 0 && ld >= heads * d;
}

#ifdef __CUDACC__
// ------------------------------------------------------------- small utils ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
__device__ __forceinline__ float ex2_mufu(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcpf_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// sigmoid / SiLU on the two MUFU ops ex2 + rcp (relative error ~2e-7); the IEEE division of x / (1 + __expf(-x)) cost
// ~10 more instructions per element in the GroupNorm apply kernels, which are issue- as much as bandwidth-limited.
__device__ __forceinline__ float sigmoid_f(float x) { return rcpf_approx(1.0f + ex2_mufu(-1.4426950408889634f * x)); }
__device__ __forceinline__ float silu_f(float x) { return x * sigmoid_f(x); }
// SiLU on ONE MUFU op: x sigmoid(x) = z + z tanh(z), z = x / 2 (tanh.approx: max relative error 2^-11, an order below
// bf16 resolution).  Used where the result is rounded to bf16 anyway (the GroupNorm -> GEMM-operand path, which is
// MUFU-/issue-bound with the two-MUFU form); fp32 consumers keep silu_f.
__device__ __forceinline__ float silu_bf16_f(float x) {
  const float z = 0.5f * x;
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(z));
  return fmaf(z, t, z);
}
__device__ __forceinline__ float gelu_tanh_f(float x) {
  const float k = 0.7978845608028654f;  // sqrt(2/pi)
  float u = k * (x + 0.044715f * x * x * x);
  // 0.5 (1 + tanh u) == 1 / (1 + e^{-2u}): two MUFU ops (ex2, rcp) instead of libm tanhf's ~25 instructions;
  // relative error ~2e-7, exact limits at +-inf
  const float e = ex2_mufu(-2.885390081777927f * u);  // e^{-2u}
  return x * rcpf_approx(1.0f + e);
}
__device__ __forceinline__ float gelu_tanh_grad_f(float x) {
  const float k = 0.7978845608028654f;
  float u = k * (x + 0.044715f * x * x * x);
  const float e = ex2_mufu(fminf(-2.885390081777927f * u, 80.0f));  // e^{-2u}, clamped so that e * sg stays finite
  const float sg = rcpf_approx(1.0f + e);  // (1 + tanh u) / 2
  float du = k * (1.0f + 3.0f * 0.044715f * x * x);
  // d/dx [x sg] with 1 - tanh^2 u = 4 e sg^2 (no cancellation near |tanh| = 1)
  return sg + 2.0f * x * du * (e * sg) * sg;
}

// 2^x for x <= 0 on the FMA/ALU pipes instead of the MUFU unit (16/clk/SM): Cody-Waite + degree-3 polynomial
// (max relative error 8.8e-5, far below bf16 resolution).  The attention forward alternates it with ex2_mufu by COLUMN
// PARITY (a fixed function of the element position -> deterministic, batch-invariant) because the softmax
// exponentials, not the tensor cores, bound the kernel when every element goes through MUFU.
__device__ __forceinline__ float ex2_poly(float x) {
  x = fmaxf(x, -126.0f);
  const float r = __fadd_rd(x, 12582912.0f);  // 1.5 * 2^23: low mantissa bits now hold floor(x)
  const float f = x - (r - 12582912.0f);      // in [0, 1)
  const float p = fmaf(fmaf(fmaf(0.0771190897f, f, 0.2275643945f), f, 0.6951461434f), f, 1.0f);
  return __int_as_float(__float_as_int(p) + ((__float_as_int(r) - 0x4B400000) << 23));
}

// Which score columns of the attention forward take the polynomial: every DDPO_EXP_POLY_FWD-th one (0 = none), column
// col with col % DDPO_EXP_POLY_FWD == DDPO_EXP_POLY_FWD - 1 (the per-lane select in attention.cu softmax_block).  The
// split is a fixed function of the element's position, so results stay deterministic and batch invariant.
// The polynomial costs ~10 issue slots against 1 for MUFU.EX2, so only the forward kernel (fewer other instructions
// per score) keeps a small share; the backward uses MUFU alone.
#ifndef DDPO_EXP_POLY_FWD
#define DDPO_EXP_POLY_FWD 8
#endif

// --------------------------------------------------------------- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (reported as a CUDA error) instead of hanging the GPU.
// try_wait already suspends the warp for a hardware-chosen interval; the clock is read once every 256 retries so the
// retry loop stays at 3 instructions.  No explicit suspend-time hint: a waiting producer or consumer should wake up as
// soon as its barrier completes.
#ifndef DDPO_MBAR_TIMEOUT_CYCLES
#define DDPO_MBAR_TIMEOUT_CYCLES 8000000000ll  // ~4 s at 2 GHz
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = 0;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 255u) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > DDPO_MBAR_TIMEOUT_CYCLES) __trap();
    }
  }
}
// mbar_wait that returns false after the same timeout instead of trapping, for code after a setmaxnreg.inc: a trap
// inside such a region makes ptxas allocate it as if the increase had not happened (and spill).  The caller traps once
// it is out of the region's hot loop.
__device__ __forceinline__ bool mbar_wait_timed(uint64_t* bar, uint32_t parity) {
  long long t0 = 0;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 255u) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > DDPO_MBAR_TIMEOUT_CYCLES) return false;
    }
  }
  return true;
}

// -------------------------------------------------------------------- TMA ----
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ------------------------------------------------------------------ wgmma ----
// Shared-memory matrix descriptor of a SWIZZLE_128B operand (sm_90): start address, leading and stride byte offsets
// (all >> 4), layout type 1 = 128-byte swizzle at bits [62, 64).  K-major tiles are rows of 64 bf16 (128 B) in 8-row
// atoms of 1 KB: SBO = 1024, LBO unused.  MN-major tiles: LBO = distance between 64-element MN blocks, SBO = distance
// between 8-row K groups.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;  // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Pins the registers of a wgmma operand at this point of the instruction order: after a wgmma_wait (the wait names no
// registers, so the compiler could hoist a use of the accumulators above it), and before a wgmma_fence (so that the
// instructions defining them are not sunk past it into the wgmma pipeline, which ptxas would serialise).
template <int N>
__device__ __forceinline__ void reg_fence(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
template <int N>
__device__ __forceinline__ void reg_fence(uint32_t (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(r[i])::"memory");
}
// barrier among `count` threads (a multiple of 32) on hardware barrier `id` (id 0 is __syncthreads)
__device__ __forceinline__ void named_barrier(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
#endif  // __CUDACC__

}  // namespace ddpo
