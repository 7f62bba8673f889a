// Host-side cost model of the wgmma GEMMs (igemm.cu, wgrad.cu), in SM clock cycles of an H100 SXM.  The planners of
// both kernels rank their candidate launches with it; only the order of the candidates matters, not the absolute time.
#pragma once
#include <math.h>

namespace ddpo {

// Rates are per SM; the L2 rate (7.7 TB/s over the chip) is the one that makes the model's choices agree with
// CUDA-event timings of every igemm tile on the U-Net's launches (tests/bench_igemm_plan.py --all), the others are
// data-sheet figures.  The L2 rate was not fitted to the weight-gradient GEMM: with its 128-row tiles the L2 term,
// (128 + BN) x 32 B per step, always exceeds the tensor term, so the wgrad planner ranks every width as L2-bound.
// tests/bench_wgrad_plan.py --all times every width and split count the planner weighs on the train pass.
constexpr int NUM_SMS = 132;
constexpr double TENSOR_FLOP_PER_CLK = 4096.0;  // dense bf16 wgmma (989 TFLOP/s = 132 SMs x 1.83 GHz x 4096)
constexpr double SMEM_BYTES_PER_CLK = 128.0;    // shared-memory bandwidth that feeds the wgmma operands
constexpr double L2_BYTES_PER_CLK = 32.0;       // TMA operand loads out of L2
constexpr double HBM_BYTES_PER_CLK = 14.0;      // 3.35 TB/s shared by 132 SMs at 1.83 GHz

// One k16 step of a BM x BN tile (BM / 64 consumer warpgroups) is paced by the slowest of: the tensor cores
// (2*64*BN*16 FLOP per warpgroup), shared memory (each warpgroup reads 2 KB of A plus BN x 32 B of B: narrow tiles,
// BN <= 64, are bound by it) and L2 ((BM + BN) x 32 B of operands per tile: low tiles re-read B, narrow ones A).
inline double k16_step_clk(int bm, int bn) {
  const double wgs = bm / 64;
  return fmax(fmax(wgs * 2.0 * 64 * bn * 16 / TENSOR_FLOP_PER_CLK, wgs * (2048.0 + 32.0 * bn) / SMEM_BYTES_PER_CLK),
              (bm + bn) * 32.0 / L2_BYTES_PER_CLK);
}

}  // namespace ddpo
