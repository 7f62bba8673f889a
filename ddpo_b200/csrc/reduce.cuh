// Second stage of the two-stage column reductions (bias / scale gradients, per-sample sums): sums `rows` partial rows
// of a row-major fp32 matrix [groups][rows][width] into out[groups][width].
//
// Deterministic: thread (tx, ty) of a 32 x 32 block adds rows ty, ty + 32, ... of column tx in ascending order and the
// 32 per-thread sums are combined in ascending ty through shared memory -- the result depends only on (rows, width),
// never on timing.  The first-stage kernels emit up to 2560 partial rows for the 64 x 64 feature maps; the previous
// one-thread-per-column loop over them (3 CTAs of 128 threads) was latency-bound; here every warp reads 128 contiguous bytes per row and 32 rows are in flight
// per column.
#pragma once
#include "common.cuh"

namespace ddpo {

// columns [0, split) go to out0[g * split + c], columns [split, width) to out1[g * (width - split) + c - split]
static __global__ void __launch_bounds__(1024) reduce_rows_kernel(const float* __restrict__ part, int rows, int width, int split,
                                                           float* __restrict__ out0, float* __restrict__ out1,
                                                           int accumulate) {
  __shared__ float sm[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx, g = blockIdx.y;
  const float* p = part + static_cast<size_t>(g) * rows * width;
  float s = 0.f;
  if (c < width) {
    int r = ty;
    for (; r + 96 < rows; r += 128) {  // 4 independent loads in flight, added in row order
      const float a0 = p[static_cast<size_t>(r) * width + c], a1 = p[static_cast<size_t>(r + 32) * width + c];
      const float a2 = p[static_cast<size_t>(r + 64) * width + c], a3 = p[static_cast<size_t>(r + 96) * width + c];
      s += a0, s += a1, s += a2, s += a3;
    }
    for (; r < rows; r += 32) s += p[static_cast<size_t>(r) * width + c];
  }
  sm[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && c < width) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) t += sm[i][tx];
    float* o = c < split ? out0 + static_cast<size_t>(g) * split + c
                         : out1 + static_cast<size_t>(g) * (width - split) + (c - split);
    *o = accumulate ? *o + t : t;
  }
}

static inline void launch_reduce_rows(const float* part, int groups, int rows, int width, int split, float* out0, float* out1,
                               int accumulate, cudaStream_t stream) {
  dim3 grid((width + 31) / 32, groups);
  reduce_rows_kernel<<<grid, 1024, 0, stream>>>(part, rows, width, split, out0, out1, accumulate);
}

}  // namespace ddpo
