// edt_thickness.cuh -- the kernels of local thickness (edtb200_local_thickness, include/edt_b200.h).
//
// Local thickness at level r is the opening by the ball of r, taken for every label at once as
// EDTB200_OPEN takes it: the seeds S_r are the voxels whose edtsq D2 is not within r (the erosion), and a
// labelled voxel is covered at r iff the edtsq d2_r of the 1-byte mask (0 on S_r, 1 elsewhere, without
// black border) is within r there.  The call computes D2 once; then per level a streaming seed kernel
// writes the mask, the unbounded passes transform it, and thickness_store_kernel keeps the largest covering
// level of each voxel.  "Within r" is v <= B for B = cut_bound(r), as in bounded_cut_kernel: the unbounded
// passes return the bounded transform's values wherever those are within B, so every level equals
// spherical_open at r bit for bit.
//
// Per-volume kernels walk volume v = blockIdx.y, gridDim.y, ... and the voxels of v by a grid stride
// along x, so that each block reads its volume's level once.
#pragma once
#include "edt_host.h"

namespace edtb200 {

// top[v] = 1 + the bits of the largest finite D2 over the labelled voxels of volume v (as_float: 4- / 8-byte
// IEEE labels, -0.0 is background), or stays 0 when there is none.  Non-negative floats order as their
// bits, so one atomicMax per block after a block-wide maximum gives it.  The caller zeroes top.
template <int Bytes>
__global__ void __launch_bounds__(256)
thickness_top_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, const float* __restrict__ d2,
                     int64_t vol, int64_t count, int as_float, unsigned* __restrict__ top) {
  __shared__ unsigned warp_max[8];
  for (int64_t v = blockIdx.y; v < count; v += gridDim.y) {
    const int64_t base = v * vol;
    unsigned best = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < vol; i += (int64_t)gridDim.x * blockDim.x) {
      const float d = d2[base + i];
      if (d < __int_as_float(0x7f800000) && label_nonzero<Bytes>(labels[base + i], as_float))
        best = max(best, (unsigned)__float_as_int(d) + 1u);
    }
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    __syncthreads();                                       // the previous volume's warp_max is read
    if ((threadIdx.x & 31) == 0) warp_max[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < (int)(blockDim.x >> 5); ++w) best = max(best, warp_max[w]);
      if (best) atomicMax(top + v, best);
    }
  }
}

// The default levels of `count` volumes, n each, descending: r[v * n + j] = r_{n-1-j} with
//   r_i = (h/2) * (2R/h)^(i/n),  R = sqrt(the largest finite labelled D2 of v), or h/2 without one,
// in double, and bound[v * n + j] = cut_bound(r[v * n + j]).
__global__ void __launch_bounds__(256)
thickness_levels_kernel(const unsigned* __restrict__ top, int64_t count, int n, double h, double* __restrict__ r,
                        float* __restrict__ bound) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < count * n; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = k / n;
    const int i = n - 1 - (int)(k - v * n);
    const unsigned t = top[v];
    const double R = t ? sqrt((double)__int_as_float((int)(t - 1u))) : 0.5 * h;
    const double level = 0.5 * h * pow(2.0 * R / h, (double)i / (double)n);
    r[k] = level;
    bound[k] = cut_bound(level);
  }
}

// Column j of the levels a caller gave: out[v * m + j] = r for every volume v.
__global__ void __launch_bounds__(256)
thickness_fill_kernel(double* __restrict__ out, int64_t count, int m, int j, double r) {
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < count; v += (int64_t)gridDim.x * blockDim.x)
    out[v * m + j] = r;
}

// The seeds of one level: mask = 0 where D2 is not within the level (D2 > B), 1 elsewhere.
__global__ void __launch_bounds__(256)
thickness_seed_kernel(const float* __restrict__ d2, int64_t vol, int64_t count, ThicknessLevel level,
                      uint8_t* __restrict__ mask) {
  for (int64_t v = blockIdx.y; v < count; v += gridDim.y) {
    const float b = level.r ? level.bound[v * level.vstride] : level.b0;
    const int64_t base = v * vol;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < vol; i += (int64_t)gridDim.x * blockDim.x)
      mask[base + i] = d2[base + i] > b ? 0 : 1;
  }
}

// The store of one level: a labelled voxel whose distance to the seeds is within the level (d2r <= B)
// is covered at fl32(r).  first: out = that or 0 everywhere; otherwise out = max(out, that), which reads
// out only where the voxel is within the level and the labels only where out is below fl32(r).
template <int Bytes>
__global__ void __launch_bounds__(256, 4)
thickness_store_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, int as_float,
                       const float* __restrict__ d2r, int64_t vol, int64_t count, ThicknessLevel level, int first,
                       float* __restrict__ out) {
  for (int64_t v = blockIdx.y; v < count; v += gridDim.y) {
    const float b = level.r ? level.bound[v * level.vstride] : level.b0;
    const float rf = (float)(level.r ? level.r[v * level.vstride] : level.r0);
    const int64_t base = v * vol;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < vol; i += (int64_t)gridDim.x * blockDim.x) {
      const int64_t p = base + i;
      const bool near = d2r[p] <= b;
      if (first) {
        out[p] = near && label_nonzero<Bytes>(labels[p], as_float) ? rf : 0.0f;
      } else if (near && out[p] < rf && label_nonzero<Bytes>(labels[p], as_float)) {
        out[p] = rf;
      }
    }
  }
}

}  // namespace edtb200
