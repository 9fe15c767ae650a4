// edt_medial.cuh -- the last step of the medial axis (edtb200_medial_axis, include/edt_b200.h).
//
// The call runs the edtsq of the labels (run_passes), then the parabolic dilation of that D^2 with its
// site codes (launch_parabolic_pass, codes into one plane per axis), and then medial_mark_kernel: every
// labelled voxel p follows the codes to its site q(p) -- the maximiser of D^2(y) - |p - y|^2_w, the power
// (Laguerre) site of p -- and marks it.  The marked voxels are the reduced discrete medial axis: the balls
// B(y, D(y)) that are the power maximiser of at least one labelled voxel.
#pragma once
#include "edt_host.h"

namespace edtb200 {

// For every voxel p of the stack: where L(p) != 0 (as_float: 4- / 8-byte IEEE labels, -0.0 is zero), follow
// the parabolic passes' codes as resolve_sites_kernel does -- q_z from the Z code at p, q_y from the Y code
// at (p_x, p_y, q_z), q_x from the X code at (p_x, q_y, q_z), rows within p's own volume -- and store
// medial[q] = 1 in p's volume; a p without a site stores nothing.  Many voxels may mark one q: concurrent
// stores of the same byte are benign, and the caller zeroes `medial` first.  dist non-null: it holds D^2
// and every voxel's value becomes __fsqrt_rn of it, correctly rounded, as edt's last store.
template <int Bytes>
__global__ void __launch_bounds__(256)
medial_mark_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, SiteCodes c, int as_float,
                   uint8_t* __restrict__ medial, float* __restrict__ dist) {
  using LT = typename LabelOf<Bytes>::type;
  const int64_t plane = c.sx * c.sy;
  const int64_t total = plane * c.sz;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    if (dist) dist[i] = __fsqrt_rn(dist[i]);
    LT v = labels[i];
    if constexpr (Bytes >= 4)
      if (as_float) v = (LT)(v << 1);                  // every bit but the sign
    if (v == 0) continue;
    const int64_t pz = i / plane;
    const int64_t rem = i - pz * plane;
    const int64_t py = rem / c.sx;
    const int64_t px = rem - py * c.sx;
    const int64_t z0 = c.depth == c.sz ? 0 : pz / c.depth * c.depth;     // the volume's first slice
    int64_t q[3] = {px, py, pz - z0};
    int step = kStepVertex;
#pragma unroll
    for (int k = 2; k >= 1; --k) {
      if (k >= c.ndim || step != kStepVertex) continue;
      int row = 0;
      step = site_step(false, __ldg(c.axis[k] + px + c.sx * (q[1] + c.sy * (z0 + q[2]))), &row);
      if (step != kStepNone) q[k] = row;
    }
    if (step == kStepVertex) {
      const int code = __ldg(c.axis[0] + px + c.sx * (q[1] + c.sy * (z0 + q[2])));
      if (code == kSiteNone) step = kStepNone;
      else q[0] = code;
    }
    if (step == kStepNone) continue;
    medial[q[0] + c.sx * (q[1] + c.sy * (z0 + q[2]))] = 1;
  }
}

}  // namespace edtb200
