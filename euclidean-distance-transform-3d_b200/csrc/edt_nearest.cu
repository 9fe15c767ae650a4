// The nearest-labels passes for every label width and k (see edt_nearest.cuh), and their plan.
#include "edt_nearest.cuh"

namespace edtb200 {
namespace host {

NearestPlan nearest_plan(int ndim, const float w[3], double max_distance, int k, int label_bytes) {
  const BoundedPlan bp = bounded_plan(ndim, w, max_distance, false);
  NearestPlan p;
  p.bound = bp.bound;
  for (int a = 0; a < 3; ++a) {
    p.radius[a] = a < ndim ? bp.radius[a] : 0;
    if (a >= ndim) p.variant[a] = -1;
    else if (bp.radius[a] > kNearRadiusLimit) p.variant[a] = -1;
    else if (a == 0) p.variant[a] = kNearRowsPass;
    else p.variant[a] = nearest_smem_bytes((int)bp.radius[a], k, label_bytes) <= kNearSmemLimit ? kNearStaged : kNearGlobal;
  }
  return p;
}

int nearest_passes(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count,
                   const float w[3], const NearestPlan& p, int k, bool root, float* dist, void* lab, float* sdist,
                   void* slab, DeviceCache& dc, cudaStream_t stream) {
  const int64_t total = sx * sy * sz * count;
  return with_label_width(label_bytes, [&](auto b) {
    return with_k(k, [&](auto kk) {
      constexpr int B = decltype(b)::value, K = decltype(kk)::value;
      // 3-D: X -> out, Y -> scratch, Z -> out; 2-D: X -> scratch, Y -> out; 1-D: X -> out
      float* vx = ndim == 2 ? sdist : dist;
      void* lx = ndim == 2 ? slab : lab;
      int rc = launch_nearest_x_k<B, K>(labels, vx, lx, total, sx, w[0], (int)p.radius[0], p.bound, root && ndim == 1,
                                        dc, stream);
      const float* vin = vx;
      const void* lin = lx;
      for (int a = 1; !rc && a < ndim; ++a) {
        float* vo = a == ndim - 1 ? dist : sdist;
        void* lo = a == ndim - 1 ? lab : slab;
        LineGeom g;
        if (a == 1) {
          g.outer_count = sz * count; g.outer_stride = sx * sy; g.inner_count = sx; g.line_stride = sx; g.n = (int)sy;
        } else {
          g.outer_count = count; g.outer_stride = sx * sy * sz; g.inner_count = sx * sy; g.line_stride = sx * sy;
          g.n = (int)sz;
        }
        g.tiles_per_outer = 0;
        rc = launch_nearest_window_k<B, K>(vin, lin, vo, lo, total, g, w[a], (int)p.radius[a],
                                           p.variant[a] == kNearStaged, p.bound, root && a == ndim - 1, dc, stream);
        vin = vo;
        lin = lo;
      }
      return rc;
    });
  });
}

}  // namespace host
}  // namespace edtb200
