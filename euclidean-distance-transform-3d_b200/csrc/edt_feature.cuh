// edt_feature.cuh -- the feature transform's last step: per-pass site codes -> the nearest site.
//
// The site-tracking passes (first_axis_kernel / later_axis_long_kernel with Sites = true) leave one
// code plane per axis (see kSiteNone in edt_kernels.cuh).  The nearest site q of voxel p is found
// by following them back from the last axis:
//   qz from the Z code at p;
//   qy from the Y code at (px, py, qz), unless the Z code was direct (then qy = py);
//   qx from the X code at (px, qy, qz), unless the Z or Y code was direct (then qx = px).
// A direct code is the voxel just outside a run along its own axis, which IS the site: its own
// codes belong to another label and must not be followed.  The voxels the chain visits all carry
// p's label, so the chain never meets a code of another run.  The code planes are read at other
// voxels than the one written, so they are scratch, separate from the output planes.
#pragma once
#include "edt_kernels.cuh"

namespace edtb200 {

struct SiteCodes {
  const int* axis[3];     // x, y, z code planes (the first ndim are read)
  int ndim;
  int64_t sx, sy, sz;
};

struct SitePlanes {
  int32_t* axis[3];       // x, y, z coordinate planes (the first ndim are written)
};

// zero_is_background: label 0 is background, whose site is the voxel itself (edt, unsigned);
// otherwise (sdf) background is an ordinary label and is resolved like any other.
template <int Bytes>
__global__ void __launch_bounds__(256)
resolve_sites_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, SiteCodes c, int zero_is_background,
                     SitePlanes out) {
  const int64_t plane = c.sx * c.sy;
  const int64_t total = plane * c.sz;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pz = i / plane;
    const int64_t rem = i - pz * plane;
    const int64_t py = rem / c.sx;
    const int64_t px = rem - py * c.sx;
    int64_t q[3] = {px, py, pz};
    if (!(zero_is_background && labels[i] == 0)) {
      bool direct = false, none = false;
      if (c.ndim == 3) {
        const int code = __ldg(c.axis[2] + i);
        if (code == kSiteNone) none = true;
        else if (code < 0) { q[2] = site_direct_row(code); direct = true; }
        else q[2] = code;
      }
      if (c.ndim >= 2 && !direct && !none) {
        const int code = __ldg(c.axis[1] + px + c.sx * (py + c.sy * q[2]));
        if (code == kSiteNone) none = true;
        else if (code < 0) { q[1] = site_direct_row(code); direct = true; }
        else q[1] = code;
      }
      if (!direct && !none) {
        const int code = __ldg(c.axis[0] + px + c.sx * (q[1] + c.sy * q[2]));
        if (code == kSiteNone) none = true;
        else q[0] = code;
      }
      if (none) q[0] = q[1] = q[2] = -1;
    }
    for (int k = 0; k < c.ndim; ++k) out.axis[k][i] = (int32_t)q[k];
  }
}

}  // namespace edtb200
