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
//
// The chunked feature transform follows the same chain in two halves: slice_sites_kernel resolves
// the X and Y codes of whole slices into each voxel's site within its slice, and compose_sites_kernel
// follows the last axis's code to one of those partial sites on the voxel's own line.
#pragma once
#include "edt_kernels.cuh"

namespace edtb200 {

// A stack of volumes laid end to end along z is sz / depth volumes of depth slices each: a Z code is
// a row within its voxel's own volume, and so is the z coordinate written.
struct SiteCodes {
  const int* axis[3];     // x, y, z code planes (the first ndim are read)
  int ndim;
  int64_t sx, sy, sz;
  int64_t depth;          // slices per volume (sz: one volume)
};

struct SitePlanes {
  int32_t* axis[3];       // x, y, z coordinate planes (the first ndim are written)
};

// What one later pass's site code says about a voxel's site along that axis.
//   kStepSelf    the voxel is unsigned background, its own site (its code is not followed)
//   kStepNone    no site at all (the distance is +inf)
//   kStepDirect  the site is at `row` on this line: the voxel just outside the run (or a face)
//   kStepVertex  the site is the site of the voxel at `row` on this line, found by the earlier axes
enum : int { kStepSelf, kStepNone, kStepDirect, kStepVertex };
__device__ __forceinline__ int site_step(bool self, int code, int* row) {
  if (self) return kStepSelf;
  if (code == kSiteNone) return kStepNone;
  *row = code < 0 ? site_direct_row(code) : code;
  return code < 0 ? kStepDirect : kStepVertex;
}

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
    const int64_t z0 = c.depth == c.sz ? 0 : pz / c.depth * c.depth;     // the volume's first slice
    int64_t q[3] = {px, py, pz - z0};
    const bool self = zero_is_background && labels[i] == 0;
    int step = self ? kStepSelf : kStepVertex;
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
    if (step == kStepNone) q[0] = q[1] = q[2] = -1;
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (k < c.ndim) out.axis[k][i] = (int32_t)q[k];
  }
}

// What expand_gather_kernel reads besides the labels: a signed feature transform's squared distances
// and x-fastest index planes (the first ndim are read) over the stack of count volumes of
// (sx, sy, sz) laid back to back, `vol` voxels each.  Coordinates are within each voxel's own volume,
// and idx[0] is -1 where there is no site.
struct ExpandSites {
  const float* sqdist;
  const int32_t* axis[3];
  int ndim;
  int64_t sx, sy, sz, vol, total;
};

// expand_labels: every background voxel whose nearest site lies within the limit takes that site's
// label; every other voxel keeps its own.  A voxel grows iff it is background, has a site (idx[0]
// >= 0) inside its volume, and (double)|sqdist| <= limit_sq.  Background is a label whose bits are all
// zero, or with as_float (4- or 8-byte IEEE labels) whose value is zero, so that -0.0 is background
// too.  Labels are copied as raw bits, so -0.0 and NaN payloads survive.  A labelled voxel reads
// nothing but its label; a background voxel reads its site's distance only when it has one, and the
// other planes only when it grows.
// `out` may be `labels` itself (no __restrict__ on either): only background voxels change, and a
// background voxel reads only its own label and its site's, and a site -- the nearest voxel of
// another label to a background voxel under the signed transform -- is always a labelled voxel,
// which nobody writes.  A site outside the volume (a face position of a black_border transform) has
// no label and grows nothing.
template <int Bytes>
__global__ void __launch_bounds__(256)
expand_gather_kernel(const typename LabelOf<Bytes>::type* labels, ExpandSites s, double limit_sq, int as_float,
                     typename LabelOf<Bytes>::type* out) {
  using LT = typename LabelOf<Bytes>::type;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < s.total; i += (int64_t)gridDim.x * blockDim.x) {
    LT v = labels[i];
    const LT magnitude = as_float ? (LT)(v << 1) : v;      // the sign bit shifted out: -0.0 == 0
    if (magnitude == 0) {
      const int64_t qx = __ldg(s.axis[0] + i);
      if (qx >= 0 && (double)fabsf(__ldg(s.sqdist + i)) <= limit_sq) {
        const int64_t qy = s.ndim >= 2 ? __ldg(s.axis[1] + i) : 0;
        const int64_t qz = s.ndim >= 3 ? __ldg(s.axis[2] + i) : 0;
        if (qx < s.sx && (uint64_t)qy < (uint64_t)s.sy && (uint64_t)qz < (uint64_t)s.sz)
          v = labels[i - i % s.vol + (qz * s.sy + qy) * s.sx + qx];
      }
    }
    out[i] = v;
  }
}

// Chunked feature transform, phase 1 (3-D): the X and Y codes of a slab of whole slices
// (sx, sy, sz) -> every voxel's site (qx, qy) within its own slice, kSiteNone in both where it has
// none.  qy is written over the Y codes (each is read at its own voxel only); the X codes are read at
// other rows, so qx goes to a separate plane.
template <int Bytes>
__global__ void __launch_bounds__(256)
slice_sites_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, const int* __restrict__ xcodes,
                   int* ycodes_qy, int64_t sx, int64_t sy, int64_t sz, int zero_is_background,
                   int32_t* __restrict__ qx) {
  const int64_t total = sx * sy * sz;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t line = i / sx;                 // y + sy * z
    const int64_t px = i - line * sx;
    const int64_t py = line % sy;
    int row = 0;
    const int step = site_step(zero_is_background && labels[i] == 0, ycodes_qy[i], &row);
    int x = (int)px, y = (int)py;
    if (step == kStepNone) {
      x = y = kSiteNone;
    } else if (step != kStepSelf) {
      y = row;
      if (step == kStepVertex) {
        x = __ldg(xcodes + i + sx * ((int64_t)row - py));
        if (x == kSiteNone) y = kSiteNone;
      }
    }
    qx[i] = x;
    ycodes_qy[i] = y;
  }
}

// The box of whole lines along the last axis that one phase-2 chunk covers: `plane` voxels per
// position along those lines (3-D: width * the box's y extent; 2-D: its x extent), lines of n voxels.
// `origin` is the box's first index along the cut axis (3-D: y; 2-D: x) in the volume.
struct SiteBox {
  int ndim;
  int64_t width, plane, n, origin;
};

// Chunked feature transform, phase 2: the last axis's codes -> every voxel's site in the volume.  A
// vertex code names a row of the voxel's own line, whose partial site (px, py) came from phase 1
// (part_x, part_y; kSiteNone: none); a direct code names the row on the voxel's own line.  The last
// axis's coordinate is written over its codes (each read at its own voxel only); the partial planes
// are read at other rows, so x (and y in 3-D) go to separate planes.
template <int Bytes>
__global__ void __launch_bounds__(256)
compose_sites_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, int* codes_last,
                     const int32_t* __restrict__ part_x, const int32_t* __restrict__ part_y, SiteBox b,
                     int zero_is_background, int32_t* __restrict__ out_x, int32_t* __restrict__ out_y) {
  const int64_t total = b.plane * b.n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pos = i / b.plane;             // along the last axis
    const int64_t base = i - pos * b.plane;
    const int64_t a = base % b.width;
    // the voxel's own coordinates in the volume; in 2-D base is the x index in the box
    int x = b.ndim == 3 ? (int)a : (int)(a + b.origin), y = (int)(base / b.width + b.origin);
    int row = 0;
    const int step = site_step(zero_is_background && labels[i] == 0, codes_last[i], &row);
    int last = (int)pos;
    if (step == kStepNone) {
      x = y = last = -1;
    } else if (step != kStepSelf) {
      last = row;
      if (step == kStepVertex) {
        const int64_t j = base + (int64_t)row * b.plane;
        x = __ldg(part_x + j);
        if (b.ndim == 3) y = __ldg(part_y + j);
        if (x == kSiteNone) x = y = last = -1;
      }
    }
    out_x[i] = x;
    if (b.ndim == 3) out_y[i] = y;
    codes_last[i] = last;
  }
}

}  // namespace edtb200
