// edt_watershed.cuh -- the relaxation passes of watershed (edtb200_watershed, include/edt_b200.h).
//
// Level.  L is the least fixed point of L[v] = min(L[v], max(f[v], L[u])) over the graph neighbours u of v,
// from f on the seeds and +inf elsewhere: the lowest flood level at which water from some seed reaches v.
// min and max of float32 values round nothing, and every update only lowers a value, so every relaxation
// order that stops only where no edge can lower a value reaches that one fixed point.
//
// Label.  With L fixed, an edge u -> v is TIGHT when v is not a seed and L[v] == max(f[v], L[u]).  W holds the
// marker minus one (so that all ones can mean none and a marker of all ones still fits) and relaxes by
// W[v] = min(W[v], W[u]) over the tight edges, from the seed's own marker on the seeds and none elsewhere.
// The seeds are never written, and a value is only ever copied from a neighbour, so the fixed point is the
// least marker with a tight path from its seed -- also on plateaus, where tight edges form cycles.  A voxel
// whose own altitude is +inf has L = +inf yet can still take a W over a tight edge, so this phase queues on
// changes to W, never to L.  The phases are kept apart for the reason geodesic keeps D and S apart: carried
// together, a torn pair (new L, old smaller W) could never be undone by min.
//
// Tiles, worklists, rounds and races are those of edt_geodesic.cuh (the same control block and tiles, the same
// round-1 rule that a seed counts as changed so that a seed on a tile's face, edge or corner reaches the tiles
// beyond it), with two differences: the neighbour offsets are those with at most `connectivity` non-zero
// components, both inside the sweep and in the choice of the neighbour tiles to queue; and L is a 4-byte
// float and W 4 bytes (markers of up to 4 bytes) or 8 bytes, so every halo read is an untorn aligned load.
// With label_bytes 0 there are no labels: every voxel inside the volume is a node with the same label.
#pragma once
#include <cooperative_groups.h>

#include "edt_host.h"

namespace edtb200 {

constexpr int kWsThreads = 256;
constexpr int kWsHalo = 1000;                     // the largest staged block: (8 + 2)^3 voxels

// The control block of one phase (zeroed before its seed kernel), as geodesic's GeoControl.  Round r reads
// list[r & 1] with count[r % 3] entries, appends to list[(r + 1) & 1] / count[(r + 1) % 3] and clears
// count[(r + 2) % 3].
struct WsControl {
  unsigned int count[3];
  unsigned long long rounds, visits;
};

template <int LB> struct WsLabel { using type = typename LabelOf<LB>::type; };
template <> struct WsLabel<0> { using type = uint8_t; };   // no labels: 1 inside the volume, 0 outside

struct WsArgs {
  float* level;                     // L
  void* w;                          // W - 1 (all ones: none), 4 or 8 bytes per voxel
  const float* image;               // f, as given (canonicalised on every read)
  const void* markers;
  int marker_bytes;
  uint32_t* flag;                   // per tile: the last round it was queued for
  uint32_t* list[2];                // two worklists of one entry per tile
  WsControl* ctl;
  int64_t sx, sy, sz, vol, total;
  int64_t nx, ny, nz, ntiles;       // tiles per axis of one volume, and of the stack
  int tx, ty, tz;                   // the tile
  int ndim, connectivity;
};

// An altitude as the definition reads it: NaN as +inf, -0.0 as +0.0.
__device__ __forceinline__ float ws_altitude(float f) {
  return f != f ? __int_as_float(0x7f800000) : f == 0.0f ? 0.0f : f;
}

template <int LB>
__device__ __forceinline__ typename WsLabel<LB>::type ws_label(const void* labels, int64_t i) {
  if constexpr (LB == 0) return 1;
  else return static_cast<const typename WsLabel<LB>::type*>(labels)[i];
}

__device__ __forceinline__ unsigned long long ws_marker(const WsArgs& a, int64_t i) {
  switch (a.marker_bytes) {
    case 1: return static_cast<const uint8_t*>(a.markers)[i];
    case 2: return static_cast<const uint16_t*>(a.markers)[i];
    case 4: return static_cast<const uint32_t*>(a.markers)[i];
    default: return static_cast<const unsigned long long*>(a.markers)[i];
  }
}

__device__ __forceinline__ void ws_queue(const WsArgs& a, int64_t t, uint32_t r, int b, int c) {
  if (atomicMax(a.flag + t, r) < r) a.list[b][atomicAdd(&a.ctl->count[c], 1u)] = (uint32_t)t;
}

// The seed kernel of one phase: L = f / +inf (level phase) or W = marker - 1 / none (label phase), and the
// tiles holding a seed queued for round 1.  A seed is a voxel whose marker and label are both non-zero.
template <int LB, class WT>
__global__ void __launch_bounds__(256)
watershed_seed_kernel(const void* __restrict__ labels, WsArgs a, bool label_phase) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.total; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long m = ws_label<LB>(labels, i) != 0 ? ws_marker(a, i) : 0ull;
    const bool seed = m != 0;
    if (label_phase)
      static_cast<WT*>(a.w)[i] = seed ? (WT)(m - 1) : ~(WT)0;
    else
      a.level[i] = seed ? ws_altitude(a.image[i]) : __int_as_float(0x7f800000);
    if (seed) {
      const int64_t row = i / a.sx, x = i - row * a.sx, col = row / a.sy, y = row - col * a.sy;
      const int64_t v = col / a.sz, z = col - v * a.sz;
      ws_queue(a, ((v * a.nz + z / a.tz) * a.ny + y / a.ty) * a.nx + x / a.tx, 1u, 1, 1);
    }
  }
}

// The seed kernel of extended_maxima's reconstruction (launch_hmax_phase): the level phase on negated values.
// With f canonical (NaN read as -inf, -0.0 as +0.0) and m = fl32(fl64(f) - h) (-0.0 as +0.0), it writes the
// altitude -f into neg_image, L = -m on every node (+inf elsewhere), and queues every tile holding a node for
// round 1 (one queue per warp and tile).  The level phase then leaves L = -R, where R is the least fixed point
// of R[v] = max(R[v], min(f[v], R[u])) from m: -R[v] = min(-R[v], max(-f[v], -R[u])).
template <int LB>
__global__ void __launch_bounds__(256)
hmax_seed_kernel(const void* __restrict__ labels, WsArgs a, float* __restrict__ neg_image, double h) {
  for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x; i0 < a.total; i0 += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = i0 + threadIdx.x;
    int64_t t = -1;
    if (i < a.total) {
      float f = a.image[i];
      f = f != f ? __int_as_float(0xff800000) : f == 0.0f ? 0.0f : f;
      float m = (float)((double)f - h);
      if (m == 0.0f) m = 0.0f;
      neg_image[i] = f == 0.0f ? 0.0f : -f;
      const bool node = ws_label<LB>(labels, i) != 0;
      a.level[i] = node ? (m == 0.0f ? 0.0f : -m) : __int_as_float(0x7f800000);
      if (node) {
        const int64_t row = i / a.sx, x = i - row * a.sx, col = row / a.sy, y = row - col * a.sy;
        const int64_t v = col / a.sz, z = col - v * a.sz;
        t = ((v * a.nz + z / a.tz) * a.ny + y / a.ty) * a.nx + x / a.tx;
      }
    }
    const unsigned same = __match_any_sync(0xffffffffu, t);
    if (t >= 0 && (int)threadIdx.x % 32 == __ffs(same) - 1) ws_queue(a, t, 1u, 1, 1);
  }
}

// The rounds of one phase, in ONE cooperative launch: Label false relaxes L, true relaxes W over the tight
// edges of the fixed L.
template <int LB, class WT, bool Label>
__global__ void __launch_bounds__(kWsThreads, 2)
watershed_relax_kernel(const void* __restrict__ labels, WsArgs a) {
  using LT = typename WsLabel<LB>::type;
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  __shared__ LT sl[kWsHalo];
  __shared__ float sv[kWsHalo];
  __shared__ WT sw[Label ? kWsHalo : 1];
  __shared__ int noff[26];
  __shared__ unsigned int dirs;
  WT* const w = static_cast<WT*>(a.w);
  constexpr WT kNone = ~(WT)0;
  const float inf = __int_as_float(0x7f800000);

  // the staged block: the tile and a one-voxel halo along each of the first ndim axes
  const int hy = a.ndim >= 2, hz = a.ndim >= 3;
  const int HX = a.tx + 2, HY = a.ty + 2 * hy, HZ = a.tz + 2 * hz, HXY = HX * HY;
  const int tvox = a.tx * a.ty * a.tz, hvox = HXY * HZ;
  // the neighbour offsets: at most `connectivity` non-zero components
  int nn = 0;
  for (int dz = -hz; dz <= hz; ++dz)
    for (int dy = -hy; dy <= hy; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int nonzero = (dx != 0) + (dy != 0) + (dz != 0);
        if (nonzero == 0 || nonzero > a.connectivity) continue;
        if (threadIdx.x == 0) noff[nn] = dz * HXY + dy * HX + dx;
        ++nn;
      }
  const bool lead = blockIdx.x == 0 && threadIdx.x == 0;
  unsigned long long visits = 0;
  uint32_t r = 1;
  for (;; ++r) {
    const uint32_t n = __ldcg(&a.ctl->count[r % 3]);
    if (n == 0) break;
    visits += n;
    if (lead) a.ctl->count[(r + 2) % 3] = 0;
    for (uint32_t q = blockIdx.x; q < n; q += gridDim.x) {
      const int64_t t = __ldcg(a.list[r & 1] + q);
      int64_t rest = t / a.nx;
      const int64_t ox = (t - rest * a.nx) * a.tx;
      int64_t rest2 = rest / a.ny;
      const int64_t oy = (rest - rest2 * a.ny) * a.ty;
      const int64_t v = rest2 / a.nz, oz = (rest2 - v * a.nz) * a.tz;
      const int64_t base = v * a.vol;
      __syncthreads();                 // the previous tile's block is no longer read
      if (threadIdx.x == 0) dirs = 0;
      for (int e = threadIdx.x; e < hvox; e += kWsThreads) {
        const int lz = e / HXY, ly = (e - lz * HXY) / HX, lx = e - lz * HXY - ly * HX;
        const int64_t x = ox + lx - 1, y = oy + ly - hy, z = oz + lz - hz;
        LT lab = 0;
        float lv = inf;
        WT wv = kNone;
        if (x >= 0 && x < a.sx && y >= 0 && y < a.sy && z >= 0 && z < a.sz) {
          const int64_t i = base + (z * a.sy + y) * a.sx + x;
          lab = ws_label<LB>(labels, i);
          if (lab != 0) {
            lv = __ldcg(a.level + i);
            if (Label) wv = __ldcg(w + i);
          }
        }
        sl[e] = lab;
        sv[e] = lv;
        if (Label) sw[e] = wv;
      }
      __syncthreads();
      // the tile's voxels this thread owns: 2 in 3-D, 1 in 2-D and 1-D.  The level phase keeps each one's
      // altitude; the label phase keeps the mask of its tight in-edges (none for a seed), fixed with L.
      unsigned long long start[2];
      int own[2];
      float alt[2];
      unsigned int tight[2];
      const int mine = (tvox - (int)threadIdx.x + kWsThreads - 1) / kWsThreads;
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        const int k = threadIdx.x + m * kWsThreads;
        const int lz = k / (a.tx * a.ty), ly = (k / a.tx) % a.ty, lx = k % a.tx;
        const int c = (lz + hz) * HXY + (ly + hy) * HX + lx + 1;
        own[m] = c;
        start[m] = 0;
        alt[m] = inf;
        tight[m] = 0;
        if (m >= mine || sl[c] == 0) continue;
        start[m] = Label ? (unsigned long long)sw[c] : (unsigned long long)__float_as_uint(sv[c]);
        const int64_t i = base + ((oz + lz) * a.sy + oy + ly) * a.sx + ox + lx;
        const float f = ws_altitude(a.image[i]);
        alt[m] = f;
        if (Label && ws_marker(a, i) == 0) {
          const float lc = sv[c];
          for (int j = 0; j < nn; ++j) {
            const int u = c + noff[j];
            if (sl[u] == sl[c] && fmaxf(f, sv[u]) == lc) tight[m] |= 1u << j;
          }
        }
      }
      // sweeps until one lowers nothing
      for (;;) {
        bool lowered = false;
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          if (m >= mine) break;
          const int c = own[m];
          if (!Label) {
            const LT lab = sl[c];
            if (lab == 0) continue;
            const float cur = *(volatile float*)&sv[c];
            float best = cur;
            for (int j = 0; j < nn; ++j) {
              const int u = c + noff[j];
              if (sl[u] == lab) best = fminf(best, fmaxf(alt[m], *(volatile float*)&sv[u]));
            }
            if (best < cur) {
              *(volatile float*)&sv[c] = best;
              lowered = true;
            }
          } else {
            if (!tight[m]) continue;
            const WT cur = *(volatile WT*)&sw[c];
            WT best = cur;
            for (unsigned int bits = tight[m]; bits; bits &= bits - 1)
              best = min(best, *(volatile WT*)&sw[c + noff[__ffs(bits) - 1]]);
            if (best < cur) {
              *(volatile WT*)&sw[c] = best;
              lowered = true;
            }
          }
        }
        if (!__syncthreads_or(lowered)) break;
      }
      // write back what went down, and the directions of the neighbour tiles it touches; in round 1 the
      // seeds count as gone down (see edt_geodesic.cuh)
      const unsigned long long unset = Label ? (unsigned long long)kNone : 0x7f800000ull;
      unsigned int mydirs = 0;
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        if (m >= mine) break;
        const int k = threadIdx.x + m * kWsThreads;
        const int c = own[m];
        if (sl[c] == 0) continue;
        const unsigned long long now = Label ? (unsigned long long)sw[c] : (unsigned long long)__float_as_uint(sv[c]);
        const bool lowered = now != start[m];
        if (!lowered && !(r == 1 && now != unset)) continue;
        const int lz = k / (a.tx * a.ty), ly = (k / a.tx) % a.ty, lx = k % a.tx;
        if (lowered) {
          const int64_t i = base + ((oz + lz) * a.sy + oy + ly) * a.sx + ox + lx;
          if (Label) w[i] = (WT)now;
          else a.level[i] = __uint_as_float((unsigned int)now);
        }
        // per axis the offsets of the tiles the voxel touches: 0, and -1 / +1 on the tile's low / high face;
        // a tile across an edge or a corner only where the connectivity joins voxels across it
        const int ex = lx == 0 ? -1 : lx == a.tx - 1 ? 1 : 0;
        const int ey = !hy ? 0 : ly == 0 ? -1 : ly == a.ty - 1 ? 1 : 0;
        const int ez = !hz ? 0 : lz == 0 ? -1 : lz == a.tz - 1 ? 1 : 0;
#pragma unroll
        for (int b = 1; b < 8; ++b) {
          const int dx = b & 1 ? ex : 0, dy = b & 2 ? ey : 0, dz = b & 4 ? ez : 0;
          if ((dx || !(b & 1)) && (dy || !(b & 2)) && (dz || !(b & 4)) && __popc(b) <= a.connectivity)
            mydirs |= 1u << ((dz + 1) * 9 + (dy + 1) * 3 + dx + 1);
        }
      }
      if (mydirs) atomicOr(&dirs, mydirs);
      __syncthreads();
      const unsigned int all = dirs;
      if (threadIdx.x < 27 && (all >> threadIdx.x & 1u)) {
        const int dx = threadIdx.x % 3 - 1, dy = threadIdx.x / 3 % 3 - 1, dz = threadIdx.x / 9 - 1;
        const int64_t cx = ox / a.tx + dx, cy = oy / a.ty + dy, cz = oz / a.tz + dz;
        if (cx >= 0 && cx < a.nx && cy >= 0 && cy < a.ny && cz >= 0 && cz < a.nz)
          ws_queue(a, ((v * a.nz + cz) * a.ny + cy) * a.nx + cx, r + 1, (r + 1) & 1, (r + 1) % 3);
      }
    }
    grid.sync();
  }
  if (lead) {
    a.ctl->rounds = r - 1;
    a.ctl->visits = visits;
  }
}

// W in the markers' width (W - 1 + 1: none wraps to 0) and, with level_out, L.
template <class MT, class WT>
__global__ void __launch_bounds__(256)
watershed_store_kernel(WsArgs a, MT* __restrict__ out, float* __restrict__ level_out) {
  const WT* w = static_cast<const WT*>(a.w);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.total; i += (int64_t)gridDim.x * blockDim.x) {
    out[i] = (MT)(WT)(w[i] + 1);
    if (level_out) level_out[i] = a.level[i];
  }
}

}  // namespace edtb200
