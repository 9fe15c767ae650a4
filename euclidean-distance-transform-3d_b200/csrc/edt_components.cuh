// edt_components.cuh -- the union-find passes of connected_components and extended_maxima
// (edtb200_connected_components, edtb200_extended_maxima, include/edt_b200.h).
//
// Graph.  A voxel is a node when its key says so (a non-zero label; with label_bytes 0 every voxel inside the
// volume), and two nodes are joined when they are neighbours under `connectivity` (at most `connectivity`
// non-zero components of the offset) and their keys are equal: the label alone for connected_components, the
// label and the canonical value R (NaN read as -inf, -0.0 as +0.0, compared as floats) for the plateaus of
// extended_maxima.
//
// Parents.  P holds one 4-byte parent per voxel, an index within its volume (volumes have fewer than 2^32
// voxels, so the index 2^32 - 1 never names a voxel: it marks a non-node, and later a dropped root).  Every
// pass keeps the invariant P[v] <= v:
//   - the tile pass starts from P[k] = k and links a root only under a smaller index (atomicMin in shared
//     memory), so the root it writes for a voxel is the least index of its component within the tile;
//   - the border pass links, through global atomics, the roots of the two ends of every joined edge that leaves
//     a tile: atomicMin(&P[b], a) with a < b.  When it returns b, b was a root and now hangs under a; when it
//     returns c != b, someone linked b first, b now hangs under min(a, c), and the loop goes on to join a and
//     c, so no link is lost.  Path compression lowers a parent only with atomicMin to a root of its own tree.
// Every link joins two trees of one component, and no parent rises, so a tree never holds two components and
// the least index m of a component always keeps P[m] = m (its parent is a node of its component that is <= m).
// Once every edge has been handled each component is one tree, and its only root is m -- whatever order the
// races took.  So the root of every voxel is the least index of its component, and numbering the kept roots
// by a prefix sum in memory order numbers the components in increasing order of their least index.
//
// Numbering.  The flatten pass sets P[v] = root(v) and writes a 1 into out at every root and 0 elsewhere; for
// the plateaus the mark pass then drops (P = 2^32 - 1, out = 0) the root of every plateau with a node that has
// a joined neighbour of larger R, or R = -inf.  A prefix sum in place over out (per volume: for a stack, each
// volume's first flag is lowered by the kept roots of the volume before it, modulo the output width) leaves
// every root's number at the root, and the number pass copies it to every voxel of its component: it reads out
// only at roots, and writes at a root the value it reads there, so the copy has no race.
#pragma once
#include <cub/block/block_reduce.cuh>

#include "edt_host.h"

namespace edtb200 {

constexpr int kCcThreads = 256;
constexpr int kCcTile = 1024;                     // the largest tile: 3-D 16x8x8, 2-D 32x32, 1-D 1024
constexpr uint32_t kCcNone = 0xffffffffu;         // P of a non-node and of a dropped root
constexpr int kCcChunk = 4096;                    // voxels per block of the per-volume count

struct CcArgs {
  uint32_t* parent;                 // P: an index within the volume per voxel
  const void* labels;               // null with label_bytes 0
  const float* value;               // the plateaus' R: f as given, or -R (negated)
  bool negated;
  int64_t sx, sy, sz, vol, total;
  int64_t nx, ny, nz, ntiles;       // tiles per axis of one volume, and of the stack
  int tx, ty, tz;
  int ndim, connectivity;
};

template <int LB> struct CcLabel { using type = typename LabelOf<LB>::type; };
template <> struct CcLabel<0> { using type = uint8_t; };   // no labels: 1 inside the volume

template <int LB>
__device__ __forceinline__ typename CcLabel<LB>::type cc_label(const CcArgs& a, int64_t i) {
  if constexpr (LB == 0) return 1;
  else return static_cast<const typename CcLabel<LB>::type*>(a.labels)[i];
}

// R as the definition reads it: NaN as -inf, -0.0 as +0.0 (-R negated back first)
__device__ __forceinline__ float cc_value(const CcArgs& a, int64_t i) {
  float x = a.value[i];
  if (a.negated) x = -x;
  return x != x ? __int_as_float(0xff800000) : x == 0.0f ? 0.0f : x;
}

// The key of connected_components: the label.
template <int LB> struct CcLabelKey {
  struct type { typename CcLabel<LB>::type lab; };
  static __device__ __forceinline__ type load(const CcArgs& a, int64_t i) { return {cc_label<LB>(a, i)}; }
  static __device__ __forceinline__ type none() { return {0}; }
  static __device__ __forceinline__ bool node(type k) { return k.lab != 0; }
  static __device__ __forceinline__ bool joined(type p, type q) { return p.lab == q.lab; }
};

// The key of the plateaus: the label and R.
template <int LB> struct CcPlateauKey {
  struct type { typename CcLabel<LB>::type lab; float r; };
  static __device__ __forceinline__ type load(const CcArgs& a, int64_t i) { return {cc_label<LB>(a, i), cc_value(a, i)}; }
  static __device__ __forceinline__ type none() { return {0, 0.0f}; }
  static __device__ __forceinline__ bool node(type k) { return k.lab != 0; }
  static __device__ __forceinline__ bool joined(type p, type q) { return p.lab == q.lab && p.r == q.r; }
};

// The offset (dz, dy, dx) is a neighbour under the connectivity; `backward`: it precedes 0 in memory order.
__device__ __forceinline__ bool cc_offset(const CcArgs& a, int dz, int dy, int dx, bool backward) {
  const int nonzero = (dx != 0) + (dy != 0) + (dz != 0);
  if (nonzero == 0 || nonzero > a.connectivity) return false;
  return !backward || dz < 0 || (dz == 0 && (dy < 0 || (dy == 0 && dx < 0)));
}

__device__ __forceinline__ uint32_t cc_find_shared(volatile uint32_t* p, uint32_t k) {
  for (uint32_t q; (q = p[k]) != k;) k = q;
  return k;
}

__device__ __forceinline__ void cc_union_shared(uint32_t* p, uint32_t a, uint32_t b) {
  for (;;) {
    a = cc_find_shared(p, a);
    b = cc_find_shared(p, b);
    if (a == b) return;
    if (a > b) { const uint32_t t = a; a = b; b = t; }
    const uint32_t old = atomicMin(p + b, a);
    if (old == b) return;
    b = old;
  }
}

// The root of k in the volume's parents p, lowering every parent on the way to it (atomicMin: a parent only
// ever goes down, to a node of its own tree).
__device__ __forceinline__ uint32_t cc_find(uint32_t* p, uint32_t k) {
  uint32_t r = k;
  for (uint32_t q; (q = __ldcg(p + r)) != r;) r = q;
  while (k > r) {
    const uint32_t next = __ldcg(p + k);
    if (next > r) atomicMin(p + k, r);
    k = next;
  }
  return r;
}

__device__ __forceinline__ void cc_union(uint32_t* p, uint32_t a, uint32_t b) {
  for (;;) {
    a = cc_find(p, a);
    b = cc_find(p, b);
    if (a == b) return;
    if (a > b) { const uint32_t t = a; a = b; b = t; }
    const uint32_t old = atomicMin(p + b, a);
    if (old == b) return;
    b = old;
  }
}

// Tile pass: one CTA per tile stages its keys, joins its joined backward edges inside the tile in shared
// memory and writes every node's tile root as P (kCcNone for the other voxels).
template <class K>
__global__ void __launch_bounds__(kCcThreads, 4) components_tile_kernel(CcArgs a) {
  __shared__ uint32_t sp[kCcTile];
  __shared__ typename K::type sk[kCcTile];
  const int txy = a.tx * a.ty, tvox = txy * a.tz;
  const int hy = a.ndim >= 2, hz = a.ndim >= 3;
  for (int64_t t = blockIdx.x; t < a.ntiles; t += gridDim.x) {
    int64_t rest = t / a.nx;
    const int64_t ox = (t - rest * a.nx) * a.tx;
    const int64_t rest2 = rest / a.ny;
    const int64_t oy = (rest - rest2 * a.ny) * a.ty;
    const int64_t v = rest2 / a.nz, oz = (rest2 - v * a.nz) * a.tz;
    const int64_t base = v * a.vol;
    __syncthreads();                   // the previous tile is no longer read
    for (int k = threadIdx.x; k < tvox; k += kCcThreads) {
      const int lz = k / txy, ly = (k - lz * txy) / a.tx, lx = k - lz * txy - ly * a.tx;
      const int64_t x = ox + lx, y = oy + ly, z = oz + lz;
      const bool inside = x < a.sx && y < a.sy && z < a.sz;
      sk[k] = inside ? K::load(a, base + (z * a.sy + y) * a.sx + x) : K::none();
      sp[k] = k;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < tvox; k += kCcThreads) {
      const typename K::type key = sk[k];
      if (!K::node(key)) continue;
      const int lz = k / txy, ly = (k - lz * txy) / a.tx, lx = k - lz * txy - ly * a.tx;
      for (int dz = -hz; dz <= 0; ++dz)
        for (int dy = -hy; dy <= hy; ++dy)
          for (int dx = -1; dx <= 1; ++dx) {
            if (!cc_offset(a, dz, dy, dx, true)) continue;
            if (lz + dz < 0 || ly + dy < 0 || ly + dy >= a.ty || lx + dx < 0 || lx + dx >= a.tx) continue;
            const int u = k + dz * txy + dy * a.tx + dx;
            if (K::node(sk[u]) && K::joined(key, sk[u])) cc_union_shared(sp, k, u);
          }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < tvox; k += kCcThreads) {
      const int lz = k / txy, ly = (k - lz * txy) / a.tx, lx = k - lz * txy - ly * a.tx;
      const int64_t x = ox + lx, y = oy + ly, z = oz + lz;
      if (x >= a.sx || y >= a.sy || z >= a.sz) continue;
      uint32_t root = kCcNone;
      if (K::node(sk[k])) {
        const uint32_t r = cc_find_shared(sp, k);
        const int rz = r / txy, ry = (r - rz * txy) / a.tx, rx = r - rz * txy - ry * a.tx;
        root = (uint32_t)(((oz + rz) * a.sy + oy + ry) * a.sx + ox + rx);
      }
      a.parent[base + (z * a.sy + y) * a.sx + x] = root;
    }
  }
}

// Border pass: every node on a tile's face joins its joined backward neighbours in other tiles.
template <class K>
__global__ void __launch_bounds__(kCcThreads, 4) components_border_kernel(CcArgs a) {
  const int hy = a.ndim >= 2, hz = a.ndim >= 3;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = i / a.vol, local = i - v * a.vol;
    const int64_t row = local / a.sx, x = local - row * a.sx, z = row / a.sy, y = row - z * a.sy;
    const int lx = (int)(x % a.tx), ly = (int)(y % a.ty), lz = (int)(z % a.tz);
    const bool face = lx == 0 || lx == a.tx - 1 || (hy && (ly == 0 || ly == a.ty - 1)) || (hz && lz == 0);
    if (!face) continue;
    const typename K::type key = K::load(a, i);
    if (!K::node(key)) continue;
    uint32_t* p = a.parent + v * a.vol;
    for (int dz = -hz; dz <= 0; ++dz)
      for (int dy = -hy; dy <= hy; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
          if (!cc_offset(a, dz, dy, dx, true)) continue;
          const int mx = lx + dx, my = ly + dy, mz = lz + dz;
          if (mx >= 0 && mx < a.tx && my >= 0 && my < a.ty && mz >= 0) continue;        // inside the tile
          const int64_t ux = x + dx, uy = y + dy, uz = z + dz;
          if (ux < 0 || ux >= a.sx || uy < 0 || uy >= a.sy || uz < 0) continue;
          const int64_t u = (uz * a.sy + uy) * a.sx + ux;
          const typename K::type ku = K::load(a, v * a.vol + u);
          if (K::node(ku) && K::joined(key, ku)) cc_union(p, (uint32_t)local, (uint32_t)u);
        }
  }
}

// Flatten pass: P[v] = root(v), and the flags in out: 1 at every root, 0 elsewhere.
template <class OT>
__global__ void __launch_bounds__(kCcThreads, 4) components_flatten_kernel(CcArgs a, OT* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = i / a.vol, local = i - v * a.vol;
    const uint32_t q = __ldcg(a.parent + i);
    OT flag = 0;
    if (q != kCcNone) {
      const uint32_t r = cc_find(a.parent + v * a.vol, (uint32_t)local);
      if (r != q) a.parent[i] = r;
      flag = r == (uint32_t)local;
    }
    out[i] = flag;
  }
}

// Mark pass of the plateaus: a node with a joined neighbour (the same label) of larger R, or with R = -inf,
// drops its plateau's root.
template <int LB, class OT>
__global__ void __launch_bounds__(kCcThreads, 4) components_mark_kernel(CcArgs a, OT* __restrict__ out) {
  const int hy = a.ndim >= 2, hz = a.ndim >= 3;
  const float ninf = __int_as_float(0xff800000);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.total; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t r = __ldcg(a.parent + i);
    if (r == kCcNone) continue;                  // not a node, or a root already dropped
    const int64_t v = i / a.vol, local = i - v * a.vol;
    const int64_t row = local / a.sx, x = local - row * a.sx, z = row / a.sy, y = row - z * a.sy;
    const auto lab = cc_label<LB>(a, i);
    const float rv = cc_value(a, i);
    bool drop = rv == ninf;
    for (int dz = -hz; dz <= hz && !drop; ++dz)
      for (int dy = -hy; dy <= hy && !drop; ++dy)
        for (int dx = -1; dx <= 1 && !drop; ++dx) {
          if (!cc_offset(a, dz, dy, dx, false)) continue;
          const int64_t ux = x + dx, uy = y + dy, uz = z + dz;
          if (ux < 0 || ux >= a.sx || uy < 0 || uy >= a.sy || uz < 0 || uz >= a.sz) continue;
          const int64_t u = v * a.vol + (uz * a.sy + uy) * a.sx + ux;
          drop = cc_label<LB>(a, u) == lab && cc_value(a, u) > rv;
        }
    if (drop) {
      a.parent[v * a.vol + r] = kCcNone;
      out[v * a.vol + r] = 0;
    }
  }
}

// The kept roots of each volume of a stack: one block per kCcChunk voxels of one volume.
template <class OT>
__global__ void __launch_bounds__(kCcThreads, 4) components_count_kernel(const OT* __restrict__ flags, int64_t vol,
                                                                      int64_t chunks, unsigned long long* counts) {
  using Reduce = cub::BlockReduce<unsigned long long, kCcThreads>;
  __shared__ typename Reduce::TempStorage tmp;
  const int64_t v = blockIdx.x / chunks, c = blockIdx.x - v * chunks;
  const int64_t lo = c * kCcChunk, hi = lo + kCcChunk < vol ? lo + kCcChunk : vol;
  unsigned long long n = 0;
  for (int64_t i = lo + threadIdx.x; i < hi; i += kCcThreads) n += flags[v * vol + i];
  n = Reduce(tmp).Sum(n);
  if (threadIdx.x == 0 && n) atomicAdd(counts + v, n);
}

// Lowers the first flag of every volume after the first by the kept roots of the volume before it, so that
// one prefix sum over the stack numbers each volume from 1: with every earlier first flag lowered the same
// way, the sum carried into volume v is exactly the kept roots of volume v - 1 (modulo the output width).
template <class OT>
__global__ void components_rebase_kernel(OT* flags, int64_t vol, int64_t count, const unsigned long long* counts) {
  for (int64_t v = 1 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < count; v += (int64_t)gridDim.x * blockDim.x)
    flags[v * vol] -= (OT)counts[v - 1];
}

// Number pass: out[v] = the number of root(v) (0 for a non-node and a dropped root's plateau).
template <class OT>
__global__ void __launch_bounds__(kCcThreads, 4) components_number_kernel(CcArgs a, OT* out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = i / a.vol, local = i - v * a.vol;
    const uint32_t r = a.parent[i];
    OT n = 0;
    if (r != kCcNone && (r == (uint32_t)local || a.parent[v * a.vol + r] != kCcNone)) n = out[v * a.vol + r];
    out[i] = n;
  }
}

namespace host {
// The kernel arguments of a job (edt_components.cu), and the grid of a pass with one thread per item.
CcArgs cc_args(const ComponentsJob& j);
unsigned cc_blocks(int64_t n, const DeviceCache& dc);
}  // namespace host

}  // namespace edtb200
