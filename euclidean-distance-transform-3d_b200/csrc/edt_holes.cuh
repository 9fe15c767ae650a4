// edt_holes.cuh -- the tally and apply passes of fill_holes and dust (edtb200_fill_holes, edtb200_dust,
// include/edt_b200.h), after the union-find passes of edt_components.cuh.
//
// Union.  dust joins the voxels of every non-zero label with CcLabelKey, as connected_components does.
// fill_holes joins the background with CcHoleKey: a node is a voxel inside the volume whose label is 0, and
// every two neighbouring nodes are joined.  The tile pass fills the slots of a tile that lie outside the volume
// with K::none(), so the key carries its own node bit instead of the label: none() is a non-node although its
// "label" would read 0.  Either way P[v] is a node of v's component once the union has run, and cc_find gives
// its root, the component's least index (edt_components.cuh).
//
// Tally (one thread per voxel).  Every node v sets P[v] = root(v) and adds 1 to size[root] (uint32: volumes
// have fewer than 2^32 voxels), one atomicAdd per run of equal roots in a warp (__match_any_sync).  For
// fill_holes, a node on a face of its volume sets OPEN in state[root], and a node whose neighbour under the
// connectivity has a label L != 0 claims L at the root: atomicCAS(&claim[root], 0, L) on LabelOf::wide, and a
// return that is neither 0 nor L sets MIXED.  The result does not depend on the order of the races:
//   - size is a sum of ones and OPEN an OR of face bits, both commutative;
//   - the first CAS on a root that succeeds writes some claimed L1, and claim[root] never changes again.  If
//     every claimed label is L1, every CAS returns 0 or L1 and MIXED stays clear, so claim[root] is that one
//     label.  If some thread claims L2 != L1, its CAS fails (only one succeeds, and it wrote L1) and returns
//     L1, so it sets MIXED.  So MIXED is set exactly when the set of claimed labels has two or more elements,
//     and claim[root] is the single element whenever MIXED is clear -- the only case in which it is read.
//   - a thread that reads its root's state already OPEN or MIXED, or its claim already equal to L (or another
//     non-zero label: then it sets MIXED without a CAS), skips the CAS: it cannot change what apply reads.
// Apply (one thread per voxel).  fill_holes: a labelled voxel keeps its label; a background voxel whose root
// is neither OPEN nor MIXED, has a claim and (with max_size) a size of at most max_size takes the claim; every
// other voxel is 0.  dust: a labelled voxel keeps its label when (size[root] >= threshold) != invert, and is 0
// otherwise.  The filled voxels are counted per volume by a block reduction and one atomicAdd per block.
#pragma once
#include "edt_components.cuh"

namespace edtb200 {

constexpr uint32_t kHoleOpen = 1, kHoleMixed = 2;     // bits of state[root]
constexpr uint64_t kHoleNoBound = ~(uint64_t)0;       // fill_holes without max_size

struct HoleArgs {
  CcArgs cc;
  uint32_t* size;                   // null: fill_holes without max_size
  void* claim;                      // fill_holes: LabelOf<LB>::wide per voxel
  uint8_t* state;                   // fill_holes: OPEN / MIXED per voxel, 4-byte aligned and padded
  uint64_t bound;                   // fill_holes: max_size (kHoleNoBound: none); dust: threshold
  bool invert;
  unsigned long long* counts;       // fill_holes: voxels filled per volume, or null
  int64_t chunks;                   // blocks of kCcChunk voxels per volume (apply)
};

// The key of fill_holes: a node is a voxel inside the volume with label 0; all nodes are joined.
template <int LB> struct CcHoleKey {
  struct type { uint8_t node; };
  static __device__ __forceinline__ type load(const CcArgs& a, int64_t i) { return {cc_label<LB>(a, i) == 0}; }
  static __device__ __forceinline__ type none() { return {0}; }
  static __device__ __forceinline__ bool node(type k) { return k.node != 0; }
  static __device__ __forceinline__ bool joined(type, type) { return true; }
};

// Sets `bit` in the byte state[g] (an atomicOr on its aligned 4-byte word).
__device__ __forceinline__ void hole_flag(uint8_t* state, int64_t g, uint32_t bit) {
  atomicOr(reinterpret_cast<uint32_t*>(state) + (g >> 2), bit << (8 * (int)(g & 3)));
}

// Tally pass.  Fill: the nodes are the background voxels (P != kCcNone), else the labelled ones.  The loop's
// base is warp-uniform, so every lane of a warp reaches __match_any_sync together.
template <int LB, bool Fill>
__global__ void __launch_bounds__(kCcThreads, 4) holes_tally_kernel(HoleArgs h) {
  using Wide = typename LabelOf<LB>::wide;
  const CcArgs& a = h.cc;
  const int hy = a.ndim >= 2, hz = a.ndim >= 3;
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x - lane); base < a.total; base += stride) {
    const int64_t i = base + lane;
    unsigned long long g = ~0ull;                     // the root's index in the stack; all ones: not a node
    if (i < a.total && __ldcg(a.parent + i) != kCcNone) {
      const int64_t v = i / a.vol, local = i - v * a.vol;
      const uint32_t r = cc_find(a.parent + v * a.vol, (uint32_t)local);
      if (__ldcg(a.parent + i) != r) a.parent[i] = r;
      g = (unsigned long long)(v * a.vol + r);
      if constexpr (Fill) {
        const int64_t row = local / a.sx, x = local - row * a.sx, z = row / a.sy, y = row - z * a.sy;
        const bool face = x == 0 || x == a.sx - 1 || (hy && (y == 0 || y == a.sy - 1)) || (hz && (z == 0 || z == a.sz - 1));
        uint32_t st = __ldcg(reinterpret_cast<const uint32_t*>(h.state) + (g >> 2)) >> (8 * (int)(g & 3));
        if (face && !(st & kHoleOpen)) {
          hole_flag(h.state, (int64_t)g, kHoleOpen);
          st |= kHoleOpen;
        }
        Wide* claim = static_cast<Wide*>(h.claim) + g;
        Wide last = 0;                                 // the last label this voxel claimed
        for (int dz = -hz; dz <= hz && !(st & (kHoleOpen | kHoleMixed)); ++dz)
          for (int dy = -hy; dy <= hy; ++dy)
            for (int dx = -1; dx <= 1; ++dx) {
              if (!cc_offset(a, dz, dy, dx, false)) continue;
              const int64_t ux = x + dx, uy = y + dy, uz = z + dz;
              if (ux < 0 || ux >= a.sx || uy < 0 || uy >= a.sy || uz < 0 || uz >= a.sz) continue;
              const Wide lab = (Wide)cc_label<LB>(a, v * a.vol + (uz * a.sy + uy) * a.sx + ux);
              if (lab == 0 || lab == last || (st & kHoleMixed)) continue;
              last = lab;
              Wide c = __ldcg(claim);
              if (c == 0) c = atomicCAS(claim, (Wide)0, lab);
              if (c != 0 && c != lab) {
                hole_flag(h.state, (int64_t)g, kHoleMixed);
                st |= kHoleMixed;
              }
            }
      }
    }
    if (h.size) {
      const unsigned peers = __match_any_sync(0xffffffffu, g);
      if (g != ~0ull && lane == __ffs(peers) - 1) atomicAdd(h.size + g, (uint32_t)__popc(peers));
    }
  }
}

// Apply pass: one block per kCcChunk voxels of one volume (grid-stride over the stack's chunks).
template <int LB, bool Fill>
__global__ void __launch_bounds__(kCcThreads, 4) holes_apply_kernel(HoleArgs h, typename LabelOf<LB>::type* __restrict__ out) {
  using T = typename LabelOf<LB>::type;
  using Wide = typename LabelOf<LB>::wide;
  using Reduce = cub::BlockReduce<unsigned long long, kCcThreads>;
  __shared__ typename Reduce::TempStorage tmp;
  const CcArgs& a = h.cc;
  const T* labels = static_cast<const T*>(a.labels);
  const int64_t nblocks = h.chunks * (a.total / a.vol);
  for (int64_t b = blockIdx.x; b < nblocks; b += gridDim.x) {
    const int64_t v = b / h.chunks, c = b - v * h.chunks;
    const int64_t lo = v * a.vol + c * kCcChunk, hi = v * a.vol + (c * kCcChunk + kCcChunk < a.vol ? c * kCcChunk + kCcChunk : a.vol);
    unsigned long long filled = 0;
    for (int64_t i = lo + threadIdx.x; i < hi; i += kCcThreads) {
      const T lab = labels[i];
      T res = lab;
      if (Fill ? lab == 0 : lab != 0) {
        const int64_t g = v * a.vol + a.parent[i];
        if constexpr (Fill) {
          const Wide claim = static_cast<const Wide*>(h.claim)[g];
          if (!(h.state[g] & (kHoleOpen | kHoleMixed)) && claim != 0 && (!h.size || h.size[g] <= h.bound)) {
            res = (T)claim;
            ++filled;
          }
        } else if (((uint64_t)h.size[g] >= h.bound) == h.invert) {
          res = 0;
        }
      }
      out[i] = res;
    }
    if (Fill && h.counts) {
      filled = Reduce(tmp).Sum(filled);
      if (threadIdx.x == 0 && filled) atomicAdd(h.counts + v, filled);
      __syncthreads();                 // tmp is reused by the next chunk
    }
  }
}

}  // namespace edtb200
