// edt_surface.cuh -- the kernels of the surface distances between two label volumes
// (edtb200_surface_count / edtb200_surface_distances, include/edt_b200.h; DESIGN.md section 5).
//
// A surface voxel of key k in volume v is a voxel of label k with a face neighbour of another label,
// or on a face of its volume (scipy's mask ^ binary_erosion(mask), border_value 0).  A slot is a
// (volume, key, direction) triple, numbered s = (volume * nkeys + key) * 2 + direction; direction 0 is
// A->B (a's surface voxels, distances to b's surface), 1 is B->A.  Segment s of the output holds
// slot s's distances.  The kernels run over the volumes a range of slots [s0, s1) touches:
//   surface_mask_kernel    writes 0 into slot s's mask (set to 1 before) at every surface voxel of
//                          the volume the slot measures TO: b for A->B, a for B->A;
//   surface_count_kernel   counts the surface voxels of the volume it measures FROM into counts[s];
//   surface_gather_kernel  appends, at those voxels, slot s's distance to segment s.
// Labels are compared as raw bits; keys are sorted, distinct and non-zero, looked up by binary search
// in shared memory (global memory when they do not fit 48 KiB).  Face neighbours are read directly:
// the x neighbours come from the same coalesced rows, the y and z ones from L2.
#pragma once
#include "edt_host.h"

namespace edtb200 {

constexpr size_t kSurfaceKeySmem = 48 * 1024;    // keys beyond this are searched in global memory

// The key index of voxel i (at x, y, z of its volume) of `vol` when it is a surface voxel of one of
// the keys, else -1.  Interior voxels are rejected on their neighbours before any search.
template <class LT>
__device__ __forceinline__ int64_t surface_key(const LT* __restrict__ vol, int64_t i, int64_t x, int64_t y, int64_t z,
                                               const SurfaceSlots& g, const LT* keys) {
  const LT v = vol[i];
  bool face = x == 0 || x == g.sx - 1 || vol[i - 1] != v || vol[i + 1] != v;
  if (!face && g.ndim >= 2) face = y == 0 || y == g.sy - 1 || vol[i - g.sx] != v || vol[i + g.sx] != v;
  if (!face && g.ndim >= 3) {
    const int64_t plane = g.sx * g.sy;
    face = z == 0 || z == g.sz - 1 || vol[i - plane] != v || vol[i + plane] != v;
  }
  if (!face) return -1;
  int64_t lo = 0, hi = g.nkeys;                  // the first key >= v
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (keys[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo < g.nkeys && keys[lo] == v ? lo : -1;
}

// The keys where the kernel searches them: staged in shared memory when `in_smem`.
template <class LT>
__device__ __forceinline__ const LT* stage_keys(const LT* __restrict__ keys, int64_t nkeys, int in_smem) {
  extern __shared__ __align__(16) unsigned char surface_smem[];
  if (!in_smem) return keys;
  LT* s = reinterpret_cast<LT*>(surface_smem);
  for (int64_t k = threadIdx.x; k < nkeys; k += blockDim.x) s[k] = keys[k];
  __syncthreads();
  return s;
}

// Where voxel i of the stack lies: its volume and its x, y, z in it.
struct SurfaceVoxel {
  int64_t v, local, x, y, z;
};
__device__ __forceinline__ SurfaceVoxel surface_voxel(int64_t i, const SurfaceSlots& g) {
  SurfaceVoxel p;
  p.v = i / g.vol;
  p.local = i - p.v * g.vol;
  const int64_t row = p.local / g.sx;
  p.x = p.local - row * g.sx;
  p.z = row / g.sy;
  p.y = row - p.z * g.sy;
  return p;
}

template <int Bytes>
__global__ void __launch_bounds__(256)
surface_mask_kernel(const typename LabelOf<Bytes>::type* __restrict__ a, const typename LabelOf<Bytes>::type* __restrict__ b,
                    const typename LabelOf<Bytes>::type* __restrict__ keys_g, SurfaceSlots g, int keys_in_smem,
                    uint8_t* __restrict__ mask) {
  using LT = typename LabelOf<Bytes>::type;
  const LT* keys = stage_keys(keys_g, g.nkeys, keys_in_smem);
  const int64_t end = g.v1 * g.vol;
  for (int64_t i = g.v0 * g.vol + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < end;
       i += (int64_t)gridDim.x * blockDim.x) {
    const SurfaceVoxel p = surface_voxel(i, g);
    for (int d = 0; d < 2; ++d) {
      const int64_t k = surface_key(d == 0 ? b : a, i, p.x, p.y, p.z, g, keys);
      const int64_t s = (p.v * g.nkeys + k) * 2 + d;
      if (k >= 0 && s >= g.s0 && s < g.s1) mask[(s - g.s0) * g.vol + p.local] = 0;
    }
  }
}

// One append of `seg` (-1: none) per lane, aggregated over the lanes of the warp that share a segment:
// one atomicAdd on cursor[seg - s0] per segment and warp.  Every lane of the warp calls it.  Returns the
// lane's position in the output (unspecified for seg -1).
__device__ __forceinline__ unsigned long long append_slot(int64_t seg, int64_t s0, unsigned long long* cursor) {
  const int lane = threadIdx.x & 31;
  const unsigned peers = __match_any_sync(0xffffffffu, (unsigned long long)seg);
  const int leader = __ffs(peers) - 1;
  unsigned long long at = 0;
  if (seg >= 0 && lane == leader) at = atomicAdd(cursor + (seg - s0), (unsigned long long)__popc(peers));
  at = __shfl_sync(peers, at, leader);
  return at + __popc(peers & ((1u << lane) - 1u));
}

// The walk of surface_count_kernel (dist null) and surface_gather_kernel: the loop runs a whole warp at
// a time, so that every lane takes part in append_slot.
template <int Bytes>
__device__ __forceinline__ void surface_append(const typename LabelOf<Bytes>::type* __restrict__ a,
                                               const typename LabelOf<Bytes>::type* __restrict__ b,
                                               const typename LabelOf<Bytes>::type* __restrict__ keys_g,
                                               const SurfaceSlots& g, int keys_in_smem, const float* __restrict__ dist,
                                               unsigned long long* cursor, float* __restrict__ values) {
  using LT = typename LabelOf<Bytes>::type;
  const LT* keys = stage_keys(keys_g, g.nkeys, keys_in_smem);
  const int lane = threadIdx.x & 31;
  const int64_t end = g.v1 * g.vol;
  for (int64_t w = g.v0 * g.vol + (int64_t)blockIdx.x * blockDim.x + (threadIdx.x - lane); w < end;
       w += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = w + lane;
    SurfaceVoxel p{};
    if (i < end) p = surface_voxel(i, g);
    for (int d = 0; d < 2; ++d) {
      int64_t s = -1;
      if (i < end) {
        const int64_t k = surface_key(d == 0 ? a : b, i, p.x, p.y, p.z, g, keys);
        s = (p.v * g.nkeys + k) * 2 + d;
        if (k < 0 || s < g.s0 || s >= g.s1) s = -1;
      }
      const unsigned long long at = append_slot(s, g.s0, cursor);
      if (dist && s >= 0) values[at] = dist[(s - g.s0) * g.vol + p.local];
    }
  }
}

template <int Bytes>
__global__ void __launch_bounds__(256)
surface_count_kernel(const typename LabelOf<Bytes>::type* __restrict__ a, const typename LabelOf<Bytes>::type* __restrict__ b,
                     const typename LabelOf<Bytes>::type* __restrict__ keys_g, SurfaceSlots g, int keys_in_smem,
                     unsigned long long* counts) {
  surface_append<Bytes>(a, b, keys_g, g, keys_in_smem, nullptr, counts, nullptr);
}

template <int Bytes>
__global__ void __launch_bounds__(256)
surface_gather_kernel(const typename LabelOf<Bytes>::type* __restrict__ a, const typename LabelOf<Bytes>::type* __restrict__ b,
                      const typename LabelOf<Bytes>::type* __restrict__ keys_g, SurfaceSlots g, int keys_in_smem,
                      const float* __restrict__ dist, unsigned long long* cursor, float* __restrict__ values) {
  surface_append<Bytes>(a, b, keys_g, g, keys_in_smem, dist, cursor, values);
}

namespace host {

inline unsigned surface_blocks(const SurfaceSlots& g, const DeviceCache& dc) {
  const int64_t blocks = ((g.v1 - g.v0) * g.vol + 255) / 256, cap = (int64_t)dc.sm_count * 8;
  return (unsigned)(blocks < 1 ? 1 : blocks > cap ? cap : blocks);
}

template <int Bytes>
int launch_surface(const void* a, const void* b, const void* keys, const SurfaceSlots& g, uint8_t* mask,
                   const float* dist, unsigned long long* cursor, float* values, DeviceCache& dc, cudaStream_t stream) {
  using LT = typename LabelOf<Bytes>::type;
  const size_t key_bytes = (size_t)g.nkeys * Bytes;
  const int in_smem = key_bytes <= kSurfaceKeySmem;
  const size_t smem = in_smem ? key_bytes : 0;
  const LT *la = static_cast<const LT*>(a), *lb = static_cast<const LT*>(b), *lk = static_cast<const LT*>(keys);
  if (mask)
    surface_mask_kernel<Bytes><<<surface_blocks(g, dc), 256, smem, stream>>>(la, lb, lk, g, in_smem, mask);
  else if (values)
    surface_gather_kernel<Bytes><<<surface_blocks(g, dc), 256, smem, stream>>>(la, lb, lk, g, in_smem, dist, cursor,
                                                                               values);
  else
    surface_count_kernel<Bytes><<<surface_blocks(g, dc), 256, smem, stream>>>(la, lb, lk, g, in_smem, cursor);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace host
}  // namespace edtb200

#define EDT_INSTANTIATE_SURFACE(B)                                                                            \
  template int edtb200::host::launch_surface<B>(const void*, const void*, const void*,                        \
                                                const edtb200::SurfaceSlots&, uint8_t*, const float*,         \
                                                unsigned long long*, float*, edtb200::host::DeviceCache&,     \
                                                cudaStream_t);
