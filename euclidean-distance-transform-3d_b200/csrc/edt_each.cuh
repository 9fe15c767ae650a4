// Per-label views of a finished transform, on the device (SURVEY.md section 8f-2).
//
// The reference's headline use case is "one multi-label transform, then one image per label"
// (README.md:23, 204): edt.each (src/edt.pyx:951-994) extracts run lists per label
// (extract_runs, src/edt_voxel_graph.hpp:238-275) and copies each label's runs of the distance
// image into a blank image (transfer_run_voxels, :296-310).  What its callers (TEASAR
// skeletonisation) consume per label is the masked image, its maximum and where that maximum is.
//
// Here, with labels and distances resident on the GPU:
//   label_stats_kernel    ONE pass over (labels, dt): per label its voxel count, bounding box and
//                         maximum distance, into an open-addressing hash table keyed by the label
//                         (label 0 = background is skipped and doubles as the empty-slot marker);
//                         lanes of a warp that hold the same label are combined first
//                         (__match_any_sync), so a warp issues one set of atomics per label it sees;
//   label_argmax_kernel   second pass: the smallest linear index at which each label attains its
//                         maximum (what the reference's callers get from np.argmax on the image);
//   label_extract_kernel  dt masked to one label, restricted to that label's bounding box (the
//                         equivalent of transfer_run_voxels); the same kernel erases a box.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "edt_kernels.cuh"

namespace edtb200 {

struct LabelTable {
  unsigned long long* keys;      // [capacity]  0 = empty
  unsigned long long* count;     // [capacity]
  unsigned int* maxbits;         // [capacity]  ordered-int image of the maximum distance
  long long* argmax;             // [capacity]
  int* box;                      // [capacity][6]  x0 y0 z0 x1 y1 z1 (inclusive)
  int capacity;                  // power of two
  int* overflow;                 // raised when the table is full
};

// float -> unsigned int whose unsigned order is the float order (works for negatives too).
__device__ __forceinline__ unsigned int ordered_bits(float v) {
  const unsigned int u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float from_ordered_bits(unsigned int o) {
  const unsigned int u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, sizeof(f));
  return f;
#endif
}

__device__ __forceinline__ unsigned int hash_label(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return (unsigned int)k;
}

// Slot of `key` (inserting it if new), or -1 when the table is full.
__device__ __forceinline__ int table_slot(const LabelTable t, unsigned long long key, bool insert) {
  const unsigned int mask = (unsigned int)t.capacity - 1u;
  unsigned int s = hash_label(key) & mask;
  for (int probe = 0; probe < t.capacity; ++probe, s = (s + 1u) & mask) {
    unsigned long long cur = t.keys[s];
    if (cur == key) return (int)s;
    if (cur == 0ull) {
      if (!insert) return -1;
      cur = atomicCAS(&t.keys[s], 0ull, key);
      if (cur == 0ull || cur == key) return (int)s;
    }
  }
  return -1;
}

template <int Bytes>
__global__ void __launch_bounds__(256)
label_stats_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, const float* __restrict__ dt,
                   int64_t total, int sx, int sy, LabelTable t) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  // whole warps walk the volume together (the tail is padded with background)
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); base < total; base += stride) {
    const int64_t idx = base + lane;
    unsigned long long key = 0ull;
    float d = 0.0f;
    if (idx < total) { key = (unsigned long long)labels[idx]; d = dt[idx]; }
    const unsigned fg = __ballot_sync(full, key != 0ull);
    if (!fg) continue;
    if (key == 0ull) continue;                       // background lanes drop out; `fg` names the rest
    const unsigned same = __match_any_sync(fg, key);
    const int64_t plane = (int64_t)sx * sy;              // may exceed 2^31 (only each axis fits an int)
    const int z = (int)(idx / plane);
    const int64_t rem = idx - (int64_t)z * plane;
    const int y = (int)(rem / sx), x = (int)(rem - (int64_t)y * sx);
    const unsigned int bits = ordered_bits(d);
    const unsigned int mx = __reduce_max_sync(same, bits);
    const int x0 = __reduce_min_sync(same, x), x1 = __reduce_max_sync(same, x);
    const int y0 = __reduce_min_sync(same, y), y1 = __reduce_max_sync(same, y);
    const int z0 = __reduce_min_sync(same, z), z1 = __reduce_max_sync(same, z);
    if (lane == __ffs(same) - 1) {                   // one lane per label present in the warp
      const int s = table_slot(t, key, true);
      if (s < 0) { *t.overflow = 1; continue; }
      atomicAdd(&t.count[s], (unsigned long long)__popc(same));
      atomicMax(&t.maxbits[s], mx);
      int* b = t.box + 6 * s;
      atomicMin(b + 0, x0); atomicMin(b + 1, y0); atomicMin(b + 2, z0);
      atomicMax(b + 3, x1); atomicMax(b + 4, y1); atomicMax(b + 5, z1);
    }
  }
}

template <int Bytes>
__global__ void __launch_bounds__(256)
label_argmax_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, const float* __restrict__ dt,
                    int64_t total, LabelTable t) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += stride) {
    const unsigned long long key = (unsigned long long)labels[idx];
    if (key == 0ull) continue;
    const int s = table_slot(t, key, false);
    if (s < 0) continue;
    if (ordered_bits(dt[idx]) == t.maxbits[s]) atomicMin(&t.argmax[s], (long long)idx);
  }
}

__global__ void label_table_init_kernel(LabelTable t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= t.capacity) return;
  t.keys[i] = 0ull; t.count[i] = 0ull; t.maxbits[i] = 0u; t.argmax[i] = 0x7fffffffffffffffll;
  int* b = t.box + 6 * i;
  b[0] = b[1] = b[2] = 0x7fffffff; b[3] = b[4] = b[5] = -1;
}

// maxbits (ordered-int image) -> the float it stands for, in place; empty slots get 0.
__global__ void label_table_finish_kernel(LabelTable t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= t.capacity) return;
  const float v = t.keys[i] ? from_ordered_bits(t.maxbits[i]) : 0.0f;
  t.maxbits[i] = __float_as_uint(v);
}

// out[box] = (labels == key) ? dt : 0 over the box [x0..x1] x [y0..y1] x [z0..z1]; with
// erase != 0 the box is zeroed instead.  Rows of the box are walked by whole warps.
template <int Bytes>
__global__ void __launch_bounds__(256)
label_extract_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, const float* __restrict__ dt,
                     float* __restrict__ out, int sx, int sy, int x0, int y0, int z0, int bx, int by, int bz,
                     unsigned long long key, int erase) {
  const int64_t rows = (int64_t)by * bz;
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t row = warp; row < rows; row += nwarps) {
    const int zz = (int)(row / by), yy = (int)(row - (int64_t)zz * by);
    const int64_t base = ((int64_t)(z0 + zz) * sy + (y0 + yy)) * sx + x0;
    for (int xx = lane; xx < bx; xx += 32) {
      float v = 0.0f;
      if (!erase && (unsigned long long)labels[base + xx] == key) v = dt[base + xx];
      out[base + xx] = v;
    }
  }
}

}  // namespace edtb200
