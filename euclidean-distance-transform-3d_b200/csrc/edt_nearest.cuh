// edt_nearest.cuh -- the k nearest distinct labels of every voxel within a distance
// (edtb200_nearest_labels, include/edt_b200.h, DESIGN.md section "Nearest labels").
//
// The state between passes is, per voxel, a list of at most K (value, label) pairs with distinct labels,
// sorted by value and then by the label read as an unsigned integer, every value at most the bound B;
// an empty slot is (+inf, 0).  It lives in HBM as K float planes and K label planes, and each pass writes
// it out of place.  Every pass inserts candidates into a voxel's list with NearList::insert (a label keeps
// its least value, the list keeps the K least pairs), and walks its window outwards, d = 1, 2, ... R,
// stopping once fl32(w2 d^2) -- the least any farther candidate can be -- EXCEEDS the K-th value: a tie
// can still change the label in slot K, so reaching it is not enough.
//
// Kernels (templated on <label bytes, K>):
//   nearest_x_kernel        X pass.  A CTA stages kNearXThreads consecutive voxels of the x-fastest
//       volume plus R labels either side in shared memory (coalesced; rows of any length, a stack's
//       volumes back to back), and each thread walks the row of its voxel: the voxel itself at 0 when
//       its label is non-zero, and every non-zero label d samples away at fl32(w2 d^2).
//   nearest_window_kernel   Y / Z passes.  Lanes on 32 adjacent lines, a warp per row at a time, as
//       window_tiles (edt_bounded.cuh) walks them.  Row i starts from its own list, and row i +- d adds its
//       entries, each v as fl32(fl64(w2 d^2) + fl64(v)).  Staged: the tile's kNearRows rows and R rows
//       either side are staged in shared memory ((kNearRows + 2R) 32 K (4 + label bytes) bytes); Global:
//       the window is read from global memory through L1.  Both run the same walk and insert.
// The last pass writes sqrtf of each value when asked (correctly rounded, as edt does).
#pragma once
#include "edt_host.h"

namespace edtb200 {

constexpr int kNearXThreads = 256;      // voxels per X tile
constexpr int kNearRows = 64;           // rows of a later-pass tile along the pass axis
constexpr int kNearWarps = 8;           // a warp per row at a time, lanes on 32 adjacent lines

// Shared memory of a staged later-pass tile.
__host__ __device__ constexpr size_t nearest_smem_bytes(int radius, int k, int label_bytes) {
  return (size_t)(kNearRows + 2 * radius) * 32 * (size_t)k * (sizeof(float) + (size_t)label_bytes);
}

// The sorted list of one voxel.  Slots are compile-time indices only, so the list stays in registers.
template <class LT, int K>
struct NearList {
  float v[K];
  LT l[K];

  __device__ __forceinline__ static bool less(float a, LT la, float b, LT lb) { return a < b || (a == b && la < lb); }

  __device__ __forceinline__ void clear() {
#pragma unroll
    for (int q = 0; q < K; ++q) { v[q] = __int_as_float(0x7f800000); l[q] = 0; }
  }
  // The K-th value: +inf while a slot is empty.
  __device__ __forceinline__ float kth() const { return v[K - 1]; }

  // Offers (c, lab), c <= the bound, lab != 0.  A label already held keeps the smaller value; otherwise
  // the pair takes the last slot when it is less than the pair there.  Either way the slot it takes held
  // a greater pair, so one backward bubble restores the order.
  __device__ __forceinline__ void insert(float c, LT lab) {
    if (!less(c, lab, v[K - 1], l[K - 1])) return;
    int at = K - 1;
#pragma unroll
    for (int q = 0; q < K; ++q)
      if (l[q] == lab && v[q] != __int_as_float(0x7f800000)) {
        if (v[q] <= c) return;
        at = q;
      }
#pragma unroll
    for (int q = 0; q < K; ++q)
      if (q == at) { v[q] = c; l[q] = lab; }
#pragma unroll
    for (int q = K - 1; q > 0; --q)
      if (less(v[q], l[q], v[q - 1], l[q - 1])) {
        const float tv = v[q]; v[q] = v[q - 1]; v[q - 1] = tv;
        const LT tl = l[q]; l[q] = l[q - 1]; l[q - 1] = tl;
      }
  }

  // Writes slot q to planes vout / lout (q * plane apart) at voxel `at`; root: sqrtf of the values.
  __device__ __forceinline__ void store(float* __restrict__ vout, LT* __restrict__ lout, int64_t plane, int64_t at,
                                        bool root) const {
#pragma unroll
    for (int q = 0; q < K; ++q) {
      vout[q * plane + at] = root ? __fsqrt_rn(v[q]) : v[q];
      lout[q * plane + at] = l[q];
    }
  }
};

// fl32(fl64(w2 d^2)): d^2 <= 2^16 and w2 has 24 significant bits, so the product is exact in double.
__device__ __forceinline__ double near_wall(double w2, int d) { return __dmul_rn(w2, (double)(d * d)); }

// X pass over `total` voxels of rows of sx samples (x-fastest, a stack's volumes back to back).
template <int Bytes, int K>
__global__ void __launch_bounds__(kNearXThreads)
nearest_x_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, float* __restrict__ vout,
                 typename LabelOf<Bytes>::type* __restrict__ lout, int64_t total, int64_t sx, double w2, int radius,
                 float bound, bool root) {
  using LT = typename LabelOf<Bytes>::type;
  extern __shared__ __align__(16) unsigned char near_x_smem[];
  LT* s = reinterpret_cast<LT*>(near_x_smem);
  const int span = kNearXThreads + 2 * radius;
  for (int64_t b0 = (int64_t)blockIdx.x * kNearXThreads; b0 < total; b0 += (int64_t)gridDim.x * kNearXThreads) {
    __syncthreads();                                   // the previous tile is no longer read
    for (int t = threadIdx.x; t < span; t += kNearXThreads) {
      const int64_t g = b0 - radius + t;
      s[t] = g >= 0 && g < total ? labels[g] : (LT)0;
    }
    __syncthreads();
    const int64_t i = b0 + threadIdx.x;
    if (i >= total) continue;
    const int64_t x = i % sx;
    const int me = threadIdx.x + radius;
    NearList<LT, K> list;
    list.clear();
    if (s[me] != 0) { list.v[0] = 0.0f; list.l[0] = s[me]; }
    for (int d = 1; d <= radius; ++d) {
      const float wall = __double2float_rn(near_wall(w2, d));
      if (wall > list.kth() || wall > bound) break;
      if (x - d >= 0 && s[me - d] != 0) list.insert(wall, s[me - d]);
      if (x + d < sx && s[me + d] != 0) list.insert(wall, s[me + d]);
    }
    list.store(vout, lout, total, i, root);
  }
}

// Y / Z pass over the lines of g, lists in (vin, lin) -> (vout, lout), planes `plane` voxels apart.
template <int Bytes, int K, bool Staged>
__global__ void __launch_bounds__(kNearWarps * 32)
nearest_window_kernel(const float* __restrict__ vin, const typename LabelOf<Bytes>::type* __restrict__ lin,
                      float* __restrict__ vout, typename LabelOf<Bytes>::type* __restrict__ lout, int64_t plane,
                      LineGeom g, double w2, int radius, float bound, bool root, int64_t row_tiles, int64_t tiles) {
  using LT = typename LabelOf<Bytes>::type;
  extern __shared__ __align__(16) unsigned char near_smem[];
  const int span = kNearRows + 2 * radius;
  float* fs = reinterpret_cast<float*>(near_smem);
  LT* ls = reinterpret_cast<LT*>(near_smem + sizeof(float) * (size_t)K * 32 * span);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = g.n;
  const int64_t inner_tiles = (g.inner_count + 31) >> 5;
  const int64_t stride = g.line_stride;
  const float inf = __int_as_float(0x7f800000);

  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int64_t rest = t / row_tiles;
    const int i0 = (int)(t - rest * row_tiles) * kNearRows;
    const int64_t outer = rest / inner_tiles;
    const int64_t j = (rest - outer * inner_tiles) * 32 + lane;
    const bool live = j < g.inner_count;
    const int64_t base = outer * g.outer_stride + j;
    const int s0 = i0 - radius;                        // the row in shared slot 0
    if constexpr (Staged) {
      const int lo = max(s0, 0), hi = min(i0 + kNearRows + radius, n);
      __syncthreads();                                 // the previous tile is no longer read
      if (live)
        for (int r = lo + warp; r < hi; r += kNearWarps)
#pragma unroll
          for (int q = 0; q < K; ++q) {
            fs[((r - s0) * K + q) * 32 + lane] = vin[q * plane + base + (int64_t)r * stride];
            ls[((r - s0) * K + q) * 32 + lane] = lin[q * plane + base + (int64_t)r * stride];
          }
      __syncthreads();
    }
    if (!live) continue;
    auto value = [&](int r, int q) {
      if constexpr (Staged) return fs[((r - s0) * K + q) * 32 + lane];
      else return vin[q * plane + base + (int64_t)r * stride];
    };
    auto label = [&](int r, int q) {
      if constexpr (Staged) return ls[((r - s0) * K + q) * 32 + lane];
      else return lin[q * plane + base + (int64_t)r * stride];
    };
    const int iend = min(i0 + kNearRows, n);
    for (int i = i0 + warp; i < iend; i += kNearWarps) {
      NearList<LT, K> list;
#pragma unroll
      for (int q = 0; q < K; ++q) { list.v[q] = value(i, q); list.l[q] = label(i, q); }
      for (int d = 1; d <= radius; ++d) {
        const double wall64 = near_wall(w2, d);
        const float wall = __double2float_rn(wall64);
        if (wall > list.kth() || wall > bound) break;
#pragma unroll
        for (int side = 0; side < 2; ++side) {
          const int r = side ? i + d : i - d;
          if (r < 0 || r >= n) continue;
#pragma unroll
          for (int q = 0; q < K; ++q) {
            const float v = value(r, q);
            if (v == inf) break;                       // the rest of row r's list is empty
            const float c = __double2float_rn(__dadd_rn(wall64, (double)v));
            if (c > list.kth() || c > bound) break;    // row r's later entries are no less
            list.insert(c, label(r, q));
          }
        }
      }
      list.store(vout, lout, plane, base + (int64_t)i * stride, root);
    }
  }
}

namespace host {

template <int Bytes, int K>
int launch_nearest_x_k(const void* labels, float* vout, void* lout, int64_t total, int64_t sx, float w, int radius,
                       float bound, bool root, DeviceCache& dc, cudaStream_t stream) {
  using LT = typename LabelOf<Bytes>::type;
  const size_t smem = (size_t)(kNearXThreads + 2 * radius) * sizeof(LT);
  int64_t blocks = (total + kNearXThreads - 1) / kNearXThreads;
  const int64_t cap = (int64_t)dc.sm_count * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  nearest_x_kernel<Bytes, K><<<(unsigned)blocks, kNearXThreads, smem, stream>>>(
      static_cast<const LT*>(labels), vout, static_cast<LT*>(lout), total, sx, (double)(w * w), radius, bound, root);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

template <int Bytes, int K>
int launch_nearest_window_k(const float* vin, const void* lin, float* vout, void* lout, int64_t plane,
                            const LineGeom& g, float w, int radius, bool staged, float bound, bool root,
                            DeviceCache& dc, cudaStream_t stream) {
  using LT = typename LabelOf<Bytes>::type;
  const size_t smem = staged ? nearest_smem_bytes(radius, K, Bytes) : 0;
  if (smem > (size_t)dc.max_smem_optin)
    return fail(EDTB200_ELIMIT, "a staged window of radius %d exceeds the shared memory", radius);
  auto kern = staged ? nearest_window_kernel<Bytes, K, true> : nearest_window_kernel<Bytes, K, false>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t row_tiles = (g.n + kNearRows - 1) / kNearRows;
  const int64_t tiles = ((g.inner_count + 31) >> 5) * row_tiles * g.outer_count;
  int per_sm = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kNearWarps * 32, smem));
  int64_t blocks = (int64_t)dc.sm_count * (per_sm > 0 ? per_sm : 1);      // one persistent wave
  if (blocks > tiles) blocks = tiles;
  if (blocks < 1) blocks = 1;
  kern<<<(unsigned)blocks, kNearWarps * 32, smem, stream>>>(vin, static_cast<const LT*>(lin), vout,
                                                            static_cast<LT*>(lout), plane, g, (double)(w * w), radius,
                                                            bound, root, row_tiles, tiles);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// f(integral_constant<int, K>) for K = k in 1..4.
template <class F>
int with_k(int k, F&& f) {
  switch (k) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 3: return f(std::integral_constant<int, 3>{});
    case 4: return f(std::integral_constant<int, 4>{});
  }
  return fail(EDTB200_EINVAL, "k must be 1, 2, 3 or 4 (got %d)", k);
}

}  // namespace host
}  // namespace edtb200
