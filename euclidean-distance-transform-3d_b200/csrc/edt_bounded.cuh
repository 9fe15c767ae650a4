// edt_bounded.cuh -- the kernels of the bounded transforms (max_distance, include/edt_b200.h).
//
// With a bound, a later-axis pass at row i only needs the samples v with w2 (i - v)^2 <= B (the
// largest float32 whose double is at most max_distance^2): a window of 2R + 1 rows.  The window
// kernel takes the minimum over it directly -- no hull, no vertex stack, no long-line scratch -- and
// writes every row whose value exceeds B as +inf.  Why that is exact is DESIGN.md section 5:
//   (a) wherever the true pass value is at most B, the pass returns it bit for bit;
//   (b) everywhere else it returns that true value or +inf.
// Passes that do not take the window kernel run the unbounded kernels unchanged, and
// bounded_cut_kernel applies the cut (and the last pass's sqrt / sign) afterwards.
#pragma once
#include "edt_host.h"

namespace edtb200 {

constexpr int kWindowRows = 64;       // rows of a tile along the pass axis
constexpr int kWindowWarps = 8;       // a warp per row at a time, lanes on 32 adjacent lines

// Shared memory of a window tile: kWindowRows + 2 radius rows of 32 distances and 32 labels.
inline size_t window_smem_bytes(int radius, int label_bytes) {
  return (size_t)(kWindowRows + 2 * radius) * 32 * (sizeof(float) + (size_t)label_bytes);
}

// ---------------------------------------------------------------------------------------
// Later-axis pass over a window of `radius` rows either side, out of place (fin -> fout).
// A CTA walks tiles of 32 adjacent lines (128-byte rows, as the tile kernel) by kWindowRows rows,
// staging the distances and labels of the tile's rows and `radius` rows either side in shared
// memory.  Row i of a line then takes the minimum of
//   its own sample, and for d = 1, 2, ... <= radius on each side while the run of i's label lasts,
//   the sample d rows away, c = w2 d^2 + f, formed as later_axis_long_kernel forms it (one fused
//   multiply-add, or from dbl_from on a double sum rounded once), and where the run ends within the
//   window its border term fl32(w2 d^2) (a face only with border_lo / border_hi);
// and stops early once fl32(w2 d^2) -- the least any farther candidate can be -- reaches the best so
// far.  A value above `bound` is written as +inf.  Sites: the codes later_axis_long_kernel writes
// (the winning row, site_direct for a border term, kSiteNone for +inf), so the resolver is shared.
// Epi: flags' sqrt / sign in the store (the last pass).
// The walk is window_tiles below; the kernels differ in their store only: later_axis_window_kernel
// writes the distance (and site code), later_axis_window_select_kernel the morphology's label or mask.
// ---------------------------------------------------------------------------------------
// store(at, best, site, label): row `at` of the pass has the value `best` (+inf above bound), won by
// `site`, and the label `label`.
template <int Bytes, class Store>
__device__ __forceinline__ void window_tiles(const typename LabelOf<Bytes>::type* __restrict__ labels,
                                             const float* __restrict__ fin, const LineGeom& g, float w2, int radius,
                                             int border_lo, int border_hi, int dbl_from, float bound,
                                             int64_t row_tiles, int64_t tiles, Store&& store) {
  using LT = typename LabelOf<Bytes>::type;
  extern __shared__ __align__(16) unsigned char window_smem[];
  const int span = kWindowRows + 2 * radius;
  float* fs = reinterpret_cast<float*>(window_smem);
  LT* ls = reinterpret_cast<LT*>(window_smem + sizeof(float) * 32 * (size_t)span);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = g.n;
  const int64_t inner_tiles = (g.inner_count + 31) >> 5;
  const int64_t stride = g.line_stride;
  const float inf = __int_as_float(0x7f800000);

  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int64_t rest = t / row_tiles;
    const int i0 = (int)(t - rest * row_tiles) * kWindowRows;
    const int64_t outer = rest / inner_tiles;
    const int64_t j = (rest - outer * inner_tiles) * 32 + lane;
    const bool live = j < g.inner_count;
    const int64_t base = outer * g.outer_stride + j;
    const int s0 = i0 - radius;                          // the row in shared slot 0
    const int lo = max(s0, 0), hi = min(i0 + kWindowRows + radius, n);
    __syncthreads();                                     // the previous tile is no longer read
    if (live) {
      for (int r = lo + warp; r < hi; r += kWindowWarps) {
        fs[(r - s0) * 32 + lane] = fin[base + (int64_t)r * stride];
        ls[(r - s0) * 32 + lane] = labels[base + (int64_t)r * stride];
      }
    }
    __syncthreads();
    if (!live) continue;
    const int iend = min(i0 + kWindowRows, n);
    for (int i = i0 + warp; i < iend; i += kWindowWarps) {
      const int si = i - s0;
      const LT mine = ls[si * 32 + lane];
      float best = fs[si * 32 + lane];
      int site = i;
      bool down = true, up = true;                       // the run of `mine` goes on that way
      for (int d = 1; d <= radius && (down || up); ++d) {
        const float wall = parabola_at(w2, d, 0.0f);
        if (wall >= best) break;
        if (down) {
          const int r = i - d;
          if (r < 0 || ls[(r - s0) * 32 + lane] != mine) {
            down = false;
            if ((r >= 0 || border_lo) && wall < best) { best = wall; site = site_direct(r); }
          } else {
            const float c = parabola_at(w2, d, fs[(r - s0) * 32 + lane], dbl_from);
            if (c < best) { best = c; site = r; }
          }
        }
        if (up) {
          const int r = i + d;
          if (r >= n || ls[(r - s0) * 32 + lane] != mine) {
            up = false;
            if ((r < n || border_hi) && wall < best) { best = wall; site = site_direct(r); }
          } else {
            const float c = parabola_at(w2, d, fs[(r - s0) * 32 + lane], dbl_from);
            if (c < best) { best = c; site = r; }
          }
        }
      }
      if (!(best <= bound)) best = inf;
      store(base + (int64_t)i * stride, best, site, mine);
    }
  }
}

template <int Bytes, bool Sites, bool Epi>
__global__ void __launch_bounds__(kWindowWarps * 32)
later_axis_window_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, const float* __restrict__ fin,
                         float* __restrict__ fout, int* __restrict__ codes, LineGeom g, float w2, int radius,
                         int border_lo, int border_hi, int flags, int dbl_from, float bound, int64_t row_tiles,
                         int64_t tiles) {
  using LT = typename LabelOf<Bytes>::type;
  const float inf = __int_as_float(0x7f800000);
  window_tiles<Bytes>(labels, fin, g, w2, radius, border_lo, border_hi, dbl_from, bound, row_tiles, tiles,
                      [&](int64_t at, float best, int site, LT mine) {
                        if constexpr (Sites) codes[at] = best < inf ? site : kSiteNone;
                        if constexpr (Epi) best = finish_value(best, mine == 0, flags);
                        fout[at] = best;
                      });
}

// The cut of a pass that did not take the window kernel (or of a 1-D transform's X pass): in place
// over `total` voxels, a value above `bound` becomes +inf (and its site code, when codes is given,
// kSiteNone), then flags' sqrt / sign.
template <int Bytes>
__global__ void __launch_bounds__(256)
bounded_cut_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, float* __restrict__ f,
                   int* __restrict__ codes, int64_t total, float bound, int flags) {
  const float inf = __int_as_float(0x7f800000);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float v = f[i];
    if (!(v <= bound)) {
      v = inf;
      if (codes) codes[i] = kSiteNone;
    }
    f[i] = flags ? finish_value(v, labels[i] == 0, flags) : v;
  }
}

namespace host {

template <int Bytes>
int launch_later_window(const void* labels, const float* fin, float* fout, int* codes, const LineGeom& g, float w,
                        int radius, int border_lo, int border_hi, int flags, PassArith arith, float bound,
                        DeviceCache& dc, cudaStream_t stream) {
  using LT = typename LabelOf<Bytes>::type;
  if (radius < 0 || radius > kWindowRadiusLimit) return fail(EDTB200_EINVAL, "window radius %d out of range", radius);
  const size_t smem = window_smem_bytes(radius, Bytes);
  if (smem > (size_t)dc.max_smem_optin) return fail(EDTB200_ELIMIT, "a window of radius %d exceeds the shared memory", radius);
  const int64_t row_tiles = (g.n + kWindowRows - 1) / kWindowRows;
  const int64_t tiles = ((g.inner_count + 31) >> 5) * row_tiles * g.outer_count;
  auto kern = codes ? (flags ? later_axis_window_kernel<Bytes, true, true> : later_axis_window_kernel<Bytes, true, false>)
                    : (flags ? later_axis_window_kernel<Bytes, false, true> : later_axis_window_kernel<Bytes, false, false>);
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kWindowWarps * 32, smem));
  int64_t blocks = (int64_t)dc.sm_count * (per_sm > 0 ? per_sm : 1);      // one persistent wave
  if (blocks > tiles) blocks = tiles;
  if (blocks < 1) blocks = 1;
  kern<<<(unsigned)blocks, kWindowWarps * 32, smem, stream>>>(
      static_cast<const LT*>(labels), fin, fout, codes, g, w * w, radius, border_lo, border_hi, flags,
      arith.exact ? 4096 : 0, bound, row_tiles, tiles);
  CUDA_TRY(cudaGetLastError());
  g_last_later = LaterLaunch{2, radius, 0, 0, 0, 0, flags != 0, !arith.exact};
  return 0;
}

template <int Bytes>
int launch_bounded_cut(const void* labels, float* f, int* codes, int64_t total, float bound, int flags,
                       DeviceCache& dc, cudaStream_t stream) {
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = (int64_t)dc.sm_count * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  bounded_cut_kernel<Bytes><<<(unsigned)blocks, 256, 0, stream>>>(
      static_cast<const typename LabelOf<Bytes>::type*>(labels), f, codes, total, bound, flags);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace host
}  // namespace edtb200

#define EDT_INSTANTIATE_BOUNDED(B)                                                                            \
  template int edtb200::host::launch_later_window<B>(const void*, const float*, float*, int*,                 \
                                                     const edtb200::LineGeom&, float, int, int, int, int,     \
                                                     edtb200::host::PassArith, float,                         \
                                                     edtb200::host::DeviceCache&, cudaStream_t);              \
  template int edtb200::host::launch_bounded_cut<B>(const void*, float*, int*, int64_t, float, int,           \
                                                    edtb200::host::DeviceCache&, cudaStream_t);
