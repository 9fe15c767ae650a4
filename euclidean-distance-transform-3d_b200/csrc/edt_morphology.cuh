// edt_morphology.cuh -- the stores of the spherical morphology (edtb200_morphology, include/edt_b200.h).
//
// A morphology step is a bounded transform (run_bounded_passes) whose last store does not write the
// distance: it writes, for each voxel, a label or a 0/1 mask chosen by MorphSelect's truth table from
// two bits -- whether the caller's label there is non-zero, and whether the squared distance is within
// the bound ("near": value <= bound).  Where the last pass takes the window kernel the choice is made
// in its store (later_axis_window_select_kernel); otherwise morph_select_kernel makes it after the
// passes, in place of bounded_cut_kernel.  No float result leaves the call.
#pragma once
#include "edt_bounded.cuh"

namespace edtb200 {

// The select of voxel `at`: near = its value is within the bound.
template <int SrcBytes>
__device__ __forceinline__ void morph_store(const MorphSelect& sel, int64_t at, bool near) {
  using ST = typename LabelOf<SrcBytes>::type;
  const ST v = static_cast<const ST*>(sel.src)[at];
  const bool keep = (sel.table >> ((label_nonzero<SrcBytes>(v, sel.as_float) ? 2 : 0) + (near ? 1 : 0))) & 1;
  if (sel.mask_out)
    static_cast<uint8_t*>(sel.out)[at] = keep ? 1 : 0;
  else
    static_cast<ST*>(sel.out)[at] = keep ? v : (ST)0;
}

// The last later pass over a window, as later_axis_window_kernel, storing the select instead of the
// distance.  Bytes: the transform's labels (the runs); SrcBytes: sel.src's.
template <int Bytes, int SrcBytes>
__global__ void __launch_bounds__(kWindowWarps * 32)
later_axis_window_select_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels,
                                const float* __restrict__ fin, LineGeom g, float w2, int radius, int border_lo,
                                int border_hi, int dbl_from, float bound, int64_t row_tiles, int64_t tiles,
                                MorphSelect sel) {
  using LT = typename LabelOf<Bytes>::type;
  window_tiles<Bytes>(labels, fin, g, w2, radius, border_lo, border_hi, dbl_from, bound, row_tiles, tiles,
                      [&](int64_t at, float best, int, LT) { morph_store<SrcBytes>(sel, at, best <= bound); });
}

// The select over `total` voxels of the last pass's values f.
template <int SrcBytes>
__global__ void __launch_bounds__(256)
morph_select_kernel(const float* __restrict__ f, int64_t total, float bound, MorphSelect sel) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    morph_store<SrcBytes>(sel, i, f[i] <= bound);
}

// The labels the transforms of float labels compare: -0.0 becomes +0.0, every other value keeps its bits.
template <int Bytes>
__global__ void __launch_bounds__(256)
fold_float_labels_kernel(const typename LabelOf<Bytes>::type* __restrict__ in, typename LabelOf<Bytes>::type* out,
                         int64_t total) {
  using LT = typename LabelOf<Bytes>::type;
  const LT sign = (LT)1 << (8 * Bytes - 1);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const LT v = in[i];
    out[i] = v == sign ? (LT)0 : v;
  }
}

namespace host {

inline int64_t stream_blocks(int64_t total, const DeviceCache& dc) {
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = (int64_t)dc.sm_count * 8;
  if (blocks > cap) blocks = cap;
  return blocks < 1 ? 1 : blocks;
}

template <int Bytes, int SrcBytes>
int window_select(const void* labels, const float* fin, const LineGeom& g, float w, int radius, int border_lo,
                  int border_hi, PassArith arith, float bound, const MorphSelect& sel, DeviceCache& dc,
                  cudaStream_t stream) {
  using LT = typename LabelOf<Bytes>::type;
  if (radius < 0 || radius > kWindowRadiusLimit) return fail(EDTB200_EINVAL, "window radius %d out of range", radius);
  const size_t smem = window_smem_bytes(radius, Bytes);
  if (smem > (size_t)dc.max_smem_optin) return fail(EDTB200_ELIMIT, "a window of radius %d exceeds the shared memory", radius);
  const int64_t row_tiles = (g.n + kWindowRows - 1) / kWindowRows;
  const int64_t tiles = ((g.inner_count + 31) >> 5) * row_tiles * g.outer_count;
  auto kern = later_axis_window_select_kernel<Bytes, SrcBytes>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kWindowWarps * 32, smem));
  int64_t blocks = (int64_t)dc.sm_count * (per_sm > 0 ? per_sm : 1);      // one persistent wave
  if (blocks > tiles) blocks = tiles;
  if (blocks < 1) blocks = 1;
  kern<<<(unsigned)blocks, kWindowWarps * 32, smem, stream>>>(static_cast<const LT*>(labels), fin, g, w * w, radius,
                                                              border_lo, border_hi, arith.exact ? 4096 : 0, bound,
                                                              row_tiles, tiles, sel);
  CUDA_TRY(cudaGetLastError());
  g_last_later = LaterLaunch{2, radius, 0, 0, 0, 0, 0, !arith.exact};
  return 0;
}

int launch_window_select(const void* labels, int label_bytes, const float* fin, const LineGeom& g, float w,
                         int radius, int border_lo, int border_hi, PassArith arith, float bound,
                         const MorphSelect& sel, DeviceCache& dc, cudaStream_t stream) {
  return with_label_width(sel.src_bytes, [&](auto s) {
    if (label_bytes == 1)
      return window_select<1, s>(labels, fin, g, w, radius, border_lo, border_hi, arith, bound, sel, dc, stream);
    if (label_bytes == s)
      return window_select<s, s>(labels, fin, g, w, radius, border_lo, border_hi, arith, bound, sel, dc, stream);
    return fail(EDTB200_EINVAL, "a window select of %d-byte labels from %d-byte runs", (int)s, label_bytes);
  });
}

int launch_morph_select(const float* f, int64_t total, float bound, const MorphSelect& sel, DeviceCache& dc,
                        cudaStream_t stream) {
  return with_label_width(sel.src_bytes, [&](auto s) {
    morph_select_kernel<s><<<(unsigned)stream_blocks(total, dc), 256, 0, stream>>>(f, total, bound, sel);
    CUDA_TRY(cudaGetLastError());
    return 0;
  });
}

int launch_fold_float_labels(const void* in, int label_bytes, void* out, int64_t total, DeviceCache& dc,
                             cudaStream_t stream) {
  auto go = [&](auto k) {
    using LT = typename LabelOf<decltype(k)::value>::type;
    fold_float_labels_kernel<decltype(k)::value><<<(unsigned)stream_blocks(total, dc), 256, 0, stream>>>(
        static_cast<const LT*>(in), static_cast<LT*>(out), total);
    CUDA_TRY(cudaGetLastError());
    return 0;
  };
  if (label_bytes == 4) return go(std::integral_constant<int, 4>{});
  if (label_bytes == 8) return go(std::integral_constant<int, 8>{});
  return fail(EDTB200_EINVAL, "float labels have 4 or 8 bytes (got %d)", label_bytes);
}

}  // namespace host
}  // namespace edtb200
