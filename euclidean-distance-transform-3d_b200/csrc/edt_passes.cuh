// edt_passes.cuh -- launchers of the axis-pass kernels, templated on the label width.
//
// Included by edt_passes_b{1,2,4,8}.cu, each of which instantiates launch_first / launch_later
// for ONE label width (the kernel templates are large; four translation units build in parallel).
// These launchers play the role of the per-axis loops of the reference's volume driver
// (pyedt::_edt3dsq, src/edt.hpp:428-475): which kernel variant, which tile shape, which grid.
#pragma once
#include "edt_host.h"

#include <cstdlib>
#include <cstring>

namespace edtb200 {
namespace host {

template <int Bytes>
int launch_first(const void* labels, float* f, int64_t nlines, int64_t sx, float w, int border, int flags,
                 DeviceCache& dc, cudaStream_t stream) {
  const float* table = nullptr;
  int trc = step_table(dc, w, (int)sx + 1, stream, &table);
  if (trc) return trc;
  RunStat stat;
  stat.counter = dc.stat_counter; stat.ticket = dc.stat_ticket; stat.publish = dc.stat_publish_dev;
  stat.voxels = (unsigned long long)nlines * (unsigned long long)sx;

  using LT = typename LabelOf<Bytes>::type;
  // register-resident vector kernel when rows are short and 16-byte aligned
  if (sx % 4 == 0 && sx <= 1024 && reinterpret_cast<uintptr_t>(labels) % (4 * Bytes) == 0 &&
      reinterpret_cast<uintptr_t>(f) % 16 == 0) {
    const size_t smem = sizeof(float) * (size_t)(sx + 2);
    int64_t blocks = (nlines + 7) / 8;
    static const int xgrid = getenv("EDTB200_X_GRID") ? atoi(getenv("EDTB200_X_GRID")) : 0;     // A/B switch
    const int64_t cap = (int64_t)dc.sm_count * (xgrid ? xgrid : (sx > 512 ? 12 : 15));   // whole waves at 5 (rows <= 512) / 3 CTAs per SM
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    const LT* lab = static_cast<const LT*>(labels);
#define EDT_LAUNCH_VEC(KK)                                                                              \
  do {                                                                                                  \
    if (flags == 0)                                                                                     \
      first_axis_vec_kernel<Bytes, KK, true><<<(unsigned)blocks, 256, smem, stream>>>(                  \
          lab, f, nlines, (int)sx, table, border, flags, stat);                                         \
    else                                                                                                \
      first_axis_vec_kernel<Bytes, KK, false><<<(unsigned)blocks, 256, smem, stream>>>(                 \
          lab, f, nlines, (int)sx, table, border, flags, stat);                                         \
  } while (0)
    if (sx <= 128)      EDT_LAUNCH_VEC(1);
    else if (sx <= 256) EDT_LAUNCH_VEC(2);
    else if (sx <= 512) EDT_LAUNCH_VEC(4);
    else                EDT_LAUNCH_VEC(8);
#undef EDT_LAUNCH_VEC
    CUDA_TRY(cudaGetLastError());
    return step_table_used(dc, table, stream);
  }
  const int nwords = (int)(sx >> 5) + 1;
  const size_t per_warp = sizeof(uint32_t) * 4 * (size_t)nwords;
  int warps = 8;
  while (warps > 1 && per_warp * warps > (size_t)dc.max_smem_optin) warps >>= 1;
  if (per_warp * warps > (size_t)dc.max_smem_optin) {
    return fail(EDTB200_ELIMIT, "first axis of %lld voxels exceeds the shared-memory line buffer",
                (long long)sx);
  }
  const size_t smem = per_warp * warps;
  auto kern = first_axis_kernel<Bytes>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int64_t blocks = (nlines + warps - 1) / warps;
  const int64_t cap = (int64_t)dc.sm_count * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  kern<<<(unsigned)blocks, warps * 32, smem, stream>>>(static_cast<const LT*>(labels), f, nlines, (int)sx, table,
                                                       border, flags, stat);
  CUDA_TRY(cudaGetLastError());
  return step_table_used(dc, table, stream);
}

// Did the first-axis pass of the PREVIOUS transform on this device see label noise (at least nine
// runs per ten voxels along x)?  A prediction for the current volume, read from mapped host memory
// without any synchronisation; a wrong guess only costs speed (both kernel variants are complete).
inline bool noise_predicted(const DeviceCache& dc) {
  static const int forced = getenv("EDTB200_TILE_CTAS") ? atoi(getenv("EDTB200_TILE_CTAS")) : 0;   // A/B switch
  if (forced == 2) return true;
  if (forced == 3) return false;
  const volatile unsigned long long* p = dc.stat_publish_host;
  if (!p) return false;
  const unsigned long long starts = p[0], voxels = p[1];
  return voxels > 0 && starts * 10ull >= voxels * 9ull;
}

// Tensor map over the distance volume for one later-axis pass: dims (adjacent lines, line
// length, outer), box = tx lines x box_rows.
inline bool make_tile_map(CUtensorMap* map, float* f, const LineGeom& g, int tx, int box_rows) {
  EncodeTiledFn enc = tensor_map_encoder();
  if (!enc) return false;
  const cuuint64_t dims[3] = {(cuuint64_t)g.inner_count, (cuuint64_t)g.n, (cuuint64_t)g.outer_count};
  const cuuint64_t strides[2] = {(cuuint64_t)g.line_stride * sizeof(float),
                                 (cuuint64_t)(g.outer_count > 1 ? g.outer_stride : g.line_stride * (int64_t)g.n) *
                                     sizeof(float)};
  const cuuint32_t box[3] = {(cuuint32_t)tx, (cuuint32_t)box_rows, 1u};
  const cuuint32_t estr[3] = {1u, 1u, 1u};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, f, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

inline void tile_boxes(int n, TileBoxes* tb) {
  tb->nboxes = (n + 255) / 256;
  tb->box_rows = (n + tb->nboxes - 1) / tb->nboxes;
  if (tb->nboxes > 1) tb->box_rows = (tb->box_rows + 3) & ~3;      // keeps every box 128-byte aligned
}

template <int Bytes, int TX>
int launch_tile(const void* labels, float* f, LineGeom g, float w2, int border_lo, int border_hi, int flags,
                bool use_tma, cudaStream_t stream, bool pdl, bool noise, bool int_hull) {
  using LT = typename LabelOf<Bytes>::type;
  const int nchunks = (g.n + 31) >> 5;
  TileBoxes tb;
  tile_boxes(g.n, &tb);
  g.tiles_per_outer = (int)((g.inner_count + TX - 1) / TX);
  const int64_t tiles = (int64_t)g.tiles_per_outer * g.outer_count;
  if (tiles > 0x7fffffffLL) return fail(EDTB200_ELIMIT, "too many line tiles");
  CUtensorMap map;
  memset(&map, 0, sizeof(map));
  if (use_tma && !make_tile_map(&map, f, g, TX, tb.box_rows)) use_tma = false;
  const int rows_alloc = use_tma ? tb.box_rows * tb.nboxes : g.n;
  const size_t smem = tile_smem_bytes(g.n, TX, rows_alloc);
  constexpr int SUBS = 32 / TX;
  int warps = (nchunks + SUBS - 1) / SUBS;
  const bool wide = warps > 16;                 // long lines: one tile per SM, so give it 32 warps
  if (warps > 32) warps = 32;
  const LT* lab = static_cast<const LT*>(labels);
  // Programmatic dependent launch: this pass may begin (label staging) while the previous pass of
  // the stream drains its last wave; the kernel itself waits before touching the distances.
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)tiles);
  cfg.blockDim = dim3((unsigned)(warps * 32));
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute pdl_attr[1];
  pdl_attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  pdl_attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = pdl_attr;
  static const bool pdl_off = getenv("EDTB200_NO_PDL") != nullptr;    // A/B switch for measurements
  cfg.numAttrs = (pdl && !pdl_off) ? 1 : 0;   // only when the previous kernel of the stream is our own pass
  const int w2i = int_hull ? (int)w2 : 0;
  static const bool int_off = getenv("EDTB200_NO_INT_HULL") != nullptr;     // A/B switch for measurements
  // integer hull tests are instantiated for the hot shape only (128-byte rows, TMA staging)
  const bool ih = int_hull && !int_off && TX == 32 && use_tma;
#define EDT_LAUNCH_ONE(EPI, TMA, WIDE, CTAS, IH)                                                    \
  do {                                                                                              \
    auto kern = later_axis_tile_kernel<Bytes, TX, EPI, TMA, WIDE, CTAS, IH>;                        \
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   \
    CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, map, lab, f, g, tb, w2, border_lo, border_hi, flags, w2i)); \
    g_last_later = LaterLaunch{0, TX, TMA, WIDE, CTAS, IH, EPI, 0};                                 \
  } while (0)
#define EDT_LAUNCH_TILE(EPI, TMA)                                                                   \
  do {                                                                                              \
    if constexpr (TX == 32 && TMA) {                                                                \
      if (wide) { if (ih) EDT_LAUNCH_ONE(EPI, TMA, true, 3, true); else EDT_LAUNCH_ONE(EPI, TMA, true, 3, false); } \
      else if (noise) { if (ih) EDT_LAUNCH_ONE(EPI, TMA, false, 2, true); else EDT_LAUNCH_ONE(EPI, TMA, false, 2, false); } \
      else { if (ih) EDT_LAUNCH_ONE(EPI, TMA, false, 3, true); else EDT_LAUNCH_ONE(EPI, TMA, false, 3, false); } \
    } else {                                                                                        \
      if (wide) EDT_LAUNCH_ONE(EPI, TMA, true, 3, false); else EDT_LAUNCH_ONE(EPI, TMA, false, 3, false); \
    }                                                                                               \
  } while (0)
  if (flags) { if (use_tma) EDT_LAUNCH_TILE(true, true); else EDT_LAUNCH_TILE(true, false); }
  else       { if (use_tma) EDT_LAUNCH_TILE(false, true); else EDT_LAUNCH_TILE(false, false); }
#undef EDT_LAUNCH_TILE
#undef EDT_LAUNCH_ONE
  CUDA_TRY(cudaGetLastError());
  return 0;
}

template <int Bytes>
int launch_later(const void* labels, float* f, const LineGeom& g0, float w, int border_lo, int border_hi,
                 int flags, DeviceCache& dc, cudaStream_t stream, bool pdl, double fmax, bool exact) {
  using LT = typename LabelOf<Bytes>::type;
  LineGeom g = g0;
  const float w2 = w * w;                       // float product, as src/edt.hpp:181

  // ---- shared-memory tile kernel: whole lines x TX adjacent lines per CTA ----
  // Its candidates are single fused multiply-adds, the reference's double sum rounded once only
  // when that sum is exact: passes where it may not be go the long way.
  const bool fits32 = (int64_t)g.n * g.line_stride + 64 < (1LL << 32);
  if (exact && fits32 && g.n <= 4096 && g.inner_count < (1LL << 31)) {
    const bool aligned = reinterpret_cast<uintptr_t>(f) % 16 == 0 && g.line_stride % 4 == 0 &&
                         (g.outer_count <= 1 || g.outer_stride % 4 == 0);
    // Tile width: 128-byte rows (TX = 32) keep DRAM bursts and L2 lines whole, which matters more
    // than occupancy even at one CTA per SM; narrower tiles only when a 32-wide tile cannot fit.
    int tx = 0;
    for (int cand = 32; cand >= 8 && !tx; cand >>= 1) {
      TileBoxes tb;
      tile_boxes(g.n, &tb);
      if (tile_smem_bytes(g.n, cand, tb.box_rows * tb.nboxes) <= (size_t)dc.max_smem_optin) tx = cand;
    }
    if (tx) {
      const bool use_tma = aligned && g.inner_count >= tx;
      const bool noise = noise_predicted(dc);
      // Integer hull tests: the caller vouches (fmax >= 0) that every finite sample of f is an
      // integer not above fmax; with an integer w2 and fmax + w2 * n^2 < 2^31 every g = f + w2 v^2
      // is an exact 32-bit integer.  fmax < 0 = unknown -> double.
      const bool int_hull = fmax >= 0.0 && w2 == floorf(w2) && w2 >= 1.0f && w2 < 1048576.0f &&
                            fmax + (double)w2 * (double)g.n * (double)g.n < 2147483000.0;
      switch (tx) {
        case 32: return launch_tile<Bytes, 32>(labels, f, g, w2, border_lo, border_hi, flags, use_tma, stream, pdl, noise, int_hull);
        case 16: return launch_tile<Bytes, 16>(labels, f, g, w2, border_lo, border_hi, flags, use_tma, stream, pdl, noise, int_hull);
        default: return launch_tile<Bytes, 8>(labels, f, g, w2, border_lo, border_hi, flags, use_tma, stream, pdl, noise, int_hull);
      }
    }
  }
  // ---- lines too long for a shared-memory tile: out of place through a temporary volume ----
  const int64_t lines = g.inner_count * g.outer_count;
  const size_t bytes = sizeof(float) * (size_t)lines * (size_t)g.n;
  float* tmp = nullptr;
  int* hull = nullptr;
  CUDA_TRY(scratch_alloc(dc, reinterpret_cast<void**>(&tmp), bytes, stream));
  if (scratch_alloc(dc, reinterpret_cast<void**>(&hull), bytes, stream) != cudaSuccess) {
    cudaGetLastError();
    cudaFreeAsync(tmp, stream);
    return fail(EDTB200_ENOMEM, "no device memory for the long-line scratch volumes");
  }
  const int64_t blocks = (lines + 127) / 128;
  if (blocks > 0x7fffffffLL) {
    cudaFreeAsync(tmp, stream); cudaFreeAsync(hull, stream);
    return fail(EDTB200_ELIMIT, "too many lines");
  }
  later_axis_long_kernel<Bytes><<<(unsigned)blocks, 128, 0, stream>>>(
      static_cast<const LT*>(labels), f, tmp, hull, g, w2, border_lo, border_hi, flags, exact ? 4096 : 0);
  CUDA_TRY(cudaGetLastError());
  g_last_later = LaterLaunch{1, 0, 0, 0, 0, 0, flags != 0, !exact};
  CUDA_TRY(cudaMemcpyAsync(f, tmp, bytes, cudaMemcpyDeviceToDevice, stream));
  CUDA_TRY(cudaFreeAsync(hull, stream));
  CUDA_TRY(cudaFreeAsync(tmp, stream));
  return 0;
}

}  // namespace host
}  // namespace edtb200

#define EDT_INSTANTIATE_PASSES(B)                                                                        \
  template int edtb200::host::launch_first<B>(const void*, float*, int64_t, int64_t, float, int, int,    \
                                              edtb200::host::DeviceCache&, cudaStream_t);                \
  template int edtb200::host::launch_later<B>(const void*, float*, const edtb200::LineGeom&, float, int, \
                                              int, int, edtb200::host::DeviceCache&, cudaStream_t, bool, \
                                              double, bool);
