// edt_passes.cuh -- launchers of the axis-pass kernels, templated on the label width.
//
// Included by edt_passes_b{1,2,4,8}.cu, each of which instantiates launch_first / launch_later
// for ONE label width (the kernel templates are large; four translation units build in parallel).
// edt_capi.cu reaches the instance for a run-time width through with_label_width (edt_host.h).
// These launchers play the role of the per-axis loops of the reference's volume driver
// (pyedt::_edt3dsq, src/edt.hpp:428-475): which kernel variant, which tile shape, which grid.
#pragma once
#include "edt_host.h"
#include "edt_feature.cuh"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <cstring>

namespace edtb200 {
namespace host {

// The generic first-axis kernel (any row length and alignment), one warp per row.
template <int Bytes, bool Sites>
int launch_first_generic(const void* labels, float* f, int* codes, int64_t nlines, int64_t sx, const float* table,
                         int border, int flags, RunStat stat, DeviceCache& dc, cudaStream_t stream) {
  using LT = typename LabelOf<Bytes>::type;
  const int nwords = (int)(sx >> 5) + 1;
  const size_t per_warp = sizeof(uint32_t) * 4 * (size_t)nwords;
  int warps = 8;
  while (warps > 1 && per_warp * warps > (size_t)dc.max_smem_optin) warps >>= 1;
  if (per_warp * warps > (size_t)dc.max_smem_optin) {
    return fail(EDTB200_ELIMIT, "first axis of %lld voxels exceeds the shared-memory line buffer",
                (long long)sx);
  }
  const size_t smem = per_warp * warps;
  auto kern = first_axis_kernel<Bytes, Sites>;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int64_t blocks = (nlines + warps - 1) / warps;
  const int64_t cap = (int64_t)dc.sm_count * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  kern<<<(unsigned)blocks, warps * 32, smem, stream>>>(static_cast<const LT*>(labels), f, nlines, (int)sx, table,
                                                       border, flags, stat, codes);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// Shared memory of first_axis_planes_kernel: its ring of stages of W + 1 rows, the step table.
inline size_t planes_smem_bytes(int64_t sx, int label_bytes) {
  return kPlaneBarBytes + (size_t)planes_stages(label_bytes) * (size_t)(kPlaneWarps + 1) * (size_t)sx * label_bytes +
         sizeof(float) * (size_t)(sx + 2);
}

// The register-resident X kernel for K 128-voxel blocks per row; with `planes` (planes->y non-null)
// the kernel that also writes them, compiled for labels of 4 and 8 bytes, rows of at most 512 voxels
// and the plain kernel flags only, where run_passes takes them: plan_noise takes no planes for a
// signed transform, and the X pass of any other transform of two or more axes has flags 0.
// march (may be null): the chunk count and grid asked for and launched (PlanesMarch).
template <int Bytes, int K, bool Plain>
int launch_first_vec(const void* labels, float* f, int64_t nlines, int64_t sx, const float* table, int border,
                     int flags, RunStat stat, const XPlanes* planes, DeviceCache& dc, cudaStream_t stream,
                     PlanesMarch* march) {
  using LT = typename LabelOf<Bytes>::type;
  if (!planes) {
    const size_t smem = sizeof(float) * (size_t)(sx + 2);
    int64_t blocks = (nlines + 7) / 8;
    const int64_t cap = (int64_t)dc.sm_count * (sx > 512 ? 12 : 15);   // whole waves at 5 (rows <= 512) / 3 CTAs per SM
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    first_axis_vec_kernel<Bytes, K, Plain><<<(unsigned)blocks, 256, smem, stream>>>(
        static_cast<const LT*>(labels), f, nlines, (int)sx, table, border, flags, stat);
    CUDA_TRY(cudaGetLastError());
    return 0;
  }
  if constexpr (Bytes >= 4 && K <= 4 && Plain) {
    // Bands of 8 slices that march along y through a ring of stages of 9 rows: 4 stages (74 KB) for
    // 512-voxel rows of 4-byte labels, so three CTAs per SM, each reading two stages with two more
    // (36 KB) in flight; 3 stages (110 KB) for 8-byte ones, two CTAs per SM, one stage in flight.
    constexpr int W = kPlaneWarps;
    const size_t smem = planes_smem_bytes(sx, Bytes);
    if (smem > (size_t)dc.max_smem_optin)
      return fail(EDTB200_ELIMIT, "run-start planes of %lld-voxel rows exceed the shared memory", (long long)sx);
    const bool z = planes->z != nullptr;
    auto kern = z ? first_axis_planes_kernel<Bytes, K, Plain, 2> : first_axis_planes_kernel<Bytes, K, Plain, 1>;
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, W * 32, smem));
    // One persistent wave.  The slices are cut into y-chunks so that the items -- (band, chunk) in 3-D,
    // W (image, chunk) sequences in 2-D -- fill the wave without a second one, but into no chunk shorter
    // than 67 rows, so that each chunk's leading and trailing rows, read once more, stay within 3 % of
    // its labels.
    const int64_t sy = planes->sy, nz = nlines / sy, wave = (int64_t)dc.sm_count * (per_sm > 0 ? per_sm : 1);
    const int64_t fill = z ? wave / ((nz + W - 1) / W) : wave * W / nz;
    // A march may ask for another chunk count (1 .. sy) and grid (1 .. items), checked by its caller.
    const int64_t nchunks = march && march->want_chunks ? march->want_chunks
                                                        : std::max<int64_t>(1, std::min(fill, sy * 3 / 200));
    const int64_t items = z ? march_items<W, 2>(nz, nchunks) : march_items<W, 1>(nz, nchunks);
    const int64_t blocks = march && march->want_ctas ? march->want_ctas : std::max<int64_t>(1, std::min(wave, items));
    kern<<<(unsigned)blocks, W * 32, smem, stream>>>(static_cast<const LT*>(labels), f, nlines, (int)sx, table, border,
                                                     flags, stat, *planes, (int)nchunks);
    CUDA_TRY(cudaGetLastError());
    if (march) {
      march->k = K;
      march->plain = Plain;
      march->planes = z ? 2 : 1;
      march->nchunks = nchunks;
      march->items = items;
      march->grid = blocks;
    }
    return 0;
  }
  return fail(EDTB200_EINVAL, "run-start planes asked of an X launch that cannot write them");
}

template <int Bytes>
int launch_first(const void* labels, float* f, int64_t nlines, int64_t sx, float w, int border, int flags,
                 const XPlanes* planes, DeviceCache& dc, cudaStream_t stream, PlanesMarch* march) {
  if (planes && !first_is_vec(labels, Bytes, f, sx))   // launch_first_vec refuses the rest
    return fail(EDTB200_EINVAL, "run-start planes asked of an X launch that cannot write them");
  StepTable step(dc, stream);
  int trc = step.get(w, (int)sx + 1);
  if (trc) return trc;
  const float* table = step.data();
  const RunStat stat = run_stat(dc, (unsigned long long)nlines * (unsigned long long)sx);

  // register-resident vector kernel when rows are short and 16-byte aligned
  if (first_is_vec(labels, Bytes, f, sx)) {
#define EDT_LAUNCH_VEC(KK)                                                                                        \
  (flags == 0                                                                                                    \
       ? launch_first_vec<Bytes, KK, true>(labels, f, nlines, sx, table, border, flags, stat, planes, dc, stream, march) \
       : launch_first_vec<Bytes, KK, false>(labels, f, nlines, sx, table, border, flags, stat, planes, dc, stream, march))
    const int rc = sx <= 128 ? EDT_LAUNCH_VEC(1) : sx <= 256 ? EDT_LAUNCH_VEC(2) : sx <= 512 ? EDT_LAUNCH_VEC(4)
                                                                                            : EDT_LAUNCH_VEC(8);
#undef EDT_LAUNCH_VEC
    return rc ? rc : step.queued();
  }
  const int rc = launch_first_generic<Bytes, false>(labels, f, nullptr, nlines, sx, table, border, flags, stat, dc,
                                                    stream);
  return rc ? rc : step.queued();
}

// The site-tracking X pass (feature transform): the generic kernel, which also writes the site
// codes.  It publishes no run statistic, so it does not steer the next transform's launches.
template <int Bytes>
int launch_first_sites(const void* labels, float* f, int* codes, int64_t nlines, int64_t sx, float w, int border,
                       int flags, DeviceCache& dc, cudaStream_t stream) {
  StepTable step(dc, stream);
  int trc = step.get(w, (int)sx + 1);
  if (trc) return trc;
  RunStat none;
  memset(&none, 0, sizeof(none));
  const int rc = launch_first_generic<Bytes, true>(labels, f, codes, nlines, sx, step.data(), border, flags, none,
                                                   dc, stream);
  return rc ? rc : step.queued();
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

// EDTB200_NO_INT_HULL: the later passes test their hulls in double only (A/B switch for measurements).
inline bool no_int_hull() {
  static const bool off = getenv("EDTB200_NO_INT_HULL") != nullptr;
  return off;
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

// Shared memory of one tile of `tx` lines (see later_axis_tile_kernel).
inline size_t tile_smem_bytes(int n, int tx, int rows_alloc) {
  const int nchunks = (n + 31) >> 5;
  return (size_t)rows_alloc * tx * 4 + (size_t)nchunks * tx * 12 + (size_t)((n + 3) & ~1) * 4 + 16 +
         (size_t)nchunks * tx +    // + one flag byte per (chunk, line)
         (size_t)tx * 4 + 4;       // + one word per line: chunks holding a run start
}

// Warps of a tile of `tx` lines (32-row chunks, 32 / tx lines per warp) before the cap at 32;
// more than 16 makes the wide variant.
inline int tile_warps(int n, int tx) { return (((n + 31) >> 5) * tx + 31) / 32; }

// The plan of one later-axis pass: what launch_later runs for it.  Pure host logic.
//   tma_ok       the volume is 16-byte aligned and (when asked again) its tensor map encoded
//   noise        noise_predicted: 2 CTAs per SM instead of 3
//   int_hull_off EDTB200_NO_INT_HULL
inline LaterLaunch plan_later(const LineGeom& g, bool epilogue, PassArith arith, int max_smem_optin, bool tma_ok,
                              bool noise, bool int_hull_off) {
  // ---- shared-memory tile kernel: whole lines x tx adjacent lines per CTA ----
  // Its candidates are single fused multiply-adds, the reference's double sum rounded once only
  // when that sum is exact: passes where it may not be go the long way.
  const bool fits32 = (int64_t)g.n * g.line_stride + 64 < (1LL << 32);
  if (arith.exact && fits32 && g.n <= 4096 && g.inner_count < (1LL << 31)) {
    // Tile width: 128-byte rows (TX = 32) keep DRAM bursts and L2 lines whole, which matters more
    // than occupancy even at one CTA per SM; narrower tiles only when a 32-wide tile cannot fit.
    TileBoxes tb;
    tile_boxes(g.n, &tb);
    int tx = 0;
    for (int cand = 32; cand >= 8 && !tx; cand >>= 1)
      if (tile_smem_bytes(g.n, cand, tb.box_rows * tb.nboxes) <= (size_t)max_smem_optin) tx = cand;
    const bool wide = tx && tile_warps(g.n, tx) > 16;   // long lines: one tile per SM, so give it 32 warps
    // Narrow tiles are compiled wide only: they are chosen when a 32-wide tile does not fit, which
    // with sm_90a's 227 KB happens from 1597 rows on, where a 16-wide tile has 25 warps (and an
    // 8-wide one, needed from about 3100 rows, as many).  Otherwise the long-line kernel runs.
    if (tx == 32 || wide) {
      const bool tma = tma_ok && g.inner_count >= tx;
      // 2 CTAs per SM and the integer hull tests are compiled for the hot shape only (128-byte
      // rows, TMA staging)
      return LaterLaunch{0, tx, tma, wide, tx == 32 && tma && !wide && noise ? 2 : 3,
                         arith.int_hull && !int_hull_off && tx == 32 && tma, epilogue, 0};
    }
  }
  // ---- lines too long for a shared-memory tile, or sums not exact in double ----
  return LaterLaunch{1, 0, 0, 0, 0, 0, epilogue, !arith.exact};
}

// plan_later's tma_ok before the tensor map is encoded: the distances 16-byte aligned (f16) and every
// line and outer stride of g a multiple of 4 floats.
inline bool tma_aligned(bool f16, const LineGeom& g) {
  return f16 && g.line_stride % 4 == 0 && (g.outer_count <= 1 || g.outer_stride % 4 == 0);
}

// The label-noise plan of transform t over `count` volumes laid end to end (run_passes).  Pure host
// logic.  f16: the distances are 16-byte aligned; first_vec: first_is_vec holds for its X pass; noise:
// the one reading of noise_predicted; int_hull_off, forced_group: EDTB200_NO_INT_HULL and
// EDTB200_SETTLED_GROUP.
// The run-start planes pay where the later passes only stream -- label noise with labels of 4 or 8
// bytes: there a later pass moves 4 + 1/8 bytes per voxel instead of 8 or 12, for 1/4 byte more
// written by the X pass (which stages its label rows in shared memory, bands of slices marching along
// y, to compare neighbouring rows).  On narrower labels and on structured volumes the dearer X pass
// costs more than the later passes gain (DESIGN.md section 4.1), so none are taken there; nor for
// signed transforms, whose last pass needs the labels' background bits as well.  The X pass writes a
// plane for every later axis once one later pass takes a tile kernel; a later pass reads its plane
// where it takes the label-noise tile kernel (2 CTAs per SM), otherwise the labels.
inline NoisePlan plan_noise(const Transform& t, int64_t count, bool f16, bool first_vec, bool noise, bool int_hull_off,
                            int forced_group, int max_smem_optin, int sm_count) {
  NoisePlan np;
  np.noise = noise;
  const int64_t sx = t.n[0], sy = t.n[1], sz = t.n[2];
  bool tile = false;
  for (int k = 1; k < t.ndim; ++k) {
    const LineGeom g = geom_for_axis(k, sx, sy, sz, count);
    np.later[k] = plan_later(g, kernel_flags(t.flags, false, k == t.ndim - 1) != 0, transform_arith(t.w, t.n, k),
                             max_smem_optin, tma_aligned(f16, g), noise, int_hull_off);
    tile = tile || np.later[k].kernel == 0;
  }
  if (t.ndim < 2 || t.label_bytes < 4 || (t.flags & EDTB200_SIGNED) || sx > 512 || !first_vec || !noise ||
      sz * count > 0x7fffffffLL || sy > 0x3fffffffLL || !tile)   // that X pass counts slices and rows in 32 bits
    return np;
  np.planes = t.ndim - 1;
  for (int k = 1; k < t.ndim; ++k) {
    LaterLaunch& p = np.later[k];
    np.reads[k] = p.ctas == 2;       // the label-noise variant (tile_kernel_bits)
    p.settled = np.reads[k] && skips_settled(true, p.int_hull, p.epilogue);
    // With `settled` armed, each CTA checks and runs a group of consecutive tiles: as many as make the
    // grid three to four waves of resident CTAs (at most 32, one bit per tile), so that a pass which
    // skips nearly every tile costs a few reads per SM and not one CTA per tile.  Fewer, larger groups
    // (two waves: 16 tiles at 512^3) skip no faster and serialise the tiles that run where they
    // cluster, as the Z tiles of the X pass's band rows do (DESIGN.md section 4.1).  Resident CTAs: the
    // plan's CTAs per SM (what the kernel is compiled for), so that sizing the grid adds no runtime
    // query to the launch.
    if (p.settled) {
      const LineGeom g = geom_for_axis(k, sx, sy, sz, count);
      const int64_t tiles = (g.inner_count + p.tx - 1) / p.tx * g.outer_count;
      const int64_t waves4 = 4 * (int64_t)sm_count * p.ctas;
      const int64_t group = forced_group > 0 ? forced_group : (tiles + waves4 - 1) / waves4;
      np.group[k] = (int)(group < 1 ? 1 : group > 32 ? 32 : group);
    }
  }
  // the Y pass refreshes the Z pass's settled plane where it skips tiles itself and the Z pass has
  // no epilogue and integer samples
  np.refresh = t.ndim == 3 && np.later[1].settled && kernel_flags(t.flags, false, true) == 0 &&
               transform_arith(t.w, t.n, 2).int_hull;
  return np;
}

// The plan of a bounded transform with max_distance d >= 0 (include/edt_b200.h, DESIGN.md section 5).
// Pure host logic.  B is the largest float32 with (double)B <= d^2; a later pass along axis k needs
// only the samples v with (double)w2 (i - v)^2 < nextafterf(B, +inf), i.e. within R_k rows, and takes
// the window kernel when R_k <= rmax.  R_k is found by bisection on that very test (monotone in r),
// capped at 2^62, which also stands for "no bound" (B = FLT_MAX, or w2 = 0).
inline BoundedPlan plan_bounded(int ndim, const float w[3], double d, int64_t rmax) {
  BoundedPlan p;
  p.bound = cut_bound(d);
  const double above = (double)nextafterf(p.bound, INFINITY);
  for (int k = 0; k < ndim; ++k) {
    const double w2 = (double)(w[k] * w[k]);          // the float product the passes use
    int64_t lo = 0, hi = (int64_t)1 << 62;            // w2 * lo^2 < above always holds (above > 0)
    while (lo < hi) {
      const int64_t mid = lo + (hi - lo + 1) / 2;
      if (w2 * (double)mid * (double)mid < above) lo = mid;
      else hi = mid - 1;
    }
    p.radius[k] = lo;
    p.windowed[k] = k >= 1 && lo <= rmax;
  }
  return p;
}

// The tile-kernel instance of plan p (Epi, TMA = p.epilogue, p.tma): only the variants
// plan_later can produce are compiled.
template <int Bytes>
using TileKernel = decltype(&later_axis_tile_kernel<Bytes, 32, false, false, false, 3, false>);
template <int Bytes, bool Epi, bool TMA>
TileKernel<Bytes> tile_kernel(const LaterLaunch& p) {
  if (p.tx == 16) return later_axis_tile_kernel<Bytes, 16, Epi, TMA, true, 3, false>;
  if (p.tx == 8) return later_axis_tile_kernel<Bytes, 8, Epi, TMA, true, 3, false>;
  if constexpr (TMA) {
    if (p.wide) return p.int_hull ? later_axis_tile_kernel<Bytes, 32, Epi, true, true, 3, true>
                                  : later_axis_tile_kernel<Bytes, 32, Epi, true, true, 3, false>;
    if (p.ctas == 2) return p.int_hull ? later_axis_tile_kernel<Bytes, 32, Epi, true, false, 2, true>
                                       : later_axis_tile_kernel<Bytes, 32, Epi, true, false, 2, false>;
    return p.int_hull ? later_axis_tile_kernel<Bytes, 32, Epi, true, false, 3, true>
                      : later_axis_tile_kernel<Bytes, 32, Epi, true, false, 3, false>;
  }
  return p.wide ? later_axis_tile_kernel<Bytes, 32, Epi, false, true, 3, false>
                : later_axis_tile_kernel<Bytes, 32, Epi, false, false, 3, false>;
}

// The variant of the 2-CTA tile kernel that reads the X pass's run-start plane (labels of 4 and 8
// bytes only; no background bits, so never for a signed pass).
template <int Bytes>
TileKernel<Bytes> tile_kernel_bits(const LaterLaunch& p) {
  if constexpr (Bytes >= 4) {
    if (p.epilogue) return p.int_hull ? later_axis_tile_kernel<Bytes, 32, true, true, false, 2, true, true>
                                      : later_axis_tile_kernel<Bytes, 32, true, true, false, 2, false, true>;
    return p.int_hull ? later_axis_tile_kernel<Bytes, 32, false, true, false, 2, true, true>
                      : later_axis_tile_kernel<Bytes, 32, false, true, false, 2, false, true>;
  }
  return nullptr;
}

template <int Bytes>
int launch_later(const void* labels, const LaterNoise* planned, float* f, const LineGeom& g0, float w, int border_lo,
                 int border_hi, int flags, PassArith arith, DeviceCache& dc, cudaStream_t stream, bool pdl) {
  using LT = typename LabelOf<Bytes>::type;
  LineGeom g = g0;
  const float w2 = w * w;                       // float product, as src/edt.hpp:181
  const bool aligned = tma_aligned(reinterpret_cast<uintptr_t>(f) % 16 == 0, g);
  const bool noise = planned ? planned->noise : noise_predicted(dc);
  LaterLaunch p = plan_later(g, flags != 0, arith, dc.max_smem_optin, aligned, noise, no_int_hull());

  if (p.kernel == 0) {
    TileBoxes tb;
    tile_boxes(g.n, &tb);
    g.tiles_per_outer = (int)((g.inner_count + p.tx - 1) / p.tx);
    const int64_t tiles = (int64_t)g.tiles_per_outer * g.outer_count;
    if (tiles > 0x7fffffffLL) return fail(EDTB200_ELIMIT, "too many line tiles");
    CUtensorMap map;
    memset(&map, 0, sizeof(map));
    if (p.tma && !make_tile_map(&map, f, g, p.tx, tb.box_rows))
      p = plan_later(g, flags != 0, arith, dc.max_smem_optin, false, noise, no_int_hull());
    const int warps = tile_warps(g.n, p.tx);
    // Programmatic dependent launch: this pass may begin (label staging) while the previous pass of
    // the stream drains its last wave; the kernel itself waits before touching the distances.
    cudaLaunchConfig_t cfg = {};
    cfg.blockDim = dim3((unsigned)((warps > 32 ? 32 : warps) * 32));
    cfg.dynamicSmemBytes = tile_smem_bytes(g.n, p.tx, p.tma ? tb.box_rows * tb.nboxes : g.n);
    cfg.stream = stream;
    cudaLaunchAttribute pdl_attr[1];
    pdl_attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    pdl_attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = pdl_attr;
    cfg.numAttrs = pdl ? 1 : 0;   // only when the previous kernel of the stream is our own pass
    // The run-start plane, its settled skip and its group as plan_noise armed them; only where the
    // tensor map could not be encoded is the plan another one, and the pass reads the labels.
    RunBits rb;
    memset(&rb, 0, sizeof(rb));
    rb.group = 1;
    if (planned && planned->bits.start) {
      LaterLaunch armed = planned->plan;
      armed.settled = 0;
      if (!memcmp(&p, &armed, sizeof(p))) rb = planned->bits;
    }
    p.settled = rb.settled != nullptr;
    const TileKernel<Bytes> kern =
        rb.start ? tile_kernel_bits<Bytes>(p)
        : p.epilogue ? (p.tma ? tile_kernel<Bytes, true, true>(p) : tile_kernel<Bytes, true, false>(p))
                     : (p.tma ? tile_kernel<Bytes, false, true>(p) : tile_kernel<Bytes, false, false>(p));
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg.dynamicSmemBytes));
    cfg.gridDim = dim3((unsigned)((tiles + rb.group - 1) / rb.group));
    CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, map, static_cast<const LT*>(labels), rb, f, g, tb, w2, border_lo,
                                border_hi, flags, p.int_hull ? (int)w2 : 0));
    g_last_later = p;
    CUDA_TRY(cudaGetLastError());
    return 0;
  }
  // ---- long-line kernel: out of place through a temporary volume ----
  const int64_t lines = g.inner_count * g.outer_count;
  const size_t bytes = sizeof(float) * (size_t)lines * (size_t)g.n;
  Scratch tmp, hull;                            // freed on every exit, hull first
  CUDA_TRY(tmp.alloc(dc, bytes, stream));
  if (const int rc = hull.take(dc, bytes, stream, "the long-line scratch volumes")) return rc;
  const int64_t blocks = (lines + 127) / 128;
  if (blocks > 0x7fffffffLL) return fail(EDTB200_ELIMIT, "too many lines");
  later_axis_long_kernel<Bytes><<<(unsigned)blocks, 128, 0, stream>>>(
      static_cast<const LT*>(labels), f, tmp.get<float>(), hull.get<int>(), g, w2, border_lo, border_hi, flags,
      p.all_double ? 0 : 4096, nullptr);
  CUDA_TRY(cudaGetLastError());
  g_last_later = p;
  CUDA_TRY(cudaMemcpyAsync(f, tmp.get(), bytes, cudaMemcpyDeviceToDevice, stream));
  return 0;
}

// The site-tracking later pass (feature transform): the long-line kernel on any line length, out
// of place (fin -> fout), also writing the site codes.  Its arithmetic is the one launch_later
// gives the long-line kernel, so its distances equal launch_later's for any plan.
template <int Bytes>
int launch_later_sites(const void* labels, const float* fin, float* fout, int* codes, const LineGeom& g, float w,
                       int border_lo, int border_hi, int flags, PassArith arith, DeviceCache& dc,
                       cudaStream_t stream) {
  using LT = typename LabelOf<Bytes>::type;
  const int64_t lines = g.inner_count * g.outer_count;
  const int64_t blocks = (lines + 127) / 128;
  if (blocks > 0x7fffffffLL) return fail(EDTB200_ELIMIT, "too many lines");
  Scratch hull;
  if (const int rc = hull.take(dc, sizeof(int) * (size_t)lines * (size_t)g.n, stream, "the long-line hull scratch"))
    return rc;
  later_axis_long_kernel<Bytes, true><<<(unsigned)blocks, 128, 0, stream>>>(
      static_cast<const LT*>(labels), fin, fout, hull.get<int>(), g, w * w, border_lo, border_hi, flags,
      arith.exact ? 4096 : 0, codes);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// Site codes of every pass -> one coordinate plane per axis (edt_feature.cuh), over `count` volumes
// of (sx, sy, sz) laid end to end.
template <int Bytes>
int launch_resolve_sites(const void* labels, const int* const codes[3], int ndim, int64_t sx, int64_t sy,
                         int64_t sz, int64_t count, bool zero_is_background, int32_t* const idx[3], DeviceCache& dc,
                         cudaStream_t stream) {
  const int64_t total = sx * sy * sz * count;
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = (int64_t)dc.sm_count * 8;
  if (blocks > cap) blocks = cap;
  SiteCodes c{{codes[0], codes[1], codes[2]}, ndim, sx, sy, sz * count, sz};
  SitePlanes out{{idx[0], idx[1], idx[2]}};
  resolve_sites_kernel<Bytes><<<(unsigned)blocks, 256, 0, stream>>>(
      static_cast<const typename LabelOf<Bytes>::type*>(labels), c, zero_is_background ? 1 : 0, out);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// Grid of the chunked feature transform's site kernels: one thread per voxel, at most 8 CTAs per SM
// (grid-stride loops beyond), as launch_resolve_sites.
inline unsigned site_blocks(int64_t total, const DeviceCache& dc) {
  const int64_t blocks = (total + 255) / 256, cap = (int64_t)dc.sm_count * 8;
  return (unsigned)(blocks < 1 ? 1 : blocks > cap ? cap : blocks);
}

// Chunked feature transform, phase 1 in 3-D: the X and Y codes of a slab -> each voxel's site within
// its slice (edt_feature.cuh); qy over the Y codes, qx into its own plane.
template <int Bytes>
int launch_slice_sites(const void* labels, const int* xcodes, int* ycodes_qy, int64_t sx, int64_t sy, int64_t sz,
                       bool zero_is_background, int32_t* qx, DeviceCache& dc, cudaStream_t stream) {
  slice_sites_kernel<Bytes><<<site_blocks(sx * sy * sz, dc), 256, 0, stream>>>(
      static_cast<const typename LabelOf<Bytes>::type*>(labels), xcodes, ycodes_qy, sx, sy, sz,
      zero_is_background ? 1 : 0, qx);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// Chunked feature transform, phase 2: the last axis's codes of a box of whole lines and the partial
// sites of phase 1 -> each voxel's site (edt_feature.cuh); the last coordinate over the codes.
template <int Bytes>
int launch_compose_sites(const void* labels, int* codes_last, const int32_t* part_x, const int32_t* part_y,
                         const SiteBox& box, bool zero_is_background, int32_t* out_x, int32_t* out_y, DeviceCache& dc,
                         cudaStream_t stream) {
  compose_sites_kernel<Bytes><<<site_blocks(box.plane * box.n, dc), 256, 0, stream>>>(
      static_cast<const typename LabelOf<Bytes>::type*>(labels), codes_last, part_x, part_y, box,
      zero_is_background ? 1 : 0, out_x, out_y);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

// expand_labels' gather over `count` volumes of (sx, sy, sz) laid end to end (edt_feature.cuh); out
// may be labels.
template <int Bytes>
int launch_expand_gather(const void* labels, const float* sqdist, const int32_t* const idx[3], int ndim, int64_t sx,
                         int64_t sy, int64_t sz, int64_t count, double limit_sq, bool as_float, void* out,
                         DeviceCache& dc, cudaStream_t stream) {
  using LT = typename LabelOf<Bytes>::type;
  const int64_t vol = sx * sy * sz;
  const ExpandSites s{sqdist, {idx[0], ndim >= 2 ? idx[1] : nullptr, ndim >= 3 ? idx[2] : nullptr}, ndim,
                      sx, sy, sz, vol, vol * count};
  expand_gather_kernel<Bytes><<<site_blocks(s.total, dc), 256, 0, stream>>>(
      static_cast<const LT*>(labels), s, limit_sq, as_float ? 1 : 0, static_cast<LT*>(out));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace host
}  // namespace edtb200

#define EDT_INSTANTIATE_PASSES(B)                                                                        \
  template int edtb200::host::launch_first<B>(const void*, float*, int64_t, int64_t, float, int, int,    \
                                              const edtb200::XPlanes*, edtb200::host::DeviceCache&,      \
                                              cudaStream_t, edtb200::host::PlanesMarch*);                \
  template int edtb200::host::launch_later<B>(const void*, const edtb200::host::LaterNoise*, float*,     \
                                              const edtb200::LineGeom&, float, int, int, int,            \
                                              edtb200::host::PassArith, edtb200::host::DeviceCache&,     \
                                              cudaStream_t, bool);                                       \
  template int edtb200::host::launch_first_sites<B>(const void*, float*, int*, int64_t, int64_t, float, int, \
                                                    int, edtb200::host::DeviceCache&, cudaStream_t);     \
  template int edtb200::host::launch_later_sites<B>(const void*, const float*, float*, int*,              \
                                                    const edtb200::LineGeom&, float, int, int, int,      \
                                                    edtb200::host::PassArith,                            \
                                                    edtb200::host::DeviceCache&, cudaStream_t);          \
  template int edtb200::host::launch_resolve_sites<B>(const void*, const int* const*, int, int64_t,      \
                                                      int64_t, int64_t, int64_t, bool, int32_t* const*,  \
                                                      edtb200::host::DeviceCache&, cudaStream_t);        \
  template int edtb200::host::launch_slice_sites<B>(const void*, const int*, int*, int64_t, int64_t, int64_t, \
                                                    bool, int32_t*, edtb200::host::DeviceCache&, cudaStream_t); \
  template int edtb200::host::launch_compose_sites<B>(const void*, int*, const int32_t*, const int32_t*,  \
                                                      const edtb200::SiteBox&, bool, int32_t*, int32_t*, \
                                                      edtb200::host::DeviceCache&, cudaStream_t);        \
  template int edtb200::host::launch_expand_gather<B>(const void*, const float*, const int32_t* const*, int, \
                                                      int64_t, int64_t, int64_t, int64_t, double, bool, void*, \
                                                      edtb200::host::DeviceCache&, cudaStream_t);
