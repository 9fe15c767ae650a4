// edt_host.h -- declarations shared by the host-side translation units of libedt_b200.so.
//
// The library is compiled as eighteen translation units so that the kernel templates build in
// parallel: edt_capi.cu (C ABI, staging, caches), edt_passes_b{1,2,4,8}.cu (the axis-pass
// launchers of edt_passes.cuh instantiated for one label width each), edt_plan.cu (the
// later-axis plan for host code that launches nothing), edt_bounded.cu (the bounded
// transforms' kernels), edt_surface.cu (the surface distances' kernels), edt_morphology.cu (the
// spherical morphology's label-writing stores), edt_parabolic.cu (the parabolic erosion and
// dilation passes), edt_nearest.cu (the nearest-labels passes), edt_medial.cu (the medial
// axis's mark kernel), edt_skeleton.cu (the skeleton's thinning kernel), edt_thickness.cu
// (local thickness's levels, seeds and stores), edt_geodesic.cu (geodesic_distance's relaxation
// passes), edt_watershed.cu (watershed's relaxation passes), edt_components.cu (the union-find passes of
// connected_components and extended_maxima) and edt_holes.cu (fill_holes' and dust's tally and apply
// passes).  The run-time label width
// becomes a template argument in one place, with_label_width below.
#pragma once
#include "../../include/edt_b200.h"
#include "edt_kernels.cuh"
#include "edt_feature.cuh"       // SiteBox

#include <cfloat>
#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <mutex>
#include <type_traits>

namespace edtb200 {

// The cut B of max_distance d >= 0: the largest float32 whose double is at most d^2 (FLT_MAX where d^2
// reaches it), so that a float32 squared distance v is within d iff v <= B.  Also on the device, where
// local thickness derives the cut of each level it computes there.
__host__ __device__ inline float cut_bound(double d) {
  const double L = d * d;
  if (L >= (double)FLT_MAX) return FLT_MAX;
  float b = (float)L;
  if ((double)b > L) b = nextafterf(b, -INFINITY);
  return b;
}

namespace host {

// Sets the calling thread's error message (edtb200_last_error) and returns `code`.
int fail(int code, const char* fmt, ...);

#define CUDA_TRY(expr)                                                                          \
  do {                                                                                          \
    cudaError_t e__ = (expr);                                                                   \
    if (e__ != cudaSuccess)                                                                     \
      return ::edtb200::host::fail(e__ == cudaErrorMemoryAllocation ? EDTB200_ENOMEM : EDTB200_ECUDA, \
                                   "%s failed: %s", #expr, cudaGetErrorString(e__));            \
  } while (0)

// Returns f(std::integral_constant<int, B>{}) for the label width B = label_bytes, so that f can
// name the width-templated kernel or launcher for B and its label type LabelOf<B>::type.
template <class F>
int with_label_width(int label_bytes, F&& f) {
  switch (label_bytes) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 8: return f(std::integral_constant<int, 8>{});
  }
  return fail(EDTB200_EINVAL, "label_bytes must be 1, 2, 4 or 8 (got %d)", label_bytes);
}

// with_label_width, and B = 0 for label_bytes 0 (no labels: every voxel inside the volume is a node).
template <class F>
int with_label_width_or_none(int label_bytes, F&& f) {
  if (label_bytes == 0) return f(std::integral_constant<int, 0>{});
  return with_label_width(label_bytes, f);
}

// cuTensorMapEncodeTiled, fetched through the runtime so that libcuda is not a link-time
// dependency (the library must load on machines without a driver, e.g. for the build check).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
EncodeTiledFn tensor_map_encoder();

// Per-device cached state.  `lock` guards the mutable members (buffers, tables, streams); it is
// held only while they are looked up or changed, never across a whole transform.  `host_call`
// serialises the calls that stage HOST buffers through this device's cached device buffers --
// calls on different devices run concurrently.
struct DeviceCache {
  std::mutex lock;
  std::mutex host_call;
  void* labels = nullptr;
  size_t labels_bytes = 0;
  float* dist = nullptr;
  size_t dist_bytes = 0;
  cudaStream_t stream = nullptr;
  // second slot + copy streams + events of edtb200_transform_batch (slot 0 is labels / dist above)
  void* labels2 = nullptr;
  size_t labels2_bytes = 0;
  float* dist2 = nullptr;
  size_t dist2_bytes = 0;
  cudaStream_t stream_up = nullptr, stream_down = nullptr;
  cudaEvent_t ev_up[2] = {nullptr, nullptr}, ev_comp[2] = {nullptr, nullptr}, ev_down[2] = {nullptr, nullptr};
  // step tables T[k] of the first-axis pass, keyed by the weight's bits (see step_table_kernel).
  // A table remembers the streams that used it (one event each) so that it can be retired
  // without a device-wide synchronisation when the cache is full.  `pinned` counts the launches
  // that hold the table between step_table and step_table_used -- their use is not recorded yet,
  // so the table must not be retired then.
  struct Table {
    float* data = nullptr; int count = 0; uint32_t wbits = 0; uint64_t stamp = 0;
    cudaEvent_t ready = nullptr; cudaStream_t built_on = nullptr;
    static constexpr int kUsers = 4;
    cudaStream_t user[kUsers] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t used[kUsers] = {nullptr, nullptr, nullptr, nullptr};
    bool user_set[kUsers] = {false, false, false, false};
    bool many_users = false;
    int pinned = 0;
  };
  static constexpr int kTables = 16;
  Table tables[kTables];
  uint64_t table_clock = 0;
  std::condition_variable table_unpinned;   // with `lock`: a pinned table was released
  cudaMemPool_t pool = nullptr;        // private pool of the stream-ordered scratch allocations
  // run statistic of the first-axis pass (see RunStat): a ring of device counter / ticket pairs,
  // one per X launch (run_stat), so that X passes running at the same time on different streams
  // count and publish apart; and a mapped host word pair that every launch publishes to
  static constexpr int kStatSlots = 64;
  void* stat_slots = nullptr;          // kStatSlots x 16 bytes: counter (8), ticket (4), padding
  unsigned stat_next = 0;
  volatile unsigned long long* stat_publish_host = nullptr;
  unsigned long long* stat_publish_dev = nullptr;
  int sm_count = 0;
  int max_smem_optin = 0;
  bool probed = false;
};

// Stream-ordered scratch from the device's private pool (never the process-wide default pool).
cudaError_t scratch_alloc(DeviceCache& dc, void** p, size_t bytes, cudaStream_t stream);

// One scratch_alloc allocation, freed on the stream it was taken on when its owner goes out of
// scope -- on every exit of the call that took it.
class Scratch {
 public:
  Scratch() = default;
  Scratch(Scratch&& o) noexcept : p_(o.p_), stream_(o.stream_) { o.p_ = nullptr; }
  Scratch& operator=(Scratch&&) = delete;
  ~Scratch() { if (p_) cudaFreeAsync(p_, stream_); }
  cudaError_t alloc(DeviceCache& dc, size_t bytes, cudaStream_t stream) {
    stream_ = stream;
    const cudaError_t e = scratch_alloc(dc, &p_, bytes, stream);
    if (e != cudaSuccess) p_ = nullptr;
    return e;
  }
  // alloc, failing with "no device memory for <what>" (and the sticky error cleared) when it cannot.
  int take(DeviceCache& dc, size_t bytes, cudaStream_t stream, const char* what) {
    if (alloc(dc, bytes, stream) == cudaSuccess) return 0;
    cudaGetLastError();
    return fail(EDTB200_ENOMEM, "no device memory for %s", what);
  }
  template <class T = void>
  T* get() const { return static_cast<T*>(p_); }

 private:
  void* p_ = nullptr;
  cudaStream_t stream_ = nullptr;
};

// Device table T[0..count) for weight w, cached per device; pinned until step_table_used.
int step_table(DeviceCache& dc, float w, int count, cudaStream_t stream, const float** out);
// Unpins table `data`.  queued: the kernel reading it is queued on `stream` (recorded, so that the
// table can be retired later without a device-wide synchronisation); false: the launch failed.
int step_table_used(DeviceCache& dc, const float* data, cudaStream_t stream, bool queued);

// The step table of one launch: pinned from get() until queued() says the kernel reading it is on
// the stream, or until it goes out of scope on an early return.
class StepTable {
 public:
  StepTable(DeviceCache& dc, cudaStream_t stream) : dc_(dc), stream_(stream) {}
  StepTable(const StepTable&) = delete;
  StepTable& operator=(const StepTable&) = delete;
  ~StepTable() { if (data_) step_table_used(dc_, data_, stream_, false); }
  int get(float w, int count) { return step_table(dc_, w, count, stream_, &data_); }
  const float* data() const { return data_; }
  int queued() {
    const float* d = data_;
    data_ = nullptr;
    return step_table_used(dc_, d, stream_, true);
  }

 private:
  DeviceCache& dc_;
  cudaStream_t stream_;
  const float* data_ = nullptr;
};

// The run statistic of one first-axis launch over `voxels` voxels: the next counter / ticket pair
// of the device's ring (no counters: the launch publishes nothing).
RunStat run_stat(DeviceCache& dc, unsigned long long voxels);

// Arithmetic of one later-axis pass.  int_hull: every sample is an integer and every
// g = f + w2 v^2 an exact 32-bit integer (the integer hull tests apply).  exact: every candidate
// w2 d^2 + f is exact in double, so the tile kernels' fused multiply-add rounds the reference's
// sum; otherwise the long-line kernel forms every candidate in double.
struct PassArith { bool int_hull = false, exact = false; };
// The pass along axis k of a transform with weights w[0..k] over the volume's extents n[0..k].
PassArith transform_arith(const float* w, const int64_t* n, int k);
// A pass with weight w over lines of n samples whose largest finite magnitude is fmax and whose
// lowest set bit over the finite non-zero samples is 2^low (1024: there is none).
PassArith sampled_arith(float fmax, int low, float w, int64_t n);

// One transform: each of its passes derives its kernel flags and arithmetic from these.  w and n
// are the weights and extents of the whole volume, whatever part of it a pass covers.
struct Transform {
  int label_bytes, ndim, flags, border;
  float w[3];
  int64_t n[3];
};

// Kernel flags of a pass from the ABI flags: sqrt and sign act in the store of the last pass;
// background-as-label (sdf) changes the first pass only -- later passes treat every run alike.
inline int kernel_flags(int flags, bool first, bool last) {
  const int epilogue = ((flags & EDTB200_SQRT) ? kSqrt : 0) | ((flags & EDTB200_SIGNED) ? kNegate : 0);
  return (last ? epilogue : 0) | (first && (flags & EDTB200_SIGNED) ? kZeroLabel : 0);
}

// The lines of the later pass along `axis` over `count` volumes of (sx, sy, sz) laid end to end: the
// outer dimension walks the volumes, so that no line crosses from one volume into the next.
inline LineGeom geom_for_axis(int axis, int64_t sx, int64_t sy, int64_t sz, int64_t count = 1) {
  LineGeom g;
  if (axis == 1) {
    g.outer_count = sz * count; g.outer_stride = sx * sy; g.inner_count = sx; g.line_stride = sx; g.n = (int)sy;
  } else {
    g.outer_count = count; g.outer_stride = count > 1 ? sx * sy * sz : 0; g.inner_count = sx * sy;
    g.line_stride = sx * sy; g.n = (int)sz;
  }
  g.tiles_per_outer = 0;
  return g;
}

// Whether launch_first runs the register-resident X kernels (rows of at most 1024 voxels, a multiple
// of 4, labels and distances aligned for vector access) -- the only ones that write XPlanes.
inline bool first_is_vec(const void* labels, int label_bytes, const float* f, int64_t sx) {
  return sx % 4 == 0 && sx <= 1024 && reinterpret_cast<uintptr_t>(labels) % (4 * label_bytes) == 0 &&
         reinterpret_cast<uintptr_t>(f) % 16 == 0;
}

// Axis-pass launchers, one instantiation per label width (edt_passes.cuh).  planes: the run-start
// planes the X pass writes (null: none), where noise_plan takes them.
// planned: what noise_plan planned for the later pass (null: it reads the noise prediction at launch
// and no plane).
struct LaterNoise;
// The march of the plane-writing X pass (first_axis_planes_kernel), for edtb200_noise_planes: the y-chunks
// per slice and the CTAs a caller asks for (0: launch_first_vec's own rule), then what was launched.
struct PlanesMarch {
  int64_t want_chunks = 0, want_ctas = 0;
  int k = 0, plain = 0, planes = 0;            // the instance <Bytes, K, Plain, Planes>
  int64_t nchunks = 0, items = 0, grid = 0;
};
template <int Bytes>
int launch_first(const void* labels, float* f, int64_t nlines, int64_t sx, float w, int border, int flags,
                 const XPlanes* planes, DeviceCache& dc, cudaStream_t stream, PlanesMarch* march = nullptr);
template <int Bytes>
int launch_later(const void* labels, const LaterNoise* planned, float* f, const LineGeom& g0, float w,
                 int border_lo, int border_hi, int flags, PassArith arith, DeviceCache& dc, cudaStream_t stream,
                 bool pdl);
// The site-tracking passes of the feature transform and the kernel that resolves their codes
// into coordinate planes (edt_passes.cuh, edt_feature.cuh).
template <int Bytes>
int launch_first_sites(const void* labels, float* f, int* codes, int64_t nlines, int64_t sx, float w, int border,
                       int flags, DeviceCache& dc, cudaStream_t stream);
template <int Bytes>
int launch_later_sites(const void* labels, const float* fin, float* fout, int* codes, const LineGeom& g, float w,
                       int border_lo, int border_hi, int flags, PassArith arith, DeviceCache& dc,
                       cudaStream_t stream);
template <int Bytes>
int launch_resolve_sites(const void* labels, const int* const codes[3], int ndim, int64_t sx, int64_t sy,
                         int64_t sz, int64_t count, bool zero_is_background, int32_t* const idx[3], DeviceCache& dc,
                         cudaStream_t stream);
// The two halves of that resolution for the chunked feature transform (edt_feature.cuh): phase 1
// resolves the X and Y codes of a slab into sites within each slice, phase 2 follows the last axis's
// codes of a box of whole lines to those partial sites.
template <int Bytes>
int launch_slice_sites(const void* labels, const int* xcodes, int* ycodes_qy, int64_t sx, int64_t sy, int64_t sz,
                       bool zero_is_background, int32_t* qx, DeviceCache& dc, cudaStream_t stream);
template <int Bytes>
int launch_compose_sites(const void* labels, int* codes_last, const int32_t* part_x, const int32_t* part_y,
                         const SiteBox& box, bool zero_is_background, int32_t* out_x, int32_t* out_y, DeviceCache& dc,
                         cudaStream_t stream);
// expand_labels' gather from a signed feature transform's distances and index planes over `count`
// volumes (edt_feature.cuh); as_float: 4- / 8-byte IEEE labels, -0.0 is background.  out may be labels.
template <int Bytes>
int launch_expand_gather(const void* labels, const float* sqdist, const int32_t* const idx[3], int ndim, int64_t sx,
                         int64_t sy, int64_t sz, int64_t count, double limit_sq, bool as_float, void* out,
                         DeviceCache& dc, cudaStream_t stream);

// The plan of a bounded transform (plan_bounded, edt_passes.cuh): the cut B -- the largest float32
// whose double is at most max_distance^2 -- and per axis the window radius R_k and whether the later
// pass along it takes the window kernel (edt_bounded.cuh).
struct BoundedPlan {
  float bound = 0.0f;
  int64_t radius[3] = {0, 0, 0};
  bool windowed[3] = {false, false, false};
};
// The largest radius a window kernel is launched with (its tile then holds 64 + 256 rows).
constexpr int kWindowRadiusLimit = 128;
// plan_bounded with the windows of at most EDTB200_BOUNDED_WINDOW_MAX rows (sites: the feature
// transform's EDTB200_BOUNDED_SITES_WINDOW_MAX), or EDTB200_BOUNDED_RMAX for both (an A/B switch for
// measurements; -1: no pass is windowed) (edt_plan.cu).  max_distance >= 0.
BoundedPlan bounded_plan(int ndim, const float w[3], double max_distance, bool sites);
// The B and R (in radius[0]) of one later pass with weight w that edtb200_pass_window runs: the plan
// above for that axis, every radius up to kWindowRadiusLimit windowed (edt_plan.cu).
BoundedPlan window_pass_plan(float w, double max_distance);

// The bounded transforms' kernels (edt_bounded.cuh, one instantiation per label width in
// edt_bounded.cu).  launch_later_window: the later pass along g out of place (fin -> fout) over the
// samples within `radius` rows, the rows above `bound` written as +inf; codes non-null: also the
// site codes, as launch_later_sites writes them; flags: sqrt / sign in the store (last pass only).
// launch_bounded_cut: in place over `total` voxels, +inf above `bound` (and kSiteNone in codes, when
// given), then flags' sqrt / sign.
template <int Bytes>
int launch_later_window(const void* labels, const float* fin, float* fout, int* codes, const LineGeom& g, float w,
                        int radius, int border_lo, int border_hi, int flags, PassArith arith, float bound,
                        DeviceCache& dc, cudaStream_t stream);
template <int Bytes>
int launch_bounded_cut(const void* labels, float* f, int* codes, int64_t total, float bound, int flags,
                       DeviceCache& dc, cudaStream_t stream);

// The plan of edtb200_nearest_labels (edt_nearest.cu): the bound B and radii R_a of bounded_plan, and
// per axis the kernel its pass takes -- kNearRowsPass (the X pass), kNearStaged or kNearGlobal (a later
// pass whose window tile fits kNearSmemLimit bytes of shared memory, or not), -1 for an axis >= ndim or
// a radius above kNearRadiusLimit.
constexpr int kNearRowsPass = EDTB200_NEAREST_ROWS, kNearStaged = EDTB200_NEAREST_STAGED,
              kNearGlobal = EDTB200_NEAREST_GLOBAL;
constexpr int64_t kNearRadiusLimit = 256;
constexpr size_t kNearSmemLimit = 232448;      // the opt-in shared memory of a CTA on sm_90
struct NearestPlan {
  float bound = 0.0f;
  int64_t radius[3] = {0, 0, 0};
  int variant[3] = {-1, -1, -1};
};
NearestPlan nearest_plan(int ndim, const float w[3], double max_distance, int k, int label_bytes);
// The passes of edtb200_nearest_labels over `count` volumes on the device: k value and label planes to
// dist / lab, through the scratch planes sdist / slab (2-D and 3-D); root: sqrtf in the last store.
int nearest_passes(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count,
                   const float w[3], const NearestPlan& p, int k, bool root, float* dist, void* lab, float* sdist,
                   void* slab, DeviceCache& dc, cudaStream_t stream);

}  // namespace host

// The slots of the surface kernels (edt_surface.cuh): a stack of volumes of (sx, sy, sz), `vol` voxels
// each, nkeys keys, slot s = (volume * nkeys + key) * 2 + direction.  A launch covers the slots
// [s0, s1), and so the volumes [v0, v1).
struct SurfaceSlots {
  int ndim;
  int64_t sx, sy, sz, vol, nkeys;
  int64_t s0, s1, v0, v1;
};

// The last store of a spherical morphology step (edt_morphology.cuh): at voxel p, with nz = src[p] is
// non-zero and near = p's squared distance is within the bound, bit (2 nz + near) of `table` says
// whether p is kept (mask_out: out[p] = 1, else out[p] = src[p]) or not (out[p] = 0).
struct MorphSelect {
  const void* src;     // the caller's labels, src_bytes each, raw bits
  void* out;           // 1 byte per voxel (mask_out) or src_bytes
  int src_bytes;
  int table;
  bool mask_out;
  bool as_float;       // 4- / 8-byte IEEE labels: -0.0 is zero
};

// Whether a raw label is non-zero; as_float: 4- / 8-byte IEEE labels, where -0.0 is zero too.
template <int SrcBytes>
__device__ __forceinline__ bool label_nonzero(typename LabelOf<SrcBytes>::type v, bool as_float) {
  if constexpr (SrcBytes >= 4) {
    using LT = typename LabelOf<SrcBytes>::type;
    if (as_float) return (LT)(v << 1) != 0;                // every bit but the sign
  }
  return v != 0;
}

// One level of local thickness (edt_thickness.cuh): its radius r and cut B = cut_bound(r), for volume v at
// r[v * vstride] and bound[v * vstride] (the default levels, computed on the device), or r0 and b0 for every
// volume when r is null (levels the caller gave).
struct ThicknessLevel {
  const double* r;
  const float* bound;
  int64_t vstride;
  double r0;
  float b0;
};

namespace host {

// The kernels of local thickness over `count` volumes of `vol` voxels (edt_thickness.cu).
// launch_thickness_top: top[v] = 1 + the bits of v's largest finite labelled D2 (0: none; top zeroed
// here).  launch_thickness_levels: the n default levels of every volume from top, descending, and their
// cuts.  launch_thickness_fill: out[v * m + j] = r for every volume.  launch_thickness_seed: mask = 0 where
// D2 > B, else 1.  launch_thickness_store: out = fl32(r) where the voxel is labelled and d2r <= B, taking
// the maximum with out unless `first` (then 0 elsewhere).
int launch_thickness_top(const void* labels, int label_bytes, bool as_float, const float* d2, int64_t vol,
                         int64_t count, unsigned* top, DeviceCache& dc, cudaStream_t stream);
int launch_thickness_levels(const unsigned* top, int64_t count, int n, double h, double* r, float* bound,
                            DeviceCache& dc, cudaStream_t stream);
int launch_thickness_fill(double* out, int64_t count, int m, int j, double r, DeviceCache& dc, cudaStream_t stream);
int launch_thickness_seed(const float* d2, int64_t vol, int64_t count, const ThicknessLevel& level, uint8_t* mask,
                          DeviceCache& dc, cudaStream_t stream);
int launch_thickness_store(const void* labels, int label_bytes, bool as_float, const float* d2r, int64_t vol,
                           int64_t count, const ThicknessLevel& level, bool first, float* out, DeviceCache& dc,
                           cudaStream_t stream);

// The morphology's kernels (edt_morphology.cu).  launch_window_select: the last later pass along g as
// launch_later_window, with the select in its store (label_bytes: the transform's labels, 1 or
// sel.src_bytes).  launch_morph_select: the select over `total` values f.  launch_fold_float_labels:
// out = in with -0.0 as +0.0, for 4- / 8-byte float labels.
int launch_window_select(const void* labels, int label_bytes, const float* fin, const LineGeom& g, float w,
                         int radius, int border_lo, int border_hi, PassArith arith, float bound,
                         const MorphSelect& sel, DeviceCache& dc, cudaStream_t stream);
int launch_morph_select(const float* f, int64_t total, float bound, const MorphSelect& sel, DeviceCache& dc,
                        cudaStream_t stream);
int launch_fold_float_labels(const void* in, int label_bytes, void* out, int64_t total, DeviceCache& dc,
                             cudaStream_t stream);

// One pass of a parabolic erosion (dilate: dilation) along the lines of g, in -> out (in == out: in
// place), with weight w (edt_parabolic.cu).  rows: the X pass, whose lines are g.outer_count rows of
// g.n contiguous samples g.outer_stride apart (inner_count 1, line_stride 1).  *kernel: what ran --
// 0 the tile kernel, 1 the long-line hull, 2 the brute-force minimum, 3 the copy of an overflowing w^2.
// codes non-null: the site-tracking instances, which also write every sample's site code (its winning
// row on its line, or kSiteNone) to codes, laid out like out; lines of at most kParabolicSitesN samples,
// beyond which (i-j)^2 is not exact in double.
constexpr int64_t kParabolicSitesN = (int64_t)1 << 26;
int launch_parabolic_pass(const float* in, float* out, const LineGeom& g, bool rows, float w, bool dilate,
                          DeviceCache& dc, cudaStream_t stream, int* kernel, int* codes = nullptr);

// The medial axis's last step over `count` volumes of (sx, sy, sz) (edt_medial.cu): every labelled voxel
// (as_float: 4- / 8-byte IEEE labels, -0.0 is background) follows the parabolic passes' codes to its site
// and sets medial there; dist non-null: D^2 in place -> its correctly rounded sqrt.
int launch_medial_mark(const void* labels, int label_bytes, const int* const codes[3], int ndim, int64_t sx,
                       int64_t sy, int64_t sz, int64_t count, bool as_float, uint8_t* medial, float* dist,
                       DeviceCache& dc, cudaStream_t stream);

// The skeleton's scratch (edt_skeleton.cu): two list buffers of `segments` segments of `cap` 4-byte entries
// each, and the control block (skeleton_control_bytes()).
struct SkeletonScratch {
  uint32_t* list = nullptr;
  void* control = nullptr;
  int segments = 0;
  uint32_t cap = 0;
};

// The thinning of skeletonize over `count` volumes of (sx, sy, sz) (edt_skeleton.cu): one cooperative
// launch of skeleton_thin_kernel on the edtsq r, h the least weight; keeps its state plane in skeleton and
// leaves the result there (0 / 1); dist
// non-null, the correctly rounded sqrt of r into dist (which may be r itself).
int launch_skeleton_thin(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                         int64_t count, float h, const float* r, const SkeletonScratch& scratch, uint8_t* skeleton,
                         float* dist, DeviceCache& dc, cudaStream_t stream);
size_t skeleton_control_bytes();
// The rounds, cycles and steps of the last thinning on `control` (synchronous copy).
int skeleton_stats(const void* control, unsigned long long out[3]);

// The scratch of geodesic_distance (edt_geodesic.cu): D (one double per voxel), S (one 8-byte index per
// voxel, with indices), one flag per tile, two worklists of `ntiles` 4-byte entries and the control blocks of
// the two phases (geodesic_control_bytes()).
struct GeodesicScratch {
  double* d = nullptr;
  unsigned long long* s = nullptr;
  uint32_t* flag = nullptr;
  uint32_t* list = nullptr;
  void* control = nullptr;
  int64_t ntiles = 0;
};

// The tiles of `count` volumes of (sx, sy, sz) (3-D 8x8x8, 2-D 16x16, 1-D 256 voxels each).
int64_t geodesic_tiles(int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count);
// One phase of geodesic_distance (edt_geodesic.cu): its seed kernel, then ONE cooperative launch of
// geodesic_relax_kernel that runs every round.  index false: D from the seeds; true: S over the tight edges
// of the fixed D.  step[|dx| | |dy| << 1 | |dz| << 2]: the step lengths the host formed.
int launch_geodesic_phase(const void* labels, int label_bytes, const void* seeds, int seed_bytes, int ndim,
                          int64_t sx, int64_t sy, int64_t sz, int64_t count, const double step[8],
                          const GeodesicScratch& g, bool index, DeviceCache& dc, cudaStream_t stream);
// float32(D) into dist and, with planes (null: none), S as int32 coordinate planes within each volume.
int launch_geodesic_store(int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count, const GeodesicScratch& g,
                          float* dist, int32_t* const planes[3], DeviceCache& dc, cudaStream_t stream);
size_t geodesic_control_bytes();
// The rounds and tile visits of the distance and index phases of the last call on `control` (synchronous).
int geodesic_stats(const void* control, unsigned long long out[4]);

// The scratch of watershed (edt_watershed.cu): L (one float per voxel), W (4 bytes per voxel, 8 for 8-byte
// markers), one flag per tile and two worklists of `ntiles` (geodesic_tiles) 4-byte entries, and the control
// blocks of the two phases (watershed_control_bytes()).
struct WatershedScratch {
  float* level = nullptr;
  void* w = nullptr;
  uint32_t* flag = nullptr;
  uint32_t* list = nullptr;
  void* control = nullptr;
  int64_t ntiles = 0;
};

// One phase of watershed (edt_watershed.cu): its seed kernel, then ONE cooperative launch of
// watershed_relax_kernel that runs every round.  label_phase false: L from the seeds; true: W over the tight
// edges of the fixed L.  label_bytes 0: no labels.
int launch_watershed_phase(const void* labels, int label_bytes, const void* markers, int marker_bytes,
                           const float* image, int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count,
                           int connectivity, const WatershedScratch& g, bool label_phase, DeviceCache& dc,
                           cudaStream_t stream);
// W into `out` in the markers' width (0 where there is none) and, with level_out (null: none), L.
int launch_watershed_store(int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count, int marker_bytes,
                           const WatershedScratch& g, void* out, float* level_out, DeviceCache& dc,
                           cudaStream_t stream);
size_t watershed_control_bytes();
// The rounds and tile visits of the level and label phases of the last call on `control` (synchronous).
int watershed_stats(const void* control, unsigned long long out[4]);

// The reconstruction of extended_maxima for h > 0 (edt_watershed.cu): -R, the least fixed point of
// R[v] = max(R[v], min(f[v], R[u])) from m = fl32(f - h), into g.level, by the level phase of watershed on
// negated values (altitude -f, written into neg_image, every node seeded at -m).  g as for watershed.
int launch_hmax_phase(const void* labels, int label_bytes, const float* image, double h, float* neg_image, int ndim,
                      int64_t sx, int64_t sy, int64_t sz, int64_t count, int connectivity, const WatershedScratch& g,
                      DeviceCache& dc, cudaStream_t stream);

// One call of connected_components or extended_maxima (edt_components.cu).  value null: the components of the
// labels; else the plateaus of R (value = f as given, or -R with negated) and the mark pass.
struct ComponentsJob {
  const void* labels = nullptr;
  int label_bytes = 0;              // 0: no labels
  const float* value = nullptr;
  bool negated = false;
  uint32_t* parent = nullptr;       // one 4-byte parent per voxel
  int ndim = 3;
  int64_t sx = 1, sy = 1, sz = 1, count = 1;
  int connectivity = 1;
  int out_bytes = 4;
};
// The scratch of launch_components_number (the per-volume counts of a stack and cub's scan scratch).
size_t components_temp_bytes(int64_t total, int64_t count, int out_bytes);
// The tile pass and the border pass: P[v] = a node of v's component, its least index once both have run.
int launch_components_union(const ComponentsJob& j, DeviceCache& dc, cudaStream_t stream);
// The flatten pass (P = root, flags in out) and, for the plateaus, the mark pass.
int launch_components_flatten(const ComponentsJob& j, void* out, DeviceCache& dc, cudaStream_t stream);
// The per-volume prefix sum in place over out and the number pass.
int launch_components_number(const ComponentsJob& j, void* out, void* temp, size_t temp_bytes, DeviceCache& dc,
                             cudaStream_t stream);

// One call of fill_holes or dust (edt_holes.cu): cc holds the labels, the geometry, the connectivity and the
// parents; the buffers below are indexed by root and zeroed before the tally.
struct HolesJob {
  ComponentsJob cc;
  bool fill = false;                // fill_holes, else dust
  uint32_t* size = nullptr;         // one 4-byte size per voxel (null: fill_holes without max_size)
  void* claim = nullptr;            // fill_holes: 4 bytes per voxel (8 with 8-byte labels)
  uint8_t* state = nullptr;         // fill_holes: 1 byte per voxel, 4-byte aligned, padded to 4 bytes
  uint64_t bound = 0;               // fill_holes: max_size (all ones: none); dust: threshold
  bool invert = false;              // dust
  unsigned long long* counts = nullptr;   // fill_holes: voxels filled per volume, or null
};
// The union: the tile and border passes on the background key (fill_holes) or the label key (dust).
int launch_holes_union(const HolesJob& j, DeviceCache& dc, cudaStream_t stream);
// The tally pass: P = root, sizes, and for fill_holes the OPEN / MIXED bits and the claims at the roots.
int launch_holes_tally(const HolesJob& j, DeviceCache& dc, cudaStream_t stream);
// The apply pass: out in the labels' width, and the fill counts.
int launch_holes_apply(const HolesJob& j, void* out, DeviceCache& dc, cudaStream_t stream);

// The surface kernels, one instantiation per label width in edt_surface.cu.  keys: nkeys labels on the
// device.  mask non-null: surface_mask_kernel into the masks of slots [s0, s1); else values non-null:
// surface_gather_kernel of `dist` (the masks' distances) through `cursor` (one per slot of the range);
// else surface_count_kernel, adding into `cursor`.
template <int Bytes>
int launch_surface(const void* a, const void* b, const void* keys, const SurfaceSlots& g, uint8_t* mask,
                   const float* dist, unsigned long long* cursor, float* values, DeviceCache& dc, cudaStream_t stream);

// Whether plan_later (edt_passes.cuh) sends a later-axis pass over geometry g with arithmetic
// `arith` to the long-line kernel (edt_plan.cu).
bool later_pass_is_long(const LineGeom& g, PassArith arith, int max_smem_optin);

// What a later-axis launch runs (plan_later in edt_passes.cuh); the last one launched on the
// calling thread is kept for edtb200_last_later_launch.
struct LaterLaunch {
  int kernel = -1;      // 0 = tile kernel, 1 = long-line kernel, 2 = window kernel, -1 = no launch yet
  // tx: the tile width, or the window kernel's radius
  int tx = 0, tma = 0, wide = 0, ctas = 0, int_hull = 0, epilogue = 0, all_double = 0;
  int settled = 0;      // tiles whose voxels the X pass left settled are skipped (plan_noise)
};
extern thread_local LaterLaunch g_last_later;

// The label-noise plan of one transform (plan_noise, edt_passes.cuh): the run-start planes its X pass
// writes (XPlanes) and how each later pass k >= 1 uses them.
struct NoisePlan {
  bool noise = false;          // the one reading of the noise prediction that every pass plans with
  int planes = 0;              // later axes the X pass writes planes for: 0 none, 1 y, 2 y and z
  LaterLaunch later[3];        // what launch_later plans for axis k; settled: it skips settled tiles
  bool reads[3] = {false, false, false};   // axis k reads its run-start plane instead of the labels
  int group[3] = {1, 1, 1};    // tiles per CTA of axis k
  bool refresh = false;        // the Y pass refreshes the Z pass's settled plane
};
// plan_noise for transform t over `count` volumes laid end to end at labels / f on this device, with
// one reading of the noise prediction and the A/B switches of the later passes (edt_plan.cu).  noise
// 0 / 1: plan as if the prediction were that instead (edtb200_noise_planes); -1: read it.
NoisePlan noise_plan(const Transform& t, int64_t count, const void* labels, const float* f, const DeviceCache& dc,
                     int noise = -1);

// One later pass of run_passes as noise_plan planned it: the prediction it plans with and, where it
// reads its run-start plane (bits.start non-null), the plan that plane was armed for.
struct LaterNoise {
  bool noise = false;
  RunBits bits = {};
  LaterLaunch plan;
};

}  // namespace host
}  // namespace edtb200
