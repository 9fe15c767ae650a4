// geodesic_distance's seed, relaxation and store kernels for every label width (see edt_geodesic.cuh).
#include "edt_geodesic.cuh"

namespace edtb200 {
namespace host {

namespace {

// The tile of each number of dimensions: 3-D 8x8x8, 2-D 16x16, 1-D 256 voxels.
constexpr int kGeoTile[4][3] = {{0, 0, 0}, {256, 1, 1}, {16, 16, 1}, {8, 8, 8}};

GeoArgs geo_args(const GeodesicScratch& g, int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count,
                 const double step[8]) {
  GeoArgs a{};
  a.d = g.d;
  a.flag = g.flag;
  a.list[0] = g.list;
  a.list[1] = g.list + g.ntiles;
  a.ctl = static_cast<GeoControl*>(g.control);
  a.sx = sx; a.sy = sy; a.sz = sz; a.vol = sx * sy * sz; a.total = a.vol * count;
  a.tx = kGeoTile[ndim][0]; a.ty = kGeoTile[ndim][1]; a.tz = kGeoTile[ndim][2];
  a.nx = (sx + a.tx - 1) / a.tx; a.ny = (sy + a.ty - 1) / a.ty; a.nz = (sz + a.tz - 1) / a.tz;
  a.ntiles = a.nx * a.ny * a.nz * count;
  a.ndim = ndim;
  for (int k = 0; k < 8; ++k) a.step[k] = step[k];
  return a;
}

// One phase: clear the flags and the control block, seed, then the rounds in one cooperative launch.
template <int B, bool Index>
int geo_phase(const void* labels, GeoArgs a, const GeodesicScratch& g, DeviceCache& dc, cudaStream_t stream) {
  using LT = typename LabelOf<B>::type;
  CUDA_TRY(cudaMemsetAsync(g.flag, 0, sizeof(uint32_t) * (size_t)g.ntiles, stream));
  CUDA_TRY(cudaMemsetAsync(g.control, 0, sizeof(GeoControl), stream));
  const LT* typed = static_cast<const LT*>(labels);
  int64_t blocks = (a.total + 255) / 256;
  if (blocks > (int64_t)dc.sm_count * 16) blocks = (int64_t)dc.sm_count * 16;
  geodesic_seed_kernel<B><<<(unsigned)blocks, 256, 0, stream>>>(typed, a);
  CUDA_TRY(cudaGetLastError());
  // the grid barrier needs every block resident at once: as many blocks as fit, no more than the tiles
  int per_sm = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, geodesic_relax_kernel<B, Index>, kGeoThreads, 0));
  int64_t grid = (int64_t)per_sm * dc.sm_count;
  if (grid > a.ntiles) grid = a.ntiles;
  if (grid < 1) grid = 1;
  void* args[2] = {(void*)&typed, (void*)&a};
  CUDA_TRY(cudaLaunchCooperativeKernel((const void*)geodesic_relax_kernel<B, Index>, dim3((unsigned)grid),
                                       dim3(kGeoThreads), args, 0, stream));
  return 0;
}

}  // namespace

int launch_geodesic_phase(const void* labels, int label_bytes, const void* seeds, int seed_bytes, int ndim,
                          int64_t sx, int64_t sy, int64_t sz, int64_t count, const double step[8],
                          const GeodesicScratch& g, bool index, DeviceCache& dc, cudaStream_t stream) {
  GeoArgs a = geo_args(g, ndim, sx, sy, sz, count, step);
  a.seeds = seeds;
  a.seed_bytes = seed_bytes;
  GeodesicScratch phase = g;
  if (index) {
    a.s = g.s;
    phase.control = a.ctl = static_cast<GeoControl*>(g.control) + 1;
  }
  return with_label_width(label_bytes, [&](auto b) {
    constexpr int B = decltype(b)::value;
    return index ? geo_phase<B, true>(labels, a, phase, dc, stream) : geo_phase<B, false>(labels, a, phase, dc, stream);
  });
}

int launch_geodesic_store(int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count, const GeodesicScratch& g,
                          float* dist, int32_t* const planes[3], DeviceCache& dc, cudaStream_t stream) {
  const double none[8] = {};
  GeoArgs a = geo_args(g, ndim, sx, sy, sz, count, none);
  a.s = g.s;
  int64_t blocks = (a.total + 255) / 256;
  if (blocks > (int64_t)dc.sm_count * 16) blocks = (int64_t)dc.sm_count * 16;
  geodesic_store_kernel<<<(unsigned)blocks, 256, 0, stream>>>(a, dist, planes ? planes[0] : nullptr,
                                                               planes ? planes[1] : nullptr,
                                                               planes ? planes[2] : nullptr);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int64_t geodesic_tiles(int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count) {
  const int* t = kGeoTile[ndim];
  return ((sx + t[0] - 1) / t[0]) * ((sy + t[1] - 1) / t[1]) * ((sz + t[2] - 1) / t[2]) * count;
}

size_t geodesic_control_bytes() { return 2 * sizeof(GeoControl); }

int geodesic_stats(const void* control, unsigned long long out[4]) {
  GeoControl c[2];
  CUDA_TRY(cudaMemcpy(c, control, sizeof(c), cudaMemcpyDeviceToHost));
  out[0] = c[0].rounds; out[1] = c[0].visits; out[2] = c[1].rounds; out[3] = c[1].visits;
  return 0;
}

}  // namespace host
}  // namespace edtb200
