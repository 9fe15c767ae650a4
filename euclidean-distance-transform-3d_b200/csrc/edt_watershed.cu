// watershed's seed, relaxation and store kernels for every label width, no labels included (see
// edt_watershed.cuh), and extended_maxima's reconstruction on the level phase's relaxation kernel.
#include "edt_watershed.cuh"

namespace edtb200 {
namespace host {

namespace {

// The tiles of geodesic_tiles: 3-D 8x8x8, 2-D 16x16, 1-D 256 voxels.
constexpr int kWsTile[4][3] = {{0, 0, 0}, {256, 1, 1}, {16, 16, 1}, {8, 8, 8}};

WsArgs ws_args(const WatershedScratch& g, int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count) {
  WsArgs a{};
  a.level = g.level;
  a.w = g.w;
  a.flag = g.flag;
  a.list[0] = g.list;
  a.list[1] = g.list + g.ntiles;
  a.ctl = static_cast<WsControl*>(g.control);
  a.sx = sx; a.sy = sy; a.sz = sz; a.vol = sx * sy * sz; a.total = a.vol * count;
  a.tx = kWsTile[ndim][0]; a.ty = kWsTile[ndim][1]; a.tz = kWsTile[ndim][2];
  a.nx = (sx + a.tx - 1) / a.tx; a.ny = (sy + a.ty - 1) / a.ty; a.nz = (sz + a.tz - 1) / a.tz;
  a.ntiles = a.nx * a.ny * a.nz * count;
  a.ndim = ndim;
  return a;
}

int64_t ws_blocks(int64_t total, const DeviceCache& dc) {
  const int64_t blocks = (total + 255) / 256;
  return blocks > (int64_t)dc.sm_count * 16 ? (int64_t)dc.sm_count * 16 : blocks;
}

// The rounds of one phase in one cooperative launch, after its seed kernel.
template <int LB, class WT, bool Label>
int ws_relax(const void* labels, WsArgs a, DeviceCache& dc, cudaStream_t stream) {
  // the grid barrier needs every block resident at once: as many blocks as fit, no more than the tiles
  int per_sm = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, watershed_relax_kernel<LB, WT, Label>, kWsThreads, 0));
  int64_t grid = (int64_t)per_sm * dc.sm_count;
  if (grid > a.ntiles) grid = a.ntiles;
  if (grid < 1) grid = 1;
  void* args[2] = {(void*)&labels, (void*)&a};
  CUDA_TRY(cudaLaunchCooperativeKernel((const void*)watershed_relax_kernel<LB, WT, Label>, dim3((unsigned)grid),
                                       dim3(kWsThreads), args, 0, stream));
  return 0;
}

// One phase: clear the flags and the control block, seed, then the rounds in one cooperative launch.
template <int LB, class WT, bool Label>
int ws_phase(const void* labels, WsArgs a, DeviceCache& dc, cudaStream_t stream) {
  CUDA_TRY(cudaMemsetAsync(a.flag, 0, sizeof(uint32_t) * (size_t)a.ntiles, stream));
  CUDA_TRY(cudaMemsetAsync(a.ctl, 0, sizeof(WsControl), stream));
  watershed_seed_kernel<LB, WT><<<(unsigned)ws_blocks(a.total, dc), 256, 0, stream>>>(labels, a, Label);
  CUDA_TRY(cudaGetLastError());
  return ws_relax<LB, WT, Label>(labels, a, dc, stream);
}

}  // namespace

int launch_watershed_phase(const void* labels, int label_bytes, const void* markers, int marker_bytes,
                           const float* image, int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count,
                           int connectivity, const WatershedScratch& g, bool label_phase, DeviceCache& dc,
                           cudaStream_t stream) {
  WsArgs a = ws_args(g, ndim, sx, sy, sz, count);
  a.image = image;
  a.markers = markers;
  a.marker_bytes = marker_bytes;
  a.connectivity = connectivity;
  if (label_phase) a.ctl += 1;
  return with_label_width_or_none(label_bytes, [&](auto b) {
    constexpr int LB = decltype(b)::value;
    if (!label_phase) return ws_phase<LB, uint32_t, false>(labels, a, dc, stream);
    return marker_bytes == 8 ? ws_phase<LB, unsigned long long, true>(labels, a, dc, stream)
                             : ws_phase<LB, uint32_t, true>(labels, a, dc, stream);
  });
}

int launch_hmax_phase(const void* labels, int label_bytes, const float* image, double h, float* neg_image, int ndim,
                      int64_t sx, int64_t sy, int64_t sz, int64_t count, int connectivity, const WatershedScratch& g,
                      DeviceCache& dc, cudaStream_t stream) {
  WsArgs a = ws_args(g, ndim, sx, sy, sz, count);
  a.image = image;
  a.connectivity = connectivity;
  return with_label_width_or_none(label_bytes, [&](auto b) {
    constexpr int LB = decltype(b)::value;
    CUDA_TRY(cudaMemsetAsync(a.flag, 0, sizeof(uint32_t) * (size_t)a.ntiles, stream));
    CUDA_TRY(cudaMemsetAsync(a.ctl, 0, sizeof(WsControl), stream));
    hmax_seed_kernel<LB><<<(unsigned)ws_blocks(a.total, dc), 256, 0, stream>>>(labels, a, neg_image, h);
    CUDA_TRY(cudaGetLastError());
    a.image = neg_image;
    return ws_relax<LB, uint32_t, false>(labels, a, dc, stream);
  });
}

int launch_watershed_store(int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count, int marker_bytes,
                           const WatershedScratch& g, void* out, float* level_out, DeviceCache& dc,
                           cudaStream_t stream) {
  const WsArgs a = ws_args(g, ndim, sx, sy, sz, count);
  const unsigned blocks = (unsigned)ws_blocks(a.total, dc);
  switch (marker_bytes) {
    case 1:
      watershed_store_kernel<uint8_t, uint32_t><<<blocks, 256, 0, stream>>>(a, static_cast<uint8_t*>(out), level_out);
      break;
    case 2:
      watershed_store_kernel<uint16_t, uint32_t><<<blocks, 256, 0, stream>>>(a, static_cast<uint16_t*>(out), level_out);
      break;
    case 4:
      watershed_store_kernel<uint32_t, uint32_t><<<blocks, 256, 0, stream>>>(a, static_cast<uint32_t*>(out), level_out);
      break;
    default:
      watershed_store_kernel<unsigned long long, unsigned long long><<<blocks, 256, 0, stream>>>(
          a, static_cast<unsigned long long*>(out), level_out);
      break;
  }
  CUDA_TRY(cudaGetLastError());
  return 0;
}

size_t watershed_control_bytes() { return 2 * sizeof(WsControl); }

int watershed_stats(const void* control, unsigned long long out[4]) {
  WsControl c[2];
  CUDA_TRY(cudaMemcpy(c, control, sizeof(c), cudaMemcpyDeviceToHost));
  out[0] = c[0].rounds; out[1] = c[0].visits; out[2] = c[1].rounds; out[3] = c[1].visits;
  return 0;
}

}  // namespace host
}  // namespace edtb200
