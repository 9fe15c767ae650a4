// fill_holes' and dust's union, tally and apply passes for every label width (see edt_holes.cuh).
#include "edt_holes.cuh"

namespace edtb200 {
namespace host {

namespace {

HoleArgs hole_args(const HolesJob& j) {
  HoleArgs h{};
  h.cc = cc_args(j.cc);
  h.size = j.size;
  h.claim = j.claim;
  h.state = j.state;
  h.bound = j.bound;
  h.invert = j.invert;
  h.counts = j.counts;
  h.chunks = (h.cc.vol + kCcChunk - 1) / kCcChunk;
  return h;
}

}  // namespace

int launch_holes_union(const HolesJob& j, DeviceCache& dc, cudaStream_t stream) {
  if (!j.fill) return launch_components_union(j.cc, dc, stream);
  const CcArgs a = cc_args(j.cc);
  const int64_t tile_grid = a.ntiles < (int64_t)dc.sm_count * 32 ? a.ntiles : (int64_t)dc.sm_count * 32;
  return with_label_width(j.cc.label_bytes, [&](auto b) {
    constexpr int LB = decltype(b)::value;
    components_tile_kernel<CcHoleKey<LB>><<<(unsigned)tile_grid, kCcThreads, 0, stream>>>(a);
    components_border_kernel<CcHoleKey<LB>><<<cc_blocks(a.total, dc), kCcThreads, 0, stream>>>(a);
    CUDA_TRY(cudaGetLastError());
    return 0;
  });
}

int launch_holes_tally(const HolesJob& j, DeviceCache& dc, cudaStream_t stream) {
  const HoleArgs h = hole_args(j);
  return with_label_width(j.cc.label_bytes, [&](auto b) {
    constexpr int LB = decltype(b)::value;
    if (j.fill) holes_tally_kernel<LB, true><<<cc_blocks(h.cc.total, dc), kCcThreads, 0, stream>>>(h);
    else holes_tally_kernel<LB, false><<<cc_blocks(h.cc.total, dc), kCcThreads, 0, stream>>>(h);
    CUDA_TRY(cudaGetLastError());
    return 0;
  });
}

int launch_holes_apply(const HolesJob& j, void* out, DeviceCache& dc, cudaStream_t stream) {
  const HoleArgs h = hole_args(j);
  const int64_t blocks = h.chunks * j.cc.count, cap = (int64_t)dc.sm_count * 16;
  const unsigned grid = (unsigned)(blocks < cap ? blocks : cap);
  return with_label_width(j.cc.label_bytes, [&](auto b) {
    constexpr int LB = decltype(b)::value;
    using T = typename LabelOf<LB>::type;
    if (j.fill) holes_apply_kernel<LB, true><<<grid, kCcThreads, 0, stream>>>(h, static_cast<T*>(out));
    else holes_apply_kernel<LB, false><<<grid, kCcThreads, 0, stream>>>(h, static_cast<T*>(out));
    CUDA_TRY(cudaGetLastError());
    return 0;
  });
}

}  // namespace host
}  // namespace edtb200
