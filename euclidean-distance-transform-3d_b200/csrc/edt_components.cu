// connected_components' and extended_maxima's union-find passes and numbering for every label width, no labels
// included (see edt_components.cuh).
#include <cub/device/device_scan.cuh>

#include "edt_components.cuh"

namespace edtb200 {
namespace host {

namespace {

constexpr int kCcTileDims[4][3] = {{0, 0, 0}, {1024, 1, 1}, {32, 32, 1}, {16, 8, 8}};

}  // namespace

CcArgs cc_args(const ComponentsJob& j) {
  CcArgs a{};
  a.parent = j.parent;
  a.labels = j.labels;
  a.value = j.value;
  a.negated = j.negated;
  a.sx = j.sx; a.sy = j.sy; a.sz = j.sz; a.vol = j.sx * j.sy * j.sz; a.total = a.vol * j.count;
  a.tx = kCcTileDims[j.ndim][0]; a.ty = kCcTileDims[j.ndim][1]; a.tz = kCcTileDims[j.ndim][2];
  a.nx = (j.sx + a.tx - 1) / a.tx; a.ny = (j.sy + a.ty - 1) / a.ty; a.nz = (j.sz + a.tz - 1) / a.tz;
  a.ntiles = a.nx * a.ny * a.nz * j.count;
  a.ndim = j.ndim;
  a.connectivity = j.connectivity;
  return a;
}

unsigned cc_blocks(int64_t n, const DeviceCache& dc) {
  const int64_t blocks = (n + kCcThreads - 1) / kCcThreads, cap = (int64_t)dc.sm_count * 16;
  return (unsigned)(blocks > cap ? cap : blocks < 1 ? 1 : blocks);
}

namespace {

template <class F>
int with_out_width(int out_bytes, F&& f) {
  if (out_bytes == 8) return f((unsigned long long*)nullptr);
  return f((uint32_t*)nullptr);
}

// The cub scratch of the in-place prefix sum over the stack.
template <class OT>
size_t cc_scan_bytes(int64_t total) {
  size_t bytes = 0;
  cub::DeviceScan::InclusiveSum(nullptr, bytes, (OT*)nullptr, (OT*)nullptr, total);
  return bytes;
}

}  // namespace

size_t components_temp_bytes(int64_t total, int64_t count, int out_bytes) {
  const size_t counts = count > 1 ? sizeof(unsigned long long) * (size_t)count : 0;
  const size_t scan = out_bytes == 8 ? cc_scan_bytes<unsigned long long>(total) : cc_scan_bytes<uint32_t>(total);
  return ((counts + 255) & ~(size_t)255) + scan;
}

int launch_components_union(const ComponentsJob& j, DeviceCache& dc, cudaStream_t stream) {
  const CcArgs a = cc_args(j);
  const int64_t tile_grid = a.ntiles < (int64_t)dc.sm_count * 32 ? a.ntiles : (int64_t)dc.sm_count * 32;
  return with_label_width_or_none(j.label_bytes, [&](auto b) {
    constexpr int LB = decltype(b)::value;
    if (j.value) {
      components_tile_kernel<CcPlateauKey<LB>><<<(unsigned)tile_grid, kCcThreads, 0, stream>>>(a);
      components_border_kernel<CcPlateauKey<LB>><<<cc_blocks(a.total, dc), kCcThreads, 0, stream>>>(a);
    } else {
      components_tile_kernel<CcLabelKey<LB>><<<(unsigned)tile_grid, kCcThreads, 0, stream>>>(a);
      components_border_kernel<CcLabelKey<LB>><<<cc_blocks(a.total, dc), kCcThreads, 0, stream>>>(a);
    }
    CUDA_TRY(cudaGetLastError());
    return 0;
  });
}

int launch_components_flatten(const ComponentsJob& j, void* out, DeviceCache& dc, cudaStream_t stream) {
  const CcArgs a = cc_args(j);
  const unsigned blocks = cc_blocks(a.total, dc);
  return with_out_width(j.out_bytes, [&](auto* tag) {
    using OT = std::remove_pointer_t<decltype(tag)>;
    components_flatten_kernel<OT><<<blocks, kCcThreads, 0, stream>>>(a, static_cast<OT*>(out));
    CUDA_TRY(cudaGetLastError());
    if (!j.value) return 0;
    return with_label_width_or_none(j.label_bytes, [&](auto b) {
      components_mark_kernel<decltype(b)::value, OT><<<blocks, kCcThreads, 0, stream>>>(a, static_cast<OT*>(out));
      CUDA_TRY(cudaGetLastError());
      return 0;
    });
  });
}

int launch_components_number(const ComponentsJob& j, void* out, void* temp, size_t temp_bytes, DeviceCache& dc,
                             cudaStream_t stream) {
  const CcArgs a = cc_args(j);
  return with_out_width(j.out_bytes, [&](auto* tag) {
    using OT = std::remove_pointer_t<decltype(tag)>;
    OT* flags = static_cast<OT*>(out);
    char* scan = static_cast<char*>(temp);
    size_t scan_bytes = temp_bytes;
    if (j.count > 1) {
      // each volume numbered from 1: lower its first flag by the kept roots of the volume before it, which is
      // what the prefix sum carries into it once every earlier volume's first flag has been lowered too
      auto* counts = reinterpret_cast<unsigned long long*>(scan);
      const size_t counts_bytes = (sizeof(unsigned long long) * (size_t)j.count + 255) & ~(size_t)255;
      scan += counts_bytes;
      scan_bytes -= counts_bytes;
      CUDA_TRY(cudaMemsetAsync(counts, 0, sizeof(unsigned long long) * (size_t)j.count, stream));
      const int64_t chunks = (a.vol + kCcChunk - 1) / kCcChunk;
      components_count_kernel<OT><<<(unsigned)(chunks * j.count), kCcThreads, 0, stream>>>(flags, a.vol, chunks, counts);
      CUDA_TRY(cudaGetLastError());
      components_rebase_kernel<OT><<<cc_blocks(j.count, dc), kCcThreads, 0, stream>>>(flags, a.vol, j.count, counts);
      CUDA_TRY(cudaGetLastError());
    }
    CUDA_TRY(cub::DeviceScan::InclusiveSum(scan, scan_bytes, flags, flags, a.total, stream));
    components_number_kernel<OT><<<cc_blocks(a.total, dc), kCcThreads, 0, stream>>>(a, flags);
    CUDA_TRY(cudaGetLastError());
    return 0;
  });
}

}  // namespace host
}  // namespace edtb200
