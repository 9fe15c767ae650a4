// Local thickness's kernels (see edt_thickness.cuh): the per-volume maximum of D2, the default levels, the
// seeds and the store of each level.
#include "edt_thickness.cuh"

#include <algorithm>

namespace edtb200 {
namespace host {
namespace {

int64_t flat_blocks(int64_t total, const DeviceCache& dc) {
  const int64_t blocks = std::min<int64_t>((total + 255) / 256, (int64_t)dc.sm_count * 8);
  return blocks < 1 ? 1 : blocks;
}

// Blocks of a per-volume kernel: y walks the volumes, x the voxels of one, about 8 blocks per SM in all.
dim3 volume_grid(int64_t vol, int64_t count, const DeviceCache& dc) {
  const int64_t y = std::min<int64_t>(count, 65535);
  const int64_t per_volume = std::max<int64_t>(1, ((int64_t)dc.sm_count * 8 + y - 1) / y);
  const int64_t x = std::max<int64_t>(1, std::min<int64_t>((vol + 255) / 256, per_volume));
  return dim3((unsigned)x, (unsigned)y);
}

}  // namespace

int launch_thickness_top(const void* labels, int label_bytes, bool as_float, const float* d2, int64_t vol,
                         int64_t count, unsigned* top, DeviceCache& dc, cudaStream_t stream) {
  CUDA_TRY(cudaMemsetAsync(top, 0, sizeof(unsigned) * (size_t)count, stream));
  return with_label_width(label_bytes, [&](auto b) {
    constexpr int B = decltype(b)::value;
    thickness_top_kernel<B><<<volume_grid(vol, count, dc), 256, 0, stream>>>(
        static_cast<const typename LabelOf<B>::type*>(labels), d2, vol, count, as_float ? 1 : 0, top);
    CUDA_TRY(cudaGetLastError());
    return 0;
  });
}

int launch_thickness_levels(const unsigned* top, int64_t count, int n, double h, double* r, float* bound,
                            DeviceCache& dc, cudaStream_t stream) {
  thickness_levels_kernel<<<(unsigned)flat_blocks(count * n, dc), 256, 0, stream>>>(top, count, n, h, r, bound);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_thickness_fill(double* out, int64_t count, int m, int j, double r, DeviceCache& dc, cudaStream_t stream) {
  thickness_fill_kernel<<<(unsigned)flat_blocks(count, dc), 256, 0, stream>>>(out, count, m, j, r);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_thickness_seed(const float* d2, int64_t vol, int64_t count, const ThicknessLevel& level, uint8_t* mask,
                          DeviceCache& dc, cudaStream_t stream) {
  thickness_seed_kernel<<<volume_grid(vol, count, dc), 256, 0, stream>>>(d2, vol, count, level, mask);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int launch_thickness_store(const void* labels, int label_bytes, bool as_float, const float* d2r, int64_t vol,
                           int64_t count, const ThicknessLevel& level, bool first, float* out, DeviceCache& dc,
                           cudaStream_t stream) {
  return with_label_width(label_bytes, [&](auto b) {
    constexpr int B = decltype(b)::value;
    thickness_store_kernel<B><<<volume_grid(vol, count, dc), 256, 0, stream>>>(
        static_cast<const typename LabelOf<B>::type*>(labels), as_float ? 1 : 0, d2r, vol, count, level,
        first ? 1 : 0, out);
    CUDA_TRY(cudaGetLastError());
    return 0;
  });
}

}  // namespace host
}  // namespace edtb200
