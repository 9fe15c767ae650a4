// The skeleton's thinning kernel for every label width (see edt_skeleton.cuh).
#include "edt_skeleton.cuh"

namespace edtb200 {
namespace host {

int launch_skeleton_thin(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                         int64_t count, float h, const float* r, const SkeletonScratch& scratch, uint8_t* skeleton,
                         float* dist, DeviceCache& dc, cudaStream_t stream) {
  SkelArgs a{};
  a.r = r;
  a.state = skeleton;
  a.list[0] = scratch.list;
  a.list[1] = scratch.list + (size_t)scratch.segments * scratch.cap;
  a.ctl = static_cast<SkelControl*>(scratch.control);
  a.dist = dist;
  a.sx = sx; a.sy = sy; a.sz = sz; a.count = count; a.total = sx * sy * sz * count;
  a.hx = (uint32_t)((sx + 1) / 2); a.hy = (uint32_t)((sy + 1) / 2); a.hz = (uint32_t)((sz + 1) / 2);
  a.cap = scratch.cap;
  a.ndim = ndim;
  a.h = (double)h;
  CUDA_TRY(cudaMemsetAsync(scratch.control, 0, sizeof(SkelControl), stream));
  return with_label_width(label_bytes, [&](auto b) {
    constexpr int B = decltype(b)::value;
    using LT = typename LabelOf<B>::type;
    // the grid barrier needs every block resident at once: as many blocks as fit, no more than the work
    int per_sm = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, skeleton_thin_kernel<B>, 256, 0));
    int64_t blocks = (int64_t)per_sm * dc.sm_count;
    const int64_t want = (a.total + 255) / 256;
    if (blocks > want) blocks = want;
    if (blocks < 1) blocks = 1;
    const LT* typed = static_cast<const LT*>(labels);
    void* args[2] = {(void*)&typed, (void*)&a};
    CUDA_TRY(cudaLaunchCooperativeKernel((const void*)skeleton_thin_kernel<B>, dim3((unsigned)blocks), dim3(256),
                                         args, 0, stream));
    return 0;
  });
}

size_t skeleton_control_bytes() { return sizeof(SkelControl); }

int skeleton_stats(const void* control, unsigned long long out[3]) {
  CUDA_TRY(cudaMemcpy(out, static_cast<const SkelControl*>(control)->stats, 3 * sizeof(unsigned long long),
                      cudaMemcpyDeviceToHost));
  return 0;
}

}  // namespace host
}  // namespace edtb200
