// The medial axis's mark kernel for every label width (see edt_medial.cuh).
#include "edt_medial.cuh"

namespace edtb200 {
namespace host {

int launch_medial_mark(const void* labels, int label_bytes, const int* const codes[3], int ndim, int64_t sx,
                       int64_t sy, int64_t sz, int64_t count, bool as_float, uint8_t* medial, float* dist,
                       DeviceCache& dc, cudaStream_t stream) {
  const int64_t total = sx * sy * sz * count;
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = (int64_t)dc.sm_count * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  const SiteCodes c{{codes[0], codes[1], codes[2]}, ndim, sx, sy, sz * count, sz};
  return with_label_width(label_bytes, [&](auto b) {
    constexpr int B = decltype(b)::value;
    medial_mark_kernel<B><<<(unsigned)blocks, 256, 0, stream>>>(static_cast<const typename LabelOf<B>::type*>(labels),
                                                                c, as_float ? 1 : 0, medial, dist);
    CUDA_TRY(cudaGetLastError());
    return 0;
  });
}

}  // namespace host
}  // namespace edtb200
