// include/edt.hpp -- C++ drop-in for the reference's public facade `namespace edt`
// (reference src/edt.hpp:805-954): same templates, argument order, defaults and ownership, but
// every call goes through the C ABI of edt_b200.h into the sm_90a kernels.
//
//   float* dt = edt::edt<uint32_t>(labels, sx, sy, sz, wx, wy, wz, black_border);   // x fastest
//   ... delete [] dt;                       // as with the reference: the caller owns the result
//
// `parallel` is accepted and ignored (the CUDA grid replaces the thread pool).  If `output` is
// given it is filled and returned, otherwise a `new float[sx*sy*sz]` is returned
// (reference src/edt.hpp:424-426).  The reference never reports errors; this shim throws
// std::runtime_error carrying edtb200_last_error() when the GPU path fails (there is no CPU
// fallback to hide it).  Link with -ledt_b200.
#ifndef EDT_B200_CPP_SHIM_HPP
#define EDT_B200_CPP_SHIM_HPP

#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include "edt_b200.h"

namespace edt {
namespace detail {

template <typename T>
inline float* run(T* labels, int ndim, int64_t sx, int64_t sy, int64_t sz, float wx, float wy, float wz,
                  bool black_border, int flags, float* output) {
  static_assert(sizeof(T) == 1 || sizeof(T) == 2 || sizeof(T) == 4 || sizeof(T) == 8,
                "labels must be 1, 2, 4 or 8 bytes wide");
  const int64_t voxels = sx * (ndim > 1 ? sy : 1) * (ndim > 2 ? sz : 1);
  float* out = output ? output : new float[voxels > 0 ? voxels : 1]();
  const void* src = labels;
  std::vector<double> canon;                     // scratch, used only for floating-point labels
  if constexpr (std::is_floating_point<T>::value) {   // labels compare by value: fold -0.0 onto +0.0
    canon.resize((static_cast<size_t>(voxels) * sizeof(T) + sizeof(double) - 1) / sizeof(double));
    T* folded = reinterpret_cast<T*>(canon.data());
    for (int64_t i = 0; i < voxels; ++i) folded[i] = labels[i] + T(0);
    src = folded;
  }
  int rc = edtb200_transform(src, (int)sizeof(T), ndim, sx, sy, sz, wx, wy, wz, black_border ? 1 : 0,
                             flags, out, /*device=*/0, /*stream=*/nullptr);
  if (rc == EDTB200_ENOMEM && ndim >= 2)         // larger than the device: stream it through in chunks
    rc = edtb200_transform_chunked(src, (int)sizeof(T), ndim, sx, sy, sz, wx, wy, wz, black_border ? 1 : 0, flags,
                                   out, /*device=*/0, /*device_bytes=*/0, /*chunks=*/nullptr);
  if (rc != 0) {
    if (!output) delete[] out;
    throw std::runtime_error(std::string("edt_b200: ") + edtb200_last_error());
  }
  return out;
}

}  // namespace detail

// ---- 3-D (reference src/edt.hpp:836-844, 907-922) ----
template <typename T>
float* edtsq(T* labels, const int sx, const int sy, const int sz, const float wx, const float wy,
             const float wz, const bool black_border = false, const int parallel = 1, float* output = NULL) {
  (void)parallel;
  return detail::run(labels, 3, sx, sy, sz, wx, wy, wz, black_border, 0, output);
}
template <typename T>
float* edt(T* labels, const int sx, const int sy, const int sz, const float wx, const float wy,
           const float wz, const bool black_border = false, const int parallel = 1, float* output = NULL) {
  (void)parallel;
  return detail::run(labels, 3, sx, sy, sz, wx, wy, wz, black_border, EDTB200_SQRT, output);
}

// ---- 2-D (reference src/edt.hpp:823-834, 895-905) ----
template <typename T>
float* edtsq(T* labels, const int sx, const int sy, const float wx, const float wy,
             const bool black_border = false, const int parallel = 1, float* output = NULL) {
  (void)parallel;
  return detail::run(labels, 2, sx, sy, 1, wx, wy, 1.0f, black_border, 0, output);
}
template <typename T>
float* edt(T* labels, const int sx, const int sy, const float wx, const float wy,
           const bool black_border = false, const int parallel = 1, float* output = NULL) {
  (void)parallel;
  return detail::run(labels, 2, sx, sy, 1, wx, wy, 1.0f, black_border, EDTB200_SQRT, output);
}

// ---- 1-D (reference src/edt.hpp:807-821, 884-893) ----
template <typename T>
float* edtsq(T* labels, const int sx, const float wx, const bool black_border = false) {
  return detail::run(labels, 1, sx, 1, 1, wx, 1.0f, 1.0f, black_border, 0, nullptr);
}
template <typename T>
float* edt(T* labels, const int sx, const float wx, const bool black_border = false) {
  return detail::run(labels, 1, sx, 1, 1, wx, 1.0f, 1.0f, black_border, EDTB200_SQRT, nullptr);
}

// ---- binary_* aliases: the same kernels handle binary images (reference src/edt.hpp:846-954) ----
template <typename T>
float* binary_edtsq(T* labels, const int sx, const int sy, const int sz, const float wx, const float wy,
                    const float wz, const bool black_border = false, const int parallel = 1,
                    float* output = NULL) {
  return edtsq<T>(labels, sx, sy, sz, wx, wy, wz, black_border, parallel, output);
}
template <typename T>
float* binary_edt(T* labels, const int sx, const int sy, const int sz, const float wx, const float wy,
                  const float wz, const bool black_border = false, const int parallel = 1,
                  float* output = NULL) {
  return edt<T>(labels, sx, sy, sz, wx, wy, wz, black_border, parallel, output);
}

// Signed distance function; README.md:138-142 of the reference advertises edt::sdf, which exists
// only in its Python layer (src/edt.pyx:121-202).
template <typename T>
float* sdf(T* labels, const int sx, const int sy, const int sz, const float wx, const float wy,
           const float wz, const bool black_border = false, const int parallel = 1, float* output = NULL) {
  (void)parallel;
  return detail::run(labels, 3, sx, sy, sz, wx, wy, wz, black_border, EDTB200_SQRT | EDTB200_SIGNED, output);
}

}  // namespace edt

#endif  // EDT_B200_CPP_SHIM_HPP
