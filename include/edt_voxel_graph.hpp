// include/edt_voxel_graph.hpp -- C++ drop-in for the reference's voxel-connectivity-graph drivers
// (reference src/edt_voxel_graph.hpp:54-236, namespace pyedt; the reference offers no `edt::`
// facade for them): same names, template parameters, argument order and ownership, but the work
// is done by edtb200_transform_voxel_graph on the GPU, or, for a volume whose doubled grid does not
// fit the device, by edtb200_transform_voxel_graph_chunked.
//
//   float* dt = pyedt::_edt3dsq_voxel_graph<uint32_t, uint8_t>(labels, graph, sx, sy, sz,
//                                                              wx, wy, wz, black_border);
//   ... delete [] dt;
//
// `workspace`, if given, receives the result and is returned; otherwise a `new float[voxels]` is
// (reference vg:109-111, 205-207).  Foreground is `labels[i] > 0` as in the reference (vg:76, 151),
// so floating-point labels are passed with EDTB200_LABELS_FLOAT and signed integer labels are
// rejected at compile time (the reference's Python layer only ever hands it unsigned, bool or
// floating-point data).  Failures throw std::runtime_error; there is no CPU fallback.
#ifndef EDT_B200_VOXEL_GRAPH_SHIM_HPP
#define EDT_B200_VOXEL_GRAPH_SHIM_HPP

#include <cstdint>
#include <stdexcept>
#include <string>
#include <type_traits>

#include "edt_b200.h"

namespace pyedt {
namespace detail_b200 {

template <typename T, typename GRAPH_TYPE>
inline float* voxel_graph_run(T* labels, GRAPH_TYPE* graph, int ndim, int64_t sx, int64_t sy, int64_t sz,
                              float wx, float wy, float wz, bool black_border, int flags, float* workspace) {
  static_assert(sizeof(GRAPH_TYPE) == 1, "the graph is one byte per voxel (only bits 0, 2 and 4 are read)");
  static_assert(sizeof(T) == 1 || sizeof(T) == 2 || sizeof(T) == 4 || sizeof(T) == 8,
                "labels must be 1, 2, 4 or 8 bytes wide");
  static_assert(std::is_floating_point<T>::value || std::is_unsigned<T>::value || std::is_same<T, bool>::value,
                "foreground is `label > 0`: pass unsigned, bool or floating-point labels");
  const int64_t voxels = sx * sy * (ndim > 2 ? sz : 1);
  float* out = workspace ? workspace : new float[voxels > 0 ? voxels : 1]();
  if (std::is_floating_point<T>::value) flags |= EDTB200_LABELS_FLOAT;
  const unsigned char* g = reinterpret_cast<const unsigned char*>(graph);
  int rc = edtb200_transform_voxel_graph(labels, (int)sizeof(T), g, ndim, sx, sy, sz, wx, wy, wz, black_border ? 1 : 0,
                                         flags, out, /*device=*/0, /*stream=*/nullptr);
  if (rc == EDTB200_ENOMEM)                      // larger than the device: stream it through in chunks
    rc = edtb200_transform_voxel_graph_chunked(labels, (int)sizeof(T), g, ndim, sx, sy, sz, wx, wy, wz,
                                               black_border ? 1 : 0, flags, out, /*device=*/0, /*device_bytes=*/0,
                                               /*chunks=*/nullptr);
  if (rc != 0) {
    if (!workspace) delete[] out;
    throw std::runtime_error(std::string("edt_b200: ") + edtb200_last_error());
  }
  return out;
}

}  // namespace detail_b200

// reference src/edt_voxel_graph.hpp:54-123
template <typename T, typename GRAPH_TYPE = uint8_t>
float* _edt2dsq_voxel_graph(T* labels, GRAPH_TYPE* graph, const int64_t sx, const int64_t sy,
                            const float wx, const float wy, const bool black_border = false,
                            float* workspace = NULL) {
  return detail_b200::voxel_graph_run(labels, graph, 2, sx, sy, 1, wx, wy, 1.0f, black_border, 0, workspace);
}

// reference src/edt_voxel_graph.hpp:125-214
template <typename T, typename GRAPH_TYPE = uint8_t>
float* _edt3dsq_voxel_graph(T* labels, GRAPH_TYPE* graph, const int64_t sx, const int64_t sy, const int64_t sz,
                            const float wx, const float wy, const float wz, const bool black_border = false,
                            float* workspace = NULL) {
  return detail_b200::voxel_graph_run(labels, graph, 3, sx, sy, sz, wx, wy, wz, black_border, 0, workspace);
}

// reference src/edt_voxel_graph.hpp:216-236
template <typename T, typename GRAPH_TYPE = uint8_t>
float* _edt3d_voxel_graph(T* labels, GRAPH_TYPE* graph, const int64_t sx, const int64_t sy, const int64_t sz,
                          const float wx, const float wy, const float wz, const bool black_border = false,
                          float* workspace = NULL) {
  return detail_b200::voxel_graph_run(labels, graph, 3, sx, sy, sz, wx, wy, wz, black_border, EDTB200_SQRT,
                                      workspace);
}

}  // namespace pyedt

#endif
