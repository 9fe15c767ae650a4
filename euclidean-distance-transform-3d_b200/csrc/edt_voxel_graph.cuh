// Voxel-connectivity-graph variant of the transform (reference: src/edt_voxel_graph.hpp:54-236,
// bound in src/edt.pyx:514-620 and 736-844).
//
// What the reference defines: the foreground (label > 0; the labels are NOT told apart here) is
// drawn on a grid of twice the resolution.  Cell (2x, 2y, 2z) is the voxel itself; the cell one
// step further along +x / +y / +z stands for the EDGE to that neighbour and is foreground only if
// the voxel's graph byte allows the move (bits 0, 2 and 4); the remaining cells of the 2x2x2
// block are plain foreground.  With a black border the last cell layer along every axis is
// background.  The binary transform of that grid with half the anisotropy, sampled at the even
// cells, is the result: a forbidden edge is a background point half a voxel away.
//
// Here: one kernel draws the doubled byte mask straight from the labels and the graph (two cells
// per 2-byte store, rows of a warp contiguous), the ordinary three passes run on it as a one-byte
// volume, and one kernel gathers the even cells (optionally through sqrt).  Everything stays on
// the device; nothing of this is on the north-star path, so the kernels are plain streaming code.
//
// The chunked call (edtb200_transform_voxel_graph_chunked) draws the mask of one slab at a time
// (the expand kernel's end_y / end_z place the volume's last slice), gathers two cells per voxel
// with the strided gather, and rebuilds each voxel's doubled line along the last axis from those
// two cells and its own graph byte (voxel_graph_lines_kernel).
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

namespace edtb200 {

template <int Bytes>
__device__ __forceinline__ bool voxel_is_foreground(const void* labels, int64_t idx, bool as_float) {
  if constexpr (Bytes == 1) return static_cast<const uint8_t*>(labels)[idx] != 0;
  if constexpr (Bytes == 2) return static_cast<const uint16_t*>(labels)[idx] != 0;
  if constexpr (Bytes == 4) {
    const uint32_t v = static_cast<const uint32_t*>(labels)[idx];
    return as_float ? (__uint_as_float(v) > 0.0f) : (v != 0);      // vg:76, 151: `labels[loc] > 0`
  }
  if constexpr (Bytes == 8) {
    const unsigned long long v = static_cast<const unsigned long long*>(labels)[idx];
    return as_float ? (__longlong_as_double((long long)v) > 0.0) : (v != 0);
  }
  return false;
}

// One thread per source voxel; writes its 2 x 2 (x 2) cells.  end_y / end_z: the index, in this
// volume, of the whole volume's last slice along y / z (sy - 1, sz - 1 unless the volume is a slab
// of a larger one; beyond the slab when the slab does not hold it).
template <int Bytes>
__global__ void __launch_bounds__(256)
voxel_graph_expand_kernel(const void* __restrict__ labels, const uint8_t* __restrict__ graph,
                          uint8_t* __restrict__ cells, int64_t sx, int64_t sy, int64_t sz, int ndim,
                          int border, int as_float, int64_t end_y, int64_t end_z) {
  const int64_t total = sx * sy * sz;
  const int64_t row2 = 2 * sx;                       // doubled row length
  const int64_t slice2 = row2 * 2 * sy;              // doubled slice size
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t x = idx % sx, y = (idx / sx) % sy, z = idx / (sx * sy);
    const bool fg = voxel_is_foreground<Bytes>(labels, idx, as_float != 0);
    const uint8_t g = graph[idx];
    const bool last_x = border && x == sx - 1, last_y = border && y == end_y,
               last_z = border && z == end_z;
    const int layers = ndim == 3 ? 2 : 1;
    for (int c = 0; c < layers; c++) {
      for (int b = 0; b < 2; b++) {
        // cell (a=0, b, c) and (a=1, b, c)
        bool even = fg, odd = fg;
        if (b == 0 && c == 0) odd = fg && (g & 0x01);        // +x edge
        if (b == 1 && c == 0) even = fg && (g & 0x04);       // +y edge
        if (b == 0 && c == 1) even = fg && (g & 0x10);       // +z edge
        if (last_x) odd = false;
        if ((b == 1 && last_y) || (c == 1 && last_z)) { even = false; odd = false; }
        const int64_t at = (2 * z + c) * slice2 + (2 * y + b) * row2 + 2 * x;
        *reinterpret_cast<uchar2*>(cells + at) = make_uchar2(even ? 1 : 0, odd ? 1 : 0);
      }
    }
  }
}

// out[x, y, z] = doubled[x * xs + y * ys + z * zs], through sqrt when asked: the even cells
// (2x, 2y, 2z) of a doubled volume with xs = 2, ys = 4 sx, zs = 8 sx sy.
__global__ void __launch_bounds__(256)
voxel_graph_gather_kernel(const float* __restrict__ doubled, float* __restrict__ out, int64_t sx, int64_t sy,
                          int64_t sz, int64_t xs, int64_t ys, int64_t zs, int take_sqrt) {
  const int64_t total = sx * sy * sz;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t x = idx % sx, y = (idx / sx) % sy, z = idx / (sx * sy);
    float v = doubled[z * zs + y * ys + x * xs];
    out[idx] = take_sqrt ? sqrtf(v) : v;
  }
}

// A box of whole lines along the last axis: n indices along it, `plane` voxels per index.  even /
// odd hold cells 2l and 2l + 1 of each voxel's doubled line after the passes along the first axes;
// they are interleaved into f, the box with its last axis doubled, and the line's mask is drawn as
// the expand kernel draws it: cell 2l is the voxel's foreground, cell 2l + 1 the edge to the next
// voxel along the last axis (graph bit `bit`: 0x10 in 3-D, 0x04 in 2-D), background on the volume's
// last slice under a black border.  The box holds whole lines, so l == n - 1 is that slice.
template <int Bytes>
__global__ void __launch_bounds__(256)
voxel_graph_lines_kernel(const void* __restrict__ labels, const uint8_t* __restrict__ graph,
                         const float* __restrict__ even, const float* __restrict__ odd, int64_t plane, int64_t n,
                         int bit, int border, int as_float, float* __restrict__ f, uint8_t* __restrict__ cells) {
  const int64_t total = plane * n;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = idx % plane, l = idx / plane;
    const bool fg = voxel_is_foreground<Bytes>(labels, idx, as_float != 0);
    const bool edge = fg && (graph[idx] & bit) && !(border && l == n - 1);
    const int64_t at = 2 * l * plane + p;
    f[at] = even[idx];
    f[at + plane] = odd[idx];
    cells[at] = fg ? 1 : 0;
    cells[at + plane] = edge ? 1 : 0;
  }
}

}  // namespace edtb200
