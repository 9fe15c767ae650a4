// edt_geodesic.cuh -- the relaxation passes of geodesic_distance (edtb200_geodesic, include/edt_b200.h).
//
// D is the least fixed point of D[v] = min(D[v], fl64(D[u] + w(u, v))) over the same-label 26-neighbours u
// of v (2-D: 8, 1-D: 2), from 0 on the seeds and +inf elsewhere.  Rounding is monotone and every step length
// is > 0, so every relaxation order that stops only where no edge can lower a value reaches that one fixed
// point -- Dijkstra's answer in double -- and the GPU may relax in any order it likes.
//
// Tiles.  Each volume is cut into tiles of kGeoTile[ndim] voxels (3-D 8x8x8, 2-D 16x16, 1-D 256); a tile's
// index is ((v * nz + tz) * ny + ty) * nx + tx.  A round takes the tiles of a worklist.  Its CTA stages the
// tile and a one-voxel halo of values and labels in shared memory (voxels outside the volume read as label 0,
// which no edge crosses), relaxes the tile in sweeps until a sweep lowers nothing, writes back the tile's
// voxels that went down and flags the neighbour tiles (up to 26) that a lowered voxel on a face, edge or
// corner touches.  In round 1 the seeds count as lowered: the seed kernel wrote them and queued only their
// own tiles.  A flag is the round the tile is queued for, set with atomicMax: the first flagger of a
// round appends the tile to the next worklist, so a list holds every tile at most once.  The loop ends after
// a round that queues nothing.
//
// Races.  Only a tile's owner writes its voxels, so global memory needs no atomics.  A halo value may be read
// while its owner writes it in the same round: an aligned 8-byte access is not torn, and values only go down,
// so a stale read is a valid upper bound, and the owner's write queues the reader again.  Values are read
// through L2 (ld.cg): another SM's write of an earlier round must not be hidden by a stale L1 line.
//
// Phases.  geodesic_relax_kernel<B, false> relaxes D.  With indices, geodesic_relax_kernel<B, true> then runs
// the same rounds on S with D fixed: S starts at the seed's own linear index on seeds and at kGeoNone
// elsewhere, and S[v] = min(S[v], S[u]) over the TIGHT edges, D[v] == fl64(D[u] + w(u, v)) with D[v] finite
// (the same double add as the first phase).  Tight edges strictly raise D, so they form a DAG and the fixed
// point is the least seed with a tight path to v.  The phases are kept apart: carried together, a torn pair
// (new D, old smaller S) could never be undone by min.
#pragma once
#include <cooperative_groups.h>

#include "edt_host.h"

namespace edtb200 {

constexpr unsigned long long kGeoNone = ~0ull;   // S: no seed
constexpr int kGeoThreads = 256;
constexpr int kGeoHalo = 1000;                    // the largest staged block: (8 + 2)^3 voxels

// The control block of one phase (zeroed before its seed kernel).  Round r reads list[r & 1] with
// count[r % 3] entries, appends to list[(r + 1) & 1] / count[(r + 1) % 3] and clears count[(r + 2) % 3].
struct GeoControl {
  unsigned int count[3];
  unsigned long long rounds, visits;
};

struct GeoArgs {
  double* d;                        // the distances of the stack, as doubles
  unsigned long long* s;            // the seed indices (index phase), else null
  const void* seeds;                // the seed kernel's seeds, seed_bytes wide
  int seed_bytes;
  uint32_t* flag;                   // per tile: the last round it was queued for
  uint32_t* list[2];                // two worklists of one entry per tile
  GeoControl* ctl;
  int64_t sx, sy, sz, vol, total;
  int64_t nx, ny, nz, ntiles;       // tiles per axis of one volume, and of the stack
  int tx, ty, tz;                   // the tile
  int ndim;
  double step[8];                   // step[|dx| | |dy| << 1 | |dz| << 2]: the host-formed step lengths
};

// The tile holding voxel (x, y, z) of volume v.
__device__ __forceinline__ int64_t geo_tile(const GeoArgs& a, int64_t v, int64_t x, int64_t y, int64_t z) {
  return ((v * a.nz + z / a.tz) * a.ny + y / a.ty) * a.nx + x / a.tx;
}

// Queues tile t for round r (once per round) into list `b`, count slot c.
__device__ __forceinline__ void geo_queue(const GeoArgs& a, int64_t t, uint32_t r, int b, int c) {
  if (atomicMax(a.flag + t, r) < r) a.list[b][atomicAdd(&a.ctl->count[c], 1u)] = (uint32_t)t;
}

template <class T>
__device__ __forceinline__ bool geo_nonzero(const void* p, int64_t i) {
  return static_cast<const T*>(p)[i] != 0;
}

// The seed kernel of one phase: the start values (D = 0 / +inf, or S = own index / none) and the tiles
// holding a seed, queued for round 1.  A seed is a voxel whose seed and label are both non-zero.
template <int Bytes>
__global__ void __launch_bounds__(256)
geodesic_seed_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, GeoArgs a) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.total; i += (int64_t)gridDim.x * blockDim.x) {
    bool seed = labels[i] != 0;
    if (seed) {
      switch (a.seed_bytes) {
        case 1: seed = geo_nonzero<uint8_t>(a.seeds, i); break;
        case 2: seed = geo_nonzero<uint16_t>(a.seeds, i); break;
        case 4: seed = geo_nonzero<uint32_t>(a.seeds, i); break;
        default: seed = geo_nonzero<unsigned long long>(a.seeds, i); break;
      }
    }
    if (a.s)
      a.s[i] = seed ? (unsigned long long)i : kGeoNone;
    else
      a.d[i] = seed ? 0.0 : __longlong_as_double(0x7ff0000000000000LL);
    if (seed) {
      const int64_t row = i / a.sx, x = i - row * a.sx, col = row / a.sy, y = row - col * a.sy;
      const int64_t v = col / a.sz, z = col - v * a.sz;
      geo_queue(a, geo_tile(a, v, x, y, z), 1u, 1, 1);
    }
  }
}

// The rounds of one phase, in ONE cooperative launch: Index false relaxes D, true relaxes S over the tight
// edges of the fixed D.
template <int Bytes, bool Index>
__global__ void __launch_bounds__(kGeoThreads, 2)
geodesic_relax_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, GeoArgs a) {
  using LT = typename LabelOf<Bytes>::type;
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  __shared__ LT sl[kGeoHalo];
  __shared__ double sd[kGeoHalo];
  __shared__ unsigned long long ss[Index ? kGeoHalo : 1];
  __shared__ int noff[26];
  __shared__ double nw[26];
  __shared__ unsigned int dirs;

  // the staged block: the tile and a one-voxel halo along each of the first ndim axes
  const int hy = a.ndim >= 2, hz = a.ndim >= 3;
  const int HX = a.tx + 2, HY = a.ty + 2 * hy, HZ = a.tz + 2 * hz, HXY = HX * HY;
  const int tvox = a.tx * a.ty * a.tz, hvox = HXY * HZ;
  int nn = 0;
  for (int dz = -hz; dz <= hz; ++dz)
    for (int dy = -hy; dy <= hy; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        if (!dx && !dy && !dz) continue;
        if (threadIdx.x == 0) {
          noff[nn] = dz * HXY + dy * HX + dx;
          nw[nn] = a.step[(dx != 0) | (dy != 0) << 1 | (dz != 0) << 2];
        }
        ++nn;
      }
  const bool lead = blockIdx.x == 0 && threadIdx.x == 0;
  unsigned long long visits = 0;
  uint32_t r = 1;
  for (;; ++r) {
    const uint32_t n = __ldcg(&a.ctl->count[r % 3]);
    if (n == 0) break;
    visits += n;
    if (lead) a.ctl->count[(r + 2) % 3] = 0;
    for (uint32_t q = blockIdx.x; q < n; q += gridDim.x) {
      const int64_t t = __ldcg(a.list[r & 1] + q);
      int64_t rest = t / a.nx;
      const int64_t ox = (t - rest * a.nx) * a.tx;
      int64_t rest2 = rest / a.ny;
      const int64_t oy = (rest - rest2 * a.ny) * a.ty;
      const int64_t v = rest2 / a.nz, oz = (rest2 - v * a.nz) * a.tz;
      const int64_t base = v * a.vol;
      __syncthreads();                 // the previous tile's block is no longer read
      if (threadIdx.x == 0) dirs = 0;
      for (int e = threadIdx.x; e < hvox; e += kGeoThreads) {
        const int lz = e / HXY, ly = (e - lz * HXY) / HX, lx = e - lz * HXY - ly * HX;
        const int64_t x = ox + lx - 1, y = oy + ly - hy, z = oz + lz - hz;
        LT lab = 0;
        double d = __longlong_as_double(0x7ff0000000000000LL);
        unsigned long long s = kGeoNone;
        if (x >= 0 && x < a.sx && y >= 0 && y < a.sy && z >= 0 && z < a.sz) {
          const int64_t i = base + (z * a.sy + y) * a.sx + x;
          lab = labels[i];
          if (lab != 0) {
            d = __ldcg(a.d + i);
            if (Index) s = __ldcg(a.s + i);
          }
        }
        sl[e] = lab;
        sd[e] = d;
        if (Index) ss[e] = s;
      }
      __syncthreads();
      // the tile's voxels this thread owns: 2 in 3-D, 1 in 2-D and 1-D
      unsigned long long start[2];
      int own[2];
      const int mine = (tvox - (int)threadIdx.x + kGeoThreads - 1) / kGeoThreads;
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        const int k = threadIdx.x + m * kGeoThreads;
        const int lz = k / (a.tx * a.ty), ly = (k / a.tx) % a.ty, lx = k % a.tx;
        own[m] = (lz + hz) * HXY + (ly + hy) * HX + lx + 1;
        start[m] = m < mine ? (Index ? ss[own[m]] : (unsigned long long)__double_as_longlong(sd[own[m]])) : 0;
      }
      // sweeps until one lowers nothing
      for (;;) {
        bool lowered = false;
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          if (m >= mine) break;
          const int c = own[m];
          const LT lab = sl[c];
          if (lab == 0) continue;
          if (!Index) {
            const double cur = *(volatile double*)&sd[c];
            double best = cur;
            for (int j = 0; j < nn; ++j) {
              const int u = c + noff[j];
              if (sl[u] == lab) best = fmin(best, *(volatile double*)&sd[u] + nw[j]);
            }
            if (best < cur) {
              *(volatile double*)&sd[c] = best;
              lowered = true;
            }
          } else {
            const double dc = sd[c];
            if (isinf(dc)) continue;
            const unsigned long long cur = *(volatile unsigned long long*)&ss[c];
            unsigned long long best = cur;
            for (int j = 0; j < nn; ++j) {
              const int u = c + noff[j];
              if (sl[u] == lab && sd[u] + nw[j] == dc) best = min(best, *(volatile unsigned long long*)&ss[u]);
            }
            if (best < cur) {
              *(volatile unsigned long long*)&ss[c] = best;
              lowered = true;
            }
          }
        }
        if (!__syncthreads_or(lowered)) break;
      }
      // write back what went down, and the directions of the neighbour tiles it touches.  The seed kernel
      // set the seeds' values without queueing a neighbour, so in round 1 (whose tiles are exactly those
      // holding a seed) every voxel with a value counts as gone down: a seed on a face, edge or corner
      // queues the tiles beyond it, also where it is its component's only contact with them.
      const unsigned long long unset = Index ? kGeoNone : 0x7ff0000000000000ull;
      unsigned int mydirs = 0;
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        if (m >= mine) break;
        const int k = threadIdx.x + m * kGeoThreads;
        const int c = own[m];
        const unsigned long long now = Index ? ss[c] : (unsigned long long)__double_as_longlong(sd[c]);
        const bool lowered = now != start[m];
        if (!lowered && !(r == 1 && now != unset)) continue;
        const int lz = k / (a.tx * a.ty), ly = (k / a.tx) % a.ty, lx = k % a.tx;
        if (lowered) {
          const int64_t i = base + ((oz + lz) * a.sy + oy + ly) * a.sx + ox + lx;
          if (Index) a.s[i] = now;
          else a.d[i] = __longlong_as_double((long long)now);
        }
        // per axis the offsets of the tiles the voxel touches: 0, and -1 / +1 on the tile's low / high face
        const int ex = lx == 0 ? -1 : lx == a.tx - 1 ? 1 : 0;
        const int ey = !hy ? 0 : ly == 0 ? -1 : ly == a.ty - 1 ? 1 : 0;
        const int ez = !hz ? 0 : lz == 0 ? -1 : lz == a.tz - 1 ? 1 : 0;
#pragma unroll
        for (int b = 1; b < 8; ++b) {
          const int dx = b & 1 ? ex : 0, dy = b & 2 ? ey : 0, dz = b & 4 ? ez : 0;
          if ((dx || !(b & 1)) && (dy || !(b & 2)) && (dz || !(b & 4)))
            mydirs |= 1u << ((dz + 1) * 9 + (dy + 1) * 3 + dx + 1);
        }
      }
      if (mydirs) atomicOr(&dirs, mydirs);
      __syncthreads();
      const unsigned int all = dirs;
      if (threadIdx.x < 27 && (all >> threadIdx.x & 1u)) {
        const int dx = threadIdx.x % 3 - 1, dy = threadIdx.x / 3 % 3 - 1, dz = threadIdx.x / 9 - 1;
        const int64_t cx = ox / a.tx + dx, cy = oy / a.ty + dy, cz = oz / a.tz + dz;
        if (cx >= 0 && cx < a.nx && cy >= 0 && cy < a.ny && cz >= 0 && cz < a.nz)
          geo_queue(a, ((v * a.nz + cz) * a.ny + cy) * a.nx + cx, r + 1, (r + 1) & 1, (r + 1) % 3);
      }
    }
    grid.sync();
  }
  if (lead) {
    a.ctl->rounds = r - 1;
    a.ctl->visits = visits;
  }
}

// float32(D), and with planes the seed's coordinates within its volume (-1 where there is none).
__global__ void __launch_bounds__(256)
geodesic_store_kernel(GeoArgs a, float* __restrict__ dist, int32_t* px, int32_t* py, int32_t* pz) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.total; i += (int64_t)gridDim.x * blockDim.x) {
    dist[i] = (float)a.d[i];
    if (!px) continue;
    const unsigned long long s = a.s[i];
    int32_t x = -1, y = -1, z = -1;
    if (s != kGeoNone) {
      const int64_t local = (int64_t)s - (i / a.vol) * a.vol;
      const int64_t row = local / a.sx, col = row / a.sy;
      x = (int32_t)(local - row * a.sx);
      y = (int32_t)(row - col * a.sy);
      z = (int32_t)col;
    }
    px[i] = x;
    if (py) py[i] = y;
    if (pz) pz[i] = z;
  }
}

}  // namespace edtb200
