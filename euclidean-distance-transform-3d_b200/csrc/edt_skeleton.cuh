// edt_skeleton.cuh -- the thinning of skeletonize (edtb200_skeletonize, include/edt_b200.h).
//
// The call runs the edtsq R of the labels (run_passes) and then skeleton_thin_kernel, ONE persistent
// cooperative kernel that runs every round, cycle and step with a grid barrier between them, so nothing
// returns to the host until the skeleton is written.
//
// State.  One byte per voxel, kept in the skeleton's own buffer until the last sweep turns it into 0 / 1:
// kSkelPresent (labelled and not deleted) and kSkelAdmitted (admitted by some round).
// The candidates -- admitted voxels that are present and were not retired -- live in a compact list with
// one segment per subfield k = (x&1) | (y&1)<<1 | (z&1)<<2, so that step k reads only its own segment.
// An entry is the voxel's index on its subfield's lattice, e = ((v * hz + z/2) * hy + y/2) * hx + x/2
// with (hx, hy, hz) = the halves of (sx, sy, sz) rounded up and v the volume of the stack: 4 bytes, and
// the caller checks that one segment's capacity, count * hx * hy * hz, is below 2^32.  The list is double
// buffered: each cycle's first pass copies the surviving entries from one buffer into the other.
//
// A round (threshold theta_t = (t h)^2): one sweep over the stack admits every present, not yet admitted
// voxel with R <= theta_t, appends it to its segment, and takes the least R of the voxels it leaves out,
// which gives the next round that admits anything (the rounds between admit nothing and change nothing).
// A cycle: the first pass over the list counts each entry's present neighbours of its own label and drops
// the entries with at most one -- an end point at the start of the cycle never becomes deletable again
// (its one neighbour can only go away, and an isolated voxel is not simple), so dropping it IS the end-
// point snapshot -- and the deleted entries of the last cycle.  Then the steps k = 0 .. 2^ndim - 1 each
// delete the simple entries of segment k.  No two voxels of one subfield are 26-neighbours, so a step's
// voxels read only voxels of other subfields and write only themselves: the step is race-free and equals
// any sequential order of its deletions.  The round ends after a cycle that deletes nothing.
//
// Simplicity is computed directly (no table): the present same-label voxels of the 3x3x3 block form a
// 26-bit mask, bit j for the j-th neighbour in (dz, dy, dx) order with the centre left out, and two flood
// fills over per-bit adjacency masks (kept in shared memory) count the label's 26-components and the
// complement's 6-components in N18 that touch a 6-neighbour.  In 2-D the masks are the plane's 8 bits,
// with 8-connectivity for the label and 4-connectivity for the complement, which the same 26- and
// 6-adjacency masks give restricted to one plane.  The neighbours' labels are read at each test.
#pragma once
#include <cooperative_groups.h>

#include "edt_host.h"

namespace edtb200 {

constexpr uint8_t kSkelPresent = 1, kSkelAdmitted = 2;

// The shared control block of one call (zeroed before the kernel).  The least R is kept as the bitwise
// complement of its float bits under atomicMax, so that 0 means "none".
struct SkelControl {
  unsigned int least_r[2];          // per round parity: ~bits of the least R left out by the sweep
  unsigned int changed[3];          // per cycle mod 3: a step deleted something
  unsigned int count[2][8];         // entries per buffer and segment
  unsigned long long stats[3];      // rounds, cycles and steps run
};

struct SkelArgs {
  const float* r;                   // the edtsq of the stack
  uint8_t* state;                   // one byte per voxel: the skeleton's buffer
  uint32_t* list[2];                // two buffers of 8 segments of `cap` entries
  SkelControl* ctl;
  float* dist;                      // non-null: sqrt of r into it (r may be dist itself)
  int64_t sx, sy, sz, count, total;
  uint32_t hx, hy, hz, cap;
  int ndim;
  double h;                         // the least weight
};

// theta_t = (t h)^2 in double; t = 0 stands for the final round, which admits every voxel (R = +inf too).
__device__ __forceinline__ double skel_theta(uint64_t t, double h) {
  if (t == 0) return __longlong_as_double(0x7ff0000000000000LL);
  const double th = (double)t * h;
  return th * th;
}

// The least t >= 1 with theta_t >= R, for t below 2^53; 0 (the final round) for R = +inf or beyond.
__device__ __forceinline__ uint64_t skel_round_of(float r, double h) {
  const double R = (double)r;
  if (isinf(r)) return 0;
  const double q = sqrt(R) / h;
  const uint64_t last = ((uint64_t)1 << 53) - 1;
  if (!(q < 9007199254740990.0)) return skel_theta(last, h) >= R ? last : 0;
  uint64_t t = q < 1.0 ? 1 : (uint64_t)ceil(q);
  while (t > 1 && skel_theta(t - 1, h) >= R) --t;
  while (t < last && skel_theta(t, h) < R) ++t;
  return skel_theta(t, h) >= R ? t : 0;
}

// Warp-aggregated append of one entry to segment `seg` of list buffer `b`: one atomic per segment present
// among the lanes that call it together.
__device__ __forceinline__ void skel_append(const SkelArgs& a, int b, int seg, uint32_t e) {
  const unsigned active = __activemask();
  const unsigned group = __match_any_sync(active, seg);
  const int lane = threadIdx.x & 31, leader = __ffs(group) - 1;
  unsigned base = 0;
  if (lane == leader) base = atomicAdd(&a.ctl->count[b][seg], (unsigned)__popc(group));
  base = __shfl_sync(group, base, leader);
  a.list[b][(size_t)seg * a.cap + base + __popc(group & ((1u << lane) - 1))] = e;
}

// The bits reachable from `start` within `set` through the adjacency masks `adj`.
__device__ __forceinline__ uint32_t skel_flood(uint32_t set, uint32_t start, const uint32_t* adj) {
  uint32_t seen = start, frontier = start;
  while (frontier) {
    uint32_t next = 0;
    while (frontier) {
      next |= adj[__ffs(frontier) - 1];
      frontier &= frontier - 1;
    }
    frontier = next & set & ~seen;
    seen |= frontier;
  }
  return seen;
}

// Simple: the label's neighbours `fg` form one component, and the complement within `bg_set` has exactly
// one component (complement adjacency) that contains a bit of `seeds`.
__device__ __forceinline__ bool skel_simple(uint32_t fg, uint32_t bg_set, uint32_t seeds, const uint32_t* adj_fg,
                                            const uint32_t* adj_bg) {
  if (!fg || skel_flood(fg, fg & (0u - fg), adj_fg) != fg) return false;
  const uint32_t bg = bg_set & ~fg, s = seeds & bg;
  if (!s) return false;
  return (s & ~skel_flood(bg, s & (0u - s), adj_bg)) == 0;
}

// The mask of p's present neighbours with label m (bit j: neighbour j in (dz, dy, dx) order without the
// centre); neighbours outside p's volume are never set.  2-D: the plane only.
template <class LT>
__device__ __forceinline__ uint32_t skel_mask(const SkelArgs& a, const LT* __restrict__ labels, int64_t i,
                                              int64_t x, int64_t y, int64_t z, LT m) {
  uint32_t fg = 0;
  const int64_t plane = a.sx * a.sy;
#pragma unroll
  for (int dz = -1; dz <= 1; ++dz) {
    if (a.ndim == 2 && dz != 0) continue;
    if ((dz < 0 && z == 0) || (dz > 0 && z + 1 == a.sz)) continue;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
      if ((dy < 0 && y == 0) || (dy > 0 && y + 1 == a.sy)) continue;
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) {
        if (dx == 0 && dy == 0 && dz == 0) continue;
        if ((dx < 0 && x == 0) || (dx > 0 && x + 1 == a.sx)) continue;
        const int j = (dz + 1) * 9 + (dy + 1) * 3 + (dx + 1);
        const int64_t n = i + dx + dy * a.sx + dz * plane;
        if ((__ldcg(a.state + n) & kSkelPresent) && labels[n] == m) fg |= 1u << (j < 13 ? j : j - 1);
      }
    }
  }
  return fg;
}

// Entry e of segment k -> the voxel's flat index and coordinates within its volume.
__device__ __forceinline__ int64_t skel_voxel(const SkelArgs& a, int k, uint32_t e, int64_t& x, int64_t& y,
                                              int64_t& z) {
  uint32_t r = e / a.hx;
  x = 2 * (int64_t)(e - r * a.hx) + (k & 1);
  const uint32_t r2 = r / a.hy;
  y = 2 * (int64_t)(r - r2 * a.hy) + ((k >> 1) & 1);
  const uint32_t v = r2 / a.hz;
  z = 2 * (int64_t)(r2 - v * a.hz) + ((k >> 2) & 1);
  return x + a.sx * (y + a.sy * (z + a.sz * (int64_t)v));
}

template <int Bytes>
__global__ void __launch_bounds__(256)
skeleton_thin_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, SkelArgs a) {
  using LT = typename LabelOf<Bytes>::type;
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  __shared__ uint32_t adj26[26], adj6[26];
  // the adjacency of the 26 neighbour bits: 26-adjacent for the label, 6-adjacent for the complement
  if (threadIdx.x < 26) {
    const int j = threadIdx.x < 13 ? threadIdx.x : threadIdx.x + 1;
    const int jx = j % 3, jy = j / 3 % 3, jz = j / 9;
    uint32_t m26 = 0, m6 = 0;
    for (int b = 0; b < 26; ++b) {
      const int o = b < 13 ? b : b + 1;
      const int ex = abs(o % 3 - jx), ey = abs(o / 3 % 3 - jy), ez = abs(o / 9 - jz);
      if (o != j && ex <= 1 && ey <= 1 && ez <= 1) m26 |= 1u << b;
      if (ex + ey + ez == 1) m6 |= 1u << b;
    }
    adj26[threadIdx.x] = m26;
    adj6[threadIdx.x] = m6;
  }
  __syncthreads();
  // the complement's set and the bits of p's 6- (2-D: 4-) neighbours: N18 in 3-D, the plane's 8 in 2-D
  uint32_t bg_set = 0, seeds = 0;
  for (int b = 0; b < 26; ++b) {
    const int o = b < 13 ? b : b + 1;
    const int ex = abs(o % 3 - 1), ey = abs(o / 3 % 3 - 1), ez = abs(o / 9 - 1);
    if (a.ndim == 3 ? ex + ey + ez <= 2 : ez == 0) bg_set |= 1u << b;
    if (ex + ey + ez == 1 && (a.ndim == 3 || ez == 0)) seeds |= 1u << b;
  }
  const int nseg = a.ndim == 3 ? 8 : 4;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nthreads = (int64_t)gridDim.x * blockDim.x;
  const bool lead = tid == 0;

  // init: the present voxels, and the least R among them
  float least = __int_as_float(0x7f800000);
  bool any = false;
  for (int64_t i = tid; i < a.total; i += nthreads) {
    const bool on = labels[i] != 0;
    a.state[i] = on ? kSkelPresent : 0;
    if (on) { least = fminf(least, __ldg(a.r + i)); any = true; }
  }
  if (any) atomicMax(&a.ctl->least_r[0], ~(unsigned)__float_as_int(least));
  grid.sync();

  int cur = 0;                     // the list buffer that holds the candidates
  unsigned long long rounds = 0, cycles = 0, steps = 0;
  for (int rp = 0;; rp ^= 1) {
    const unsigned lr = __ldcg(&a.ctl->least_r[rp]);
    if (lr == 0) break;            // nothing left to admit
    const double theta = skel_theta(skel_round_of(__int_as_float((int)~lr), a.h), a.h);
    // the round's sweep: admit, and the least R of the voxels left for later rounds
    least = __int_as_float(0x7f800000);
    any = false;
    for (int64_t i = tid; i < a.total; i += nthreads) {
      const uint8_t st = __ldcg(a.state + i);
      if (st != kSkelPresent) continue;
      const float r = __ldg(a.r + i);
      if ((double)r <= theta) {
        a.state[i] = kSkelPresent | kSkelAdmitted;
        const int64_t row = i / a.sx, x = i - row * a.sx;
        const int64_t col = row / a.sy, y = row - col * a.sy;
        const int64_t v = col / a.sz, z = col - v * a.sz;
        const int k = (int)(x & 1) | (int)(y & 1) << 1 | (int)(z & 1) << 2;
        skel_append(a, cur, k, (uint32_t)(((v * a.hz + (z >> 1)) * a.hy + (y >> 1)) * a.hx + (x >> 1)));
      } else {
        least = fminf(least, r);
        any = true;
      }
    }
    if (any) atomicMax(&a.ctl->least_r[rp ^ 1], ~(unsigned)__float_as_int(least));
    grid.sync();
    ++rounds;
    if (lead) a.ctl->least_r[rp] = 0;   // read by every thread above, written again only next round
    for (;;) {
      const unsigned c3 = (unsigned)(cycles % 3);
      if (lead) {
        a.ctl->changed[(c3 + 1) % 3] = 0;
        for (int k = 0; k < 8; ++k) a.ctl->count[cur ^ 1][k] = 0;
      }
      grid.sync();
      // the cycle's first pass: keep the present entries with at least two neighbours of their label
      for (int k = 0; k < nseg; ++k) {
        const uint32_t n = __ldcg(&a.ctl->count[cur][k]);
        const uint32_t* seg = a.list[cur] + (size_t)k * a.cap;
        for (int64_t q = tid; q < n; q += nthreads) {
          const uint32_t e = __ldcg(seg + q);
          int64_t x, y, z;
          const int64_t i = skel_voxel(a, k, e, x, y, z);
          if (!(__ldcg(a.state + i) & kSkelPresent)) continue;
          if (__popc(skel_mask(a, labels, i, x, y, z, labels[i])) >= 2) skel_append(a, cur ^ 1, k, e);
        }
      }
      grid.sync();
      cur ^= 1;
      // the steps: delete the simple entries of one subfield at a time
      for (int k = 0; k < nseg; ++k) {
        const uint32_t n = __ldcg(&a.ctl->count[cur][k]);
        const uint32_t* seg = a.list[cur] + (size_t)k * a.cap;
        bool deleted = false;
        for (int64_t q = tid; q < n; q += nthreads) {
          int64_t x, y, z;
          const int64_t i = skel_voxel(a, k, __ldcg(seg + q), x, y, z);
          if (skel_simple(skel_mask(a, labels, i, x, y, z, labels[i]), bg_set, seeds, adj26, adj6)) {
            a.state[i] = kSkelAdmitted;
            deleted = true;
          }
        }
        if (deleted) a.ctl->changed[c3] = 1;
        grid.sync();
        ++steps;
      }
      ++cycles;
      if (!__ldcg(&a.ctl->changed[c3])) break;
    }
  }
  if (lead) {
    a.ctl->stats[0] = rounds;
    a.ctl->stats[1] = cycles;
    a.ctl->stats[2] = steps;
  }
  for (int64_t i = tid; i < a.total; i += nthreads) {
    a.state[i] = __ldcg(a.state + i) & kSkelPresent;
    if (a.dist) a.dist[i] = __fsqrt_rn(a.r[i]);
  }
}

}  // namespace edtb200
