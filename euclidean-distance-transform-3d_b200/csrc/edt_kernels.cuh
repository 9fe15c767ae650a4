// edt_kernels.cuh -- sm_90a (H100) kernels of the multi-label squared EDT.
//
// What is computed (bit-for-bit the reference's result, see DESIGN.md "Arithmetic"):
//
//   first axis  (reference squared_edt_1d_multi_seg, src/edt.hpp:70-119)
//       out[p] = T[min(kL, kR)],  kL/kR = steps to the nearest voxel of a different label
//       (or the volume face when black_border) on either side, T[k] = fl32(a_k * a_k),
//       a_k = a_{k-1} (+) w in float32 (the reference's sequential adds), +inf if no such
//       voxel, 0 for background.
//   later axes  (reference squared_edt_1d_parabolic_multi_seg + squared_edt_1d_parabolic,
//       src/edt.hpp:168-377) for a voxel i inside a run [a,b) of equal labels:
//       out[i] = min( min_{v in [a,b)} fl32(w2*(i-v)^2 + f[v]),
//                     fl32(w2*(i-a+1)^2) if the run has a low border,
//                     fl32(w2*(b-i)^2)   if the run has a high border )
//       with w2 = fl32(w*w).  The reference finds the same minimum with a lower-envelope
//       scan; only the minimum VALUE matters (SURVEY.md section 8a-4), so the kernels are
//       free to search it any way they like.
//
// No tensor cores: there is no contraction here, the passes are HBM-bound streaming
// kernels over the label volume and one float32 volume that is transformed in place.
#pragma once
#include <cuda.h>          // CUtensorMap (type only; the encoder is fetched at run time)
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

namespace edtb200 {

// kSqrt / kNegate act in a pass's store; kZeroLabel makes the first-axis pass treat
// background (label 0) as an ordinary label instead of forcing its distance to 0.
enum : int { kSqrt = 1, kNegate = 2, kZeroLabel = 4 };

constexpr int kNoBoundary = 0x3fffffff;

// Site codes of the site-tracking passes (Sites = true), one int per voxel and pass:
//   X pass      the site's x coordinate, -1 or sx for a volume face;
//   Y / Z pass  the row of the hull vertex that won (>= 0), or a DIRECT site: the row a - 1 or b
//               just outside the run, whose border term won (the site itself, not a sample of it),
//               stored as site_direct(row) <= -1;
//   any pass    kSiteNone where the distance is +inf.
constexpr int kSiteNone = INT32_MIN;
__host__ __device__ __forceinline__ int site_direct(int row) { return -2 - row; }
__host__ __device__ __forceinline__ int site_direct_row(int code) { return -2 - code; }

template <int Bytes> struct LabelOf;
template <> struct LabelOf<1> { using type = uint8_t;  using wide = uint32_t; };
template <> struct LabelOf<2> { using type = uint16_t; using wide = uint32_t; };
template <> struct LabelOf<4> { using type = uint32_t; using wide = uint32_t; };
template <> struct LabelOf<8> { using type = uint64_t; using wide = unsigned long long; };

// Programmatic dependent launch (PDL): a kernel lets the next kernel of the stream start filling
// the SM slots that free up during its last wave; the dependent kernel does whatever does not
// touch the distance volume (staging the labels) and then waits for the whole grid before it.
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait_for_previous_grid() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}

__device__ __forceinline__ float finish_value(float v, bool background, int flags) {
  if (flags & kSqrt) v = __fsqrt_rn(v);                 // np.sqrt / std::sqrt: IEEE-correct
  if ((flags & kNegate) && background) v = -v;          // sdf: f(data) - f(data==0)
  return v;
}

// Statistic of the first-axis pass for the host's NEXT launch decisions: how many runs of equal
// labels the volume has along x.  Every warp adds its count to `counter`; the last CTA of the grid
// moves the total (and the voxel count) to `publish` -- page-locked host memory mapped into the
// device -- and resets the counters, so nothing has to be zeroed between transforms and the host
// never synchronises to read it (it looks at the value the previous transform left there).
struct RunStat {
  unsigned long long* counter;     // device
  unsigned int* ticket;            // device
  unsigned long long* publish;     // mapped host memory: [0] run starts, [1] voxels
  unsigned long long voxels;
};

__device__ __forceinline__ void publish_run_stat(const RunStat st, unsigned int warp_total, int lane) {
  if (!st.counter) return;
  if (lane == 0 && warp_total) atomicAdd(st.counter, (unsigned long long)warp_total);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    if (atomicAdd(st.ticket, 1u) == gridDim.x - 1u) {
      const unsigned long long total = atomicExch(st.counter, 0ull);
      *st.ticket = 0u;
      st.publish[0] = total;
      st.publish[1] = st.voxels;
      __threadfence_system();
    }
  }
}

// T[k] for k = 0..count-1 (see header).  One thread: the adds are sequential by definition
// (src/edt.hpp:92-118 accumulates d[i] = d[i-1] + w in float32).
static __global__ void step_table_kernel(float w, int count, float* __restrict__ table) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  float a = 0.0f;
  table[0] = 0.0f;
  for (int k = 1; k < count; ++k) {
    a = __fadd_rn(a, w);
    table[k] = __fmul_rn(a, a);
  }
}

// ---------------------------------------------------------------------------------------
// First-axis pass.  One warp per line of `sx` contiguous voxels.
//   sweep 1: 32 labels per step, one per lane (coalesced), neighbour label by shuffle,
//            __ballot -> one 32-bit word of "label changes here" bits B[0..sx] and one of
//            "is background" bits, kept in shared memory (sx/8 bytes per line);
//   sweep 2: per word, the nearest set bit below / above it (warp scan over the words);
//   sweep 3: per voxel, nearest boundary on each side with clz/ffs on its own word, then
//            the table lookup and a coalesced float store.
// B[j] (1 <= j < sx) says labels j-1 and j differ; B[0] and B[sx] are the volume faces.
// Sites: also write each voxel's site code (see kSiteNone) to `codes`, laid out like `out`.
// ---------------------------------------------------------------------------------------
template <int Bytes, bool Sites = false>
__global__ void __launch_bounds__(256)
first_axis_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels,
                  float* __restrict__ out, int64_t nlines, int sx,
                  const float* __restrict__ table, int border, int flags, RunStat stat,
                  int* __restrict__ codes) {
  using LT = typename LabelOf<Bytes>::type;
  using WT = typename LabelOf<Bytes>::wide;
  extern __shared__ uint32_t smem_u32[];

  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int warps = blockDim.x >> 5;
  const int nchunks = (sx + 31) >> 5;
  const int nwords = (sx >> 5) + 1;

  uint32_t* bnd = smem_u32 + (size_t)warp * (4 * (size_t)nwords);
  uint32_t* bkg = bnd + nwords;
  int* below = reinterpret_cast<int*>(bkg + nwords);   // nearest set bit in words < c
  int* above = below + nwords;                          // nearest set bit in words > c

  unsigned int nstarts = 0;                            // label changes seen by this warp (lane 0 counts)
  for (int64_t line = (int64_t)blockIdx.x * warps + warp; line < nlines;
       line += (int64_t)gridDim.x * warps) {
    const LT* __restrict__ src = labels + line * sx;
    float* __restrict__ dst = out + line * sx;

    // ---- sweep 1: boundary / background bit words ----
    WT carry = 0;
    for (int c0 = 0; c0 < nchunks; c0 += 4) {
      WT v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int p = ((c0 + u) << 5) + lane;
        v[u] = (p < sx) ? (WT)src[p] : (WT)0;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int c = c0 + u;
        if (c < nchunks) {                       // warp-uniform
          const int p = (c << 5) + lane;
          WT up = __shfl_up_sync(full, v[u], 1);
          if (lane == 0) up = carry;
          carry = __shfl_sync(full, v[u], 31);
          bool edge;
          if (p == 0) edge = border != 0;
          else if (p < sx) edge = (v[u] != up);
          else edge = (p == sx) && (border != 0);
          const uint32_t wb = __ballot_sync(full, edge);
          const uint32_t wz = __ballot_sync(full, (p < sx) && (v[u] == 0));
          if (lane == 0) { bnd[c] = wb; bkg[c] = wz; nstarts += __popc(wb); }
        }
      }
    }
    if ((sx & 31) == 0 && lane == 0) { bnd[nchunks] = border ? 1u : 0u; bkg[nchunks] = 0u; }
    __syncwarp();

    // ---- sweep 2: nearest set bit strictly below / above each word ----
    {
      int run = -1;
      for (int base = 0; base < nwords; base += 32) {
        const int c = base + lane;
        const uint32_t w = (c < nwords) ? bnd[c] : 0u;
        int hi = w ? ((c << 5) + 31 - __clz(w)) : -1;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
          const int o = __shfl_up_sync(full, hi, s);
          if (lane >= s) hi = max(hi, o);
        }
        int excl = __shfl_up_sync(full, hi, 1);
        if (lane == 0) excl = -1;
        excl = max(excl, run);
        if (c < nwords) below[c] = excl;
        run = max(run, __shfl_sync(full, hi, 31));
      }
      int nxt = kNoBoundary;
      for (int base = ((nwords - 1) >> 5) << 5; base >= 0; base -= 32) {
        const int c = base + lane;
        const uint32_t w = (c < nwords) ? bnd[c] : 0u;
        int lo = w ? ((c << 5) + __ffs(w) - 1) : kNoBoundary;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
          const int o = __shfl_down_sync(full, lo, s);
          if (lane + s < 32) lo = min(lo, o);
        }
        int excl = __shfl_down_sync(full, lo, 1);
        if (lane == 31) excl = kNoBoundary;
        excl = min(excl, nxt);
        if (c < nwords) above[c] = excl;
        nxt = min(nxt, __shfl_sync(full, lo, 0));
      }
    }
    __syncwarp();

    // ---- sweep 3: distances ----
    for (int c = 0; c < nchunks; ++c) {
      const int p = (c << 5) + lane;
      const uint32_t w = bnd[c];
      const uint32_t mle = w & (0xffffffffu >> (31 - lane));
      const uint32_t mgt = (lane == 31) ? 0u : (w & (0xfffffffeu << lane));
      const int jl = mle ? ((c << 5) + 31 - __clz(mle)) : below[c];
      const int jr = mgt ? ((c << 5) + __ffs(mgt) - 1) : above[c];
      const int kl = (jl >= 0) ? (p - jl + 1) : kNoBoundary;
      const int kr = (jr != kNoBoundary) ? (jr - p) : kNoBoundary;
      const int k = min(kl, kr);
      if (p < sx) {
        const bool background = (bkg[c] >> lane) & 1u;
        float val = (k >= kNoBoundary) ? __int_as_float(0x7f800000) : __ldg(table + k);
        if (background && !(flags & kZeroLabel)) val = 0.0f;
        dst[p] = finish_value(val, background, flags);
        // the site at jl - 1 (boundary bit jl is the step from it into this run) or jr; the lower
        // one on a tie
        if constexpr (Sites) codes[line * sx + p] = (k >= kNoBoundary) ? kSiteNone : (kl <= kr ? jl - 1 : jr);
      }
    }
    __syncwarp();
  }
  publish_run_stat(stat, nstarts, lane);
}

// ---------------------------------------------------------------------------------------
// First-axis pass, register-resident variant for lines of sx <= 128*K voxels with sx % 4 == 0
// (rows then start on 16-byte boundaries for the float4 stores and on 4*Bytes boundaries for
// the vector label loads).  One warp per line; a lane owns 4 consecutive voxels of each
// 128-voxel block, so every global access is a full-width vector (4*Bytes per lane in,
// 16 bytes per lane out).  Boundaries are found in registers: per lane a 4-bit mask per
// block, then a warp max-scan (nearest boundary at or below) and a warp min-scan (nearest
// boundary above) with carries across the K blocks.  The step table lives in shared memory.
// ---------------------------------------------------------------------------------------
template <int Bytes> struct Vec4Labels;
template <> struct Vec4Labels<1> {
  static __device__ __forceinline__ void load(const uint8_t* p, uint32_t v[4]) {
    const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(p));
    v[0] = w & 0xffu; v[1] = (w >> 8) & 0xffu; v[2] = (w >> 16) & 0xffu; v[3] = w >> 24;
  }
};
template <> struct Vec4Labels<2> {
  static __device__ __forceinline__ void load(const uint16_t* p, uint32_t v[4]) {
    const uint2 w = __ldg(reinterpret_cast<const uint2*>(p));
    v[0] = w.x & 0xffffu; v[1] = w.x >> 16; v[2] = w.y & 0xffffu; v[3] = w.y >> 16;
  }
};
template <> struct Vec4Labels<4> {
  static __device__ __forceinline__ void load(const uint32_t* p, uint32_t v[4]) {
    const uint4 w = __ldg(reinterpret_cast<const uint4*>(p));
    v[0] = w.x; v[1] = w.y; v[2] = w.z; v[3] = w.w;
  }
};
template <> struct Vec4Labels<8> {
  static __device__ __forceinline__ void load(const uint64_t* p, unsigned long long v[4]) {
    const ulonglong2 a = __ldg(reinterpret_cast<const ulonglong2*>(p));
    const ulonglong2 b = __ldg(reinterpret_cast<const ulonglong2*>(p) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
};

// Run-start bit planes that the X pass writes for the later passes, so that these read one bit
// per voxel instead of a label (used on label noise, see run_passes).  One bit per voxel, x fastest,
// every row (y, z) padded to wpr = ceil(sx / 32) whole words, row (y, z) at word (z * sy + y) * wpr:
//   y   bit = y == 0 || L(x, y, z) != L(x, y - 1, z)     (the Y pass's run starts)
//   z   bit = z == 0 || L(x, y, z) != L(x, y, z - 1)     (the Z pass's run starts; 3-D only, else null)
// In a stack of volumes laid end to end along z, z counts within the voxel's own volume: every
// depth-th slice starts a volume, and its z bits are all set.
// Beside them the settled planes, one word per row (y, z) at word z * sy + y: bit s set when every
// voxel of the row's 32-voxel x-segment s ends the X pass at f <= t (padding voxels past sx count as
// settled).  A later pass with w2 = t leaves such a voxel as it is (DESIGN.md section 4.1), so it may
// skip a tile whose bits are all set.
//   settled_y   t = ty, the Y pass's w2        settled_z   t = tz, the Z pass's (3-D only, else null)
struct XPlanes {
  uint32_t* y;
  uint32_t* z;
  int64_t sy;              // rows per z
  int64_t depth;           // slices per volume (z planes only)
  uint32_t* settled_y;
  uint32_t* settled_z;
  float ty, tz;
};

// Bit i of the low byte of x -> bit 4 i.
__device__ __forceinline__ uint32_t spread_nibble_bits(uint32_t x) {
  x &= 0xffu;
  x = (x | (x << 12)) & 0x000f000fu;
  x = (x | (x << 6)) & 0x03030303u;
  return (x | (x << 3)) & 0x11111111u;
}

// The run-start words of one row of at most 512 voxels, in natural x order, from every lane's nibbles
// (bits 4 b .. 4 b + 3 of the y plane, 16 + 4 b .. of the z plane: its voxels 128 b + 4 lane .. + 3 of
// block b): lane c = 4 b + w gets word c, which holds nibble b of lanes 8 w .. 8 w + 7.  One shuffle
// per source lane serves both planes.
__device__ __forceinline__ void gather_plane_words(uint32_t nibs, int lane, uint32_t& word_y, uint32_t& word_z) {
  const int src = (lane & 3) << 3, sh = lane & 12;   // sh = 4 b for lanes 0 .. 15 (the rest store nothing)
  word_y = word_z = 0u;
#pragma unroll
  for (int l = 0; l < 8; ++l) {
    const uint32_t g = __shfl_sync(0xffffffffu, nibs, src + l) >> sh;
    const uint32_t at = 15u << (4 * l);
    word_y |= (g << (4 * l)) & at;
    word_z |= (l < 4 ? g >> (16 - 4 * l) : g << (4 * l - 16)) & at;
  }
}

// The lane's labels of one row for the register-resident X kernels: v[b] = voxels 128 b + 4 lane .. + 3
// of block b, which load(q0, v[b]) fetches from q0; zeros past sx.
template <int Bytes, int K, class Load>
__device__ __forceinline__ void load_vec_row(Load load, int sx, int lane, typename LabelOf<Bytes>::wide v[K][4]) {
#pragma unroll
  for (int b = 0; b < K; ++b) {
    const int q0 = (b << 7) + (lane << 2);
    if (q0 < sx) load(q0, v[b]);
    else { v[b][0] = v[b][1] = v[b][2] = v[b][3] = 0; }
  }
}

// One row of the register-resident X kernels, from the lane's labels v (load_vec_row) to its
// distances at dst: run-start / background masks, nearest boundaries, table lookups from table_s
// (T[0..sx], +inf at sx + 1) and float4 stores.  Adds the row's label changes along x to the lane's nstarts.
// Plain = true: squared EDT, background forced to 0, no sqrt / sign (the hot configuration);
// Plain = false: behaviour selected by `flags` at run time.
// Settled = true (first_axis_planes_kernel only): also clears bit b of set_y / set_z where a value
// stored for the lane's four voxels of block b exceeds ty / tz (lanes past sx leave theirs set).
// OneRowY = true (first_axis_planes_kernel only): stores min(f, ty) for the voxels marked in one_row
// (4 bits per block, like the masks below), before the settled compare: the voxels whose y-run is
// one row long, which the Y pass would bring to exactly that value (DESIGN.md section 4.1).
template <int Bytes, int K, bool Plain, bool Settled = false, bool OneRowY = false>
__device__ __forceinline__ void first_axis_vec_row(const typename LabelOf<Bytes>::wide v[K][4], float* __restrict__ dst,
                                                   int sx, const float* table_s, int border, int flags,
                                                   bool keep_background, int lane, unsigned lt_mask, unsigned gt_mask,
                                                   unsigned int& nstarts, float ty = 0.0f, float tz = 0.0f,
                                                   uint32_t* set_y = nullptr, uint32_t* set_z = nullptr,
                                                   uint32_t one_row = 0u) {
  using WT = typename LabelOf<Bytes>::wide;
  const unsigned full = 0xffffffffu;

  // ---- labels -> per-block 4-bit "label changes here" / "is background" masks ----
  uint32_t edges = 0, zeros = 0;                   // 4 bits per block
  uint32_t occ[K];                                 // lanes owning at least one boundary
#pragma unroll
  for (int b = 0; b < K; ++b) {
    const int q0 = (b << 7) + (lane << 2);
    WT up = __shfl_up_sync(full, v[b][3], 1);
    if (b > 0) {                                   // compile-time: warp-uniform
      const WT tail = __shfl_sync(full, v[b > 0 ? b - 1 : 0][3], 31);
      if (lane == 0) up = tail;
    }
    uint32_t m = 0, z = 0;
    if (q0 < sx) {
      if ((q0 == 0) ? (border != 0) : (v[b][0] != up)) m |= 1u;
      if (v[b][1] != v[b][0]) m |= 2u;
      if (v[b][2] != v[b][1]) m |= 4u;
      if (v[b][3] != v[b][2]) m |= 8u;
      if (v[b][0] == 0) z |= 1u;
      if (v[b][1] == 0) z |= 2u;
      if (v[b][2] == 0) z |= 4u;
      if (v[b][3] == 0) z |= 8u;
    }
    occ[b] = __ballot_sync(full, m != 0);
    edges |= m << (4 * b);
    zeros |= z << (4 * b);
  }
  nstarts += __popc(edges);

  // ---- nearest boundary strictly below / above the lane's 4 voxels, per block ----
  // The ballots give the boundary-owning lanes; one shuffle fetches that lane's masks.
  int kl_in[K], kr_in[K];          // kL of the voxel just below q0, kR seed for q0 + 3
  {
    uint32_t prev_occ = 0; int prev_b = 0;
#pragma unroll
    for (int b = 0; b < K; ++b) {
      const int q0 = (b << 7) + (lane << 2);
      const uint32_t mine = occ[b] & lt_mask;
      const uint32_t pick = mine ? mine : prev_occ;
      const int pb = mine ? b : prev_b;
      const int sl = 31 - __clz(pick | 1u);
      const uint32_t nib = (__shfl_sync(full, edges, sl) >> (4 * pb)) & 15u;
      const int pos = (pb << 7) + (sl << 2) + 31 - __clz(nib | 1u);
      kl_in[b] = pick ? (q0 - pos) : kNoBoundary;          // = kL(q0 - 1) + ... see below
      if (occ[b]) { prev_occ = occ[b]; prev_b = b; }
    }
    uint32_t next_occ = 0; int next_b = 0;
#pragma unroll
    for (int b = K - 1; b >= 0; --b) {
      const int q0 = (b << 7) + (lane << 2);
      const uint32_t mine = occ[b] & gt_mask;
      const uint32_t pick = mine ? mine : next_occ;
      const int pb = mine ? b : next_b;
      const int sl = __ffs(pick | 0x80000000u) - 1;
      const uint32_t nib = (__shfl_sync(full, edges, sl) >> (4 * pb)) & 15u;
      const int pos = (pb << 7) + (sl << 2) + __ffs(nib | 8u) - 1;
      const int far = border ? (sx - (q0 + 3)) : kNoBoundary;
      kr_in[b] = pick ? (pos - (q0 + 3)) : far;
      if (occ[b]) { next_occ = occ[b]; next_b = b; }
    }
  }

  // ---- distances (chains over the 4 voxels), table lookup, vector store ----
#pragma unroll
  for (int b = 0; b < K; ++b) {
    const int q0 = (b << 7) + (lane << 2);
    if (q0 >= sx) continue;
    const uint32_t m = (edges >> (4 * b)) & 15u;
    const uint32_t z = (zeros >> (4 * b)) & 15u;
    // kL(q) = q - (nearest boundary position <= q) + 1:  1 at a boundary, else previous + 1
    int kl[4], kr[4];
    int run = kl_in[b];                    // q0 - pos: kL the voxel q0 would have without its own bit
#pragma unroll
    for (int e = 0; e < 4; ++e) { run = ((m >> e) & 1u) ? 1 : run + 1; kl[e] = run; }
    // kR(q) = (nearest boundary position > q) - q:  1 if q + 1 is a boundary, else next + 1
    run = kr_in[b];
    kr[3] = run;
#pragma unroll
    for (int e = 2; e >= 0; --e) { run = ((m >> (e + 1)) & 1u) ? 1 : run + 1; kr[e] = run; }
    float r[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      int k = min(min(kl[e], kr[e]), sx + 1);          // sx + 1 -> +inf (no boundary at all)
      const bool background = (z >> e) & 1u;
      if (background && !keep_background) k = 0;        // T[0] = 0
      float val = table_s[k];
      if (!Plain) val = finish_value(val, background, flags);
      r[e] = val;
    }
    if constexpr (OneRowY) {
      const uint32_t s = (one_row >> (4 * b)) & 15u;
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if ((s >> e) & 1u) r[e] = fminf(r[e], ty);
    }
    if constexpr (Settled) {                          // one compare per block and plane
      const float most = fmaxf(fmaxf(r[0], r[1]), fmaxf(r[2], r[3]));
      if (!(most <= ty)) *set_y &= ~(1u << b);
      if (!(most <= tz)) *set_z &= ~(1u << b);
    }
    *reinterpret_cast<float4*>(dst + q0) = make_float4(r[0], r[1], r[2], r[3]);
  }
}

template <int Bytes, int K, bool Plain>
// Registers capped for occupancy: uncapped the kernel takes 64 (rows <= 512: 4 CTAs per SM) / 99 registers
// (1024-voxel rows: 2 CTAs); at 48 / 80 it still has no spills and runs 5 / 3 CTAs per SM, which
// hides more of the label-load latency (6 CTAs would need 40 registers, and there it spills).
__global__ void __launch_bounds__(256, K >= 8 ? 3 : 5)
first_axis_vec_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels,
                      float* __restrict__ out, int64_t nlines, int sx,
                      const float* __restrict__ table, int border, int flags, RunStat stat) {
  using LT = typename LabelOf<Bytes>::type;
  using WT = typename LabelOf<Bytes>::wide;
  extern __shared__ float table_s[];                 // T[0..sx], then +inf at sx + 1
  pdl_launch_dependents();                           // the second-axis pass may start staging labels
  for (int i = threadIdx.x; i <= sx; i += blockDim.x) table_s[i] = __ldg(table + i);
  if (threadIdx.x == 0) table_s[sx + 1] = __int_as_float(0x7f800000);
  __syncthreads();

  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int warps = blockDim.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  const unsigned gt_mask = (lane == 31) ? 0u : (0xfffffffeu << lane);
  const bool keep_background = Plain ? false : (flags & kZeroLabel) != 0;
  unsigned int nstarts = 0;                          // label changes along x seen by this lane

  const int64_t step = (int64_t)gridDim.x * warps;
  for (int64_t line = (int64_t)blockIdx.x * warps + warp; line < nlines; line += step) {
    const LT* __restrict__ src = labels + line * sx;
    float* __restrict__ dst = out + line * sx;
    WT v[K][4];
    load_vec_row<Bytes, K>([&](int q0, WT* r) { Vec4Labels<Bytes>::load(src + q0, r); }, sx, lane, v);
    first_axis_vec_row<Bytes, K, Plain>(v, dst, sx, table_s, border, flags, keep_background, lane, lt_mask, gt_mask,
                                        nstarts);
  }
  if (stat.counter) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) nstarts += __shfl_xor_sync(full, nstarts, s);
  }
  publish_run_stat(stat, nstarts, lane);
}

// ---------------------------------------------------------------------------------------
// Later-axis pass (Y: line stride sx, Z: line stride sx*sy), in place on f.
//
// A CTA owns a tile of TX adjacent lines (TX = 32, 16 or 8 consecutive x: 128/64/32 B per
// row, so every global access is made of whole 32-byte sectors) times the whole line length
// n, staged in shared memory:
//     fs[n][TX] float32   the distance tile, fetched by the TMA unit (cp.async.bulk.tensor over
//                         a 3-D tensor map of the volume; ragged tiles are zero-filled by the
//                         hardware) while the threads work on the labels;
//     startw[n/32][TX]    one 32-bit "a run of equal labels starts here" word per 32 rows;
//     hullw[n/32][TX]     lower-envelope membership bits (the scan's vertex stack, 1 bit/voxel);
//     sq[n+2]             w2*e^2, the closed-form border terms.
// Thread (x = lane % TX, chunk = 32 consecutive rows) turns its label column into a run-start
// word, then produces the outputs of the runs that START in its chunk:
//   * runs of length one (the common case in dense segmentations, the only case for iid
//     labels): out = min(f, w2) -- a predicated straight-line loop over the 32 rows;
//   * every other run: Felzenszwalb-Huttenlocher lower envelope over the run, restated for
//     one thread per run: vertices with f = +inf are not sites; a vertex is dropped when
//     its intersection with the newcomer lies at or left of its intersection with the
//     vertex below it (compared by cross-multiplication in double, no division); the
//     read-out walks the hull and evaluates each candidate with one fused multiply-add,
//     which is the correctly rounded w2*d^2 + f[v] the reference computes in double and
//     rounds once (src/edt.hpp:225-230); run borders enter as sq[] terms.
// ---------------------------------------------------------------------------------------
struct LineGeom {
  int64_t outer_count;     // Y pass: sz            Z pass: 1
  int64_t outer_stride;    // Y pass: sx*sy         Z pass: 0
  int64_t inner_count;     // Y pass: sx            Z pass: sx*sy   (adjacent lines)
  int64_t line_stride;     // Y pass: sx            Z pass: sx*sy
  int n;                   // line length
  int tiles_per_outer;     // ceil(inner_count / TX)
};

struct TileBoxes {
  int box_rows;   // rows per TMA box (<= 256)
  int nboxes;     // boxes per tile; box_rows * nboxes >= n
};

// The run-start plane of one later-axis pass written by the X pass (XPlanes): for the line (outer o,
// inner j) and row i the bit (j % sx) & 31 of word  o * outer_words + (j / sx) * wpr + (j % sx) / 32
// + i * row_words.  Y pass: outer = z, inner = x; Z pass: inner = y * sx + x.
// The grouped kernel (skips_settled) reads `settled`, the pass's settled plane (XPlanes), and skips
// every tile whose voxels all have f <= w2: for the line (o, j) and row i the bit (j % sx) / 32 of word
// o * settled_outer + j / sx + i * settled_row.  With `refresh` (the Y pass: the Z pass's settled
// plane, same layout) every tile that it runs sets the bits of its rows that it leaves at
// f <= refresh_t.  `group` (1 to 32): consecutive tiles per CTA of the grouped kernel.
struct RunBits {
  const uint32_t* start;   // a run of equal labels starts at this row (always at row 0)
  int64_t row_words;
  int64_t outer_words;
  int64_t sx;
  int64_t wpr;
  const uint32_t* settled;
  int64_t settled_row;
  int64_t settled_outer;
  uint32_t* refresh;
  float refresh_t;
  int group;               // (in the tail padding: the struct keeps its size and layout)
};

// Whether the tile kernel instance <Bits, IntHull, Epilogue> is the grouped one that skips settled
// tiles and refreshes the Z pass's settled plane: only there does a skipped tile provably equal what
// the pass would store -- integer samples (with float hull tests the read-out may return a candidate
// within rounding of the minimum, DESIGN.md section 8) and no epilogue, whose sqrt / sign rewrites
// every row.  The host arms the skip by the same rule (plan_noise).
constexpr __host__ __device__ bool skips_settled(bool bits, bool int_hull, bool epilogue) {
  return bits && int_hull && !epilogue;
}

__device__ __forceinline__ uint32_t smem_addr(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, unsigned parity) {
  unsigned ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_addr(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a tile load that never completes (bad tensor map) traps instead of hanging.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
  for (unsigned spin = 0; spin < (1u << 26); ++spin)
    if (mbar_try_wait(bar, parity)) return;
  __trap();
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(smem_addr(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2),
        "r"(smem_addr(bar))
      : "memory");
}

// ---- shared-memory accessors on 32-bit shared-window addresses ----
// (explicit ld/st.shared: pointer arithmetic on generic pointers made the compiler rebuild the
// shared-window base inside every loop iteration)
// Plain loads are NOT volatile so that the compiler may schedule them freely; they are used only
// for data that is immutable once the tile is staged, and every address they use is derived from
// a token produced after the staging barrier (see `smem_token`), which keeps them below it.
__device__ __forceinline__ float lds_f32(uint32_t addr) {
  float v;
  asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
// Volatile load for words that are rewritten while the kernel runs (the hull bits).
__device__ __forceinline__ uint32_t lds_u32_volatile(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void red_shared_or(uint32_t addr, uint32_t bits) {
  asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(addr), "r"(bits) : "memory");
}
// Zero that the compiler cannot see through, produced at this point of the program order.
__device__ __forceinline__ uint32_t smem_token() {
  uint32_t t;
  asm volatile("mov.u32 %0, 0;" : "=r"(t) : : "memory");
  return t;
}
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void sts_u8(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u8 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t lds_u8_volatile(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void sts_f32(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}

// ---------------------------------------------------------------------------------------
// First-axis pass that also writes the run-start planes (XPlanes), for rows of sx <= 128*K
// voxels on which first_axis_vec_kernel runs, labels of 4 or 8 bytes.
//
// The warps march along y.  In 3-D a CTA of W warps owns a band of W consecutive slices z0 .. z0+W-1
// (warp w: slice z0 + w) and a chunk of rows ya .. yb.  A *stage* is one row y of every slice of the
// band plus the halo row (y, z0 - 1): W + 1 rows of sx labels, one 1-D bulk copy each, completed on
// the stage's mbarrier.  The z plane compares warp w's row with the stage's row of slice z0 + w - 1
// (the halo for warp 0); a slice that starts a volume (vz = 0, also inside a band of a stack) has all
// its z bits set, and a band that starts a volume loads no halo.  In 2-D the W warps take W
// independent (image, y-chunk) sequences, and there is no halo.
// Row y + 1 is the same warp's row in the next stage, so a stage is processed once it and its
// successor have landed; the compare of row y - 1 with row y is the previous row's compare with its
// successor, kept in a register.  Each chunk also stages the rows ya - 1 and yb + 1 (where they
// exist), which are only compared with.  So every row sees rows y - 1 and y + 1, and a voxel whose
// y-run is one row long (its label differs from rows y - 1 and y + 1, or the line ends there) gets
// min(f, w2) here: that is exactly what the Y pass would leave, its own sample and the border term
// w2 * 1^2 of the label change or line end next to it, which a line of sy >= 2 rows always has on one
// side -- also at rows 0 and sy - 1 without black_border.  Such voxels end the X pass settled for the
// Y pass (ty = w2).  Lines of one row have no border term and never take it.
// The stages pass through a ring of S slots, issued S ahead: two are read while the other S - 2 load.
// The (band, chunk) items are numbered band fastest and dealt out round robin over one persistent
// wave, so the CTAs of neighbouring bands and the same chunk start together and march at one rate:
// a halo row is staged by the band below at about the same time, and is expected to come from L2.
//
// Shared memory: S mbarriers (64 bytes), the ring of S stages of (W+1)*sx labels, the step table.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void bulk_load(void* dst, const void* src, unsigned bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar))
               : "memory");
}

// Four labels of 4 or 8 bytes from shared memory: one or two 16-byte reads.
template <int Bytes>
__device__ __forceinline__ void load4_shared(const typename LabelOf<Bytes>::type* p,
                                             typename LabelOf<Bytes>::wide v[4]) {
  if constexpr (Bytes == 4) {
    const uint4 w = *reinterpret_cast<const uint4*>(p);
    v[0] = w.x; v[1] = w.y; v[2] = w.z; v[3] = w.w;
  } else {
    const ulonglong2 a = reinterpret_cast<const ulonglong2*>(p)[0];
    const ulonglong2 b = reinterpret_cast<const ulonglong2*>(p)[1];
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
}

constexpr int kPlaneBarBytes = 64;     // room for the ring's mbarriers (S <= 8)
// W slices per band, S stages in the ring.  Four stages of 9 rows of 512 4-byte labels (72 KB) leave
// room for 3 CTAs per SM; three of 9 rows of 8-byte labels (108 KB) for 2.
constexpr int kPlaneWarps = 8;
__host__ __device__ constexpr int planes_stages(int label_bytes) { return label_bytes == 8 ? 3 : 4; }

// Labels a[0..3] against b[0..3]: bit e set where they differ.
template <class WT>
__device__ __forceinline__ uint32_t label_changes(const WT a[4], const WT b[4]) {
  return (a[0] != b[0] ? 1u : 0u) | (a[1] != b[1] ? 2u : 0u) | (a[2] != b[2] ? 4u : 0u) | (a[3] != b[3] ? 8u : 0u);
}

// One row source of the march: row source r of item j (0: the halo, 1 + w: warp w's slice) is slice z,
// rows ya .. yb; ok = false: none.  Planes: 2 in 3-D (items are (band, chunk), band fastest), 1 in 2-D
// (warp w of item j takes the (image, chunk) sequence j * W + w, chunk fastest).  Slices and rows are
// counted in 32 bits (take_run_planes), lines and voxels in 64.
struct MarchSource {
  int z, ya, yb;
  bool ok;
};
template <int W, int Planes>
__device__ __forceinline__ MarchSource march_source(int64_t j, int r, int nz, int sy, int depth, int nchunks) {
  MarchSource m;
  int k;
  if constexpr (Planes == 2) {
    const int nbands = (nz + W - 1) / W, z0 = (int)(j % nbands) * W;
    k = (int)(j / nbands);
    m.z = z0 + r - 1;
    m.ok = r == 0 ? (z0 % depth) != 0 : m.z < nz;
  } else {
    const int64_t q = j * W + r - 1;
    m.z = (int)(q / nchunks);
    k = (int)(q - (int64_t)m.z * nchunks);
    m.ok = r > 0 && m.z < nz;
  }
  m.ya = (int)((int64_t)k * sy / nchunks);
  m.yb = (int)((int64_t)(k + 1) * sy / nchunks) - 1;
  return m;
}

// Items of the march over nz slices in nchunks y-chunks each (see march_source).
template <int W, int Planes>
__host__ __device__ __forceinline__ int64_t march_items(int64_t nz, int64_t nchunks) {
  return Planes == 2 ? (nz + W - 1) / W * nchunks : (nz * nchunks + W - 1) / W;
}

// Planes: 1 the y plane, 2 the y and z planes.  nchunks: y-chunks per slice (launch_first_vec).
// Registers capped at the CTAs per SM that the ring leaves room for: 3 for 4-byte labels, 2 for 8-byte ones.
template <int Bytes, int K, bool Plain, int Planes>
__global__ void __launch_bounds__(32 * kPlaneWarps, Bytes == 8 ? 2 : 3)
first_axis_planes_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels,
                         float* __restrict__ out, int64_t nlines, int sx,
                         const float* __restrict__ table, int border, int flags, RunStat stat, XPlanes planes,
                         int nchunks) {
  static_assert(Bytes >= 4 && Planes >= 1 && Planes <= 2, "the bulk copies need 16-byte label rows");
  static_assert(K <= 4, "a lane's nibbles of both planes share one word (gather_plane_words)");
  using LT = typename LabelOf<Bytes>::type;
  using WT = typename LabelOf<Bytes>::wide;
  constexpr int W = kPlaneWarps, S = planes_stages(Bytes);
  extern __shared__ __align__(16) unsigned char planes_smem[];
  pdl_launch_dependents();                           // the second-axis pass may start staging labels

  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int sy = (int)planes.sy, nz = (int)(nlines / planes.sy), depth = (int)planes.depth;
  const unsigned row_bytes = (unsigned)sx * Bytes;
  const int stage_labels = (W + 1) * sx;
  uint64_t* bar = reinterpret_cast<uint64_t*>(planes_smem);
  LT* ring = reinterpret_cast<LT*>(planes_smem + kPlaneBarBytes);
  float* table_s = reinterpret_cast<float*>(planes_smem + kPlaneBarBytes + (size_t)S * stage_labels * Bytes);

  // this CTA's items blockIdx.x + n * gridDim.x; every item takes nst stages (the longest chunk, its
  // leading and trailing rows), stage i holding row ya - 1 + i of each source
  const int64_t items = march_items<W, Planes>(nz, nchunks);
  const int nst = (sy + nchunks - 1) / nchunks + 2;
  // warp 0: the item and stage to issue next; lane r <= W: row source r's next row (src_y, at src_row)
  // and the last row it stages (-1: none)
  int64_t issue_j = blockIdx.x;
  int issue_i = 0, issue_slot = 0, src_y = 0, src_last = -1;
  const LT* src_row = labels;
  auto issue_source = [&]() {
    const MarchSource m = march_source<W, Planes>(issue_j, lane, nz, sy, depth, nchunks);
    src_y = m.ya - 1;
    src_last = m.ok && lane <= W ? min(m.yb + 1, sy - 1) : -1;
    src_row = labels + ((int64_t)m.z * sy + src_y) * sx;
  };
  auto issue_next = [&]() {
    const bool load = src_y >= 0 && src_y <= src_last;
    const unsigned rows = __ballot_sync(full, load);
    uint64_t* b = bar + issue_slot;
    if (lane == 0) mbar_expect_tx(b, __popc(rows) * row_bytes);
    __syncwarp();
    if (load) bulk_load(ring + issue_slot * stage_labels + lane * sx, src_row, row_bytes, b);
    ++src_y;
    src_row += sx;
    if (++issue_slot == S) issue_slot = 0;
    if (++issue_i == nst) {
      issue_i = 0;
      issue_j += gridDim.x;
      issue_source();
    }
  };
  if (threadIdx.x == 0)
    for (int s = 0; s < S; ++s) mbar_init(bar + s, 1);
  __syncwarp();
  if (warp == 0) {
    issue_source();
    for (int s = 0; s < S && issue_j < items; ++s) issue_next();
  }
  for (int i = threadIdx.x; i <= sx; i += blockDim.x) table_s[i] = __ldg(table + i);
  if (threadIdx.x == 0) table_s[sx + 1] = __int_as_float(0x7f800000);
  __syncthreads();

  const unsigned lt_mask = (1u << lane) - 1u;
  const unsigned gt_mask = (lane == 31) ? 0u : (0xfffffffeu << lane);
  const bool keep_background = Plain ? false : (flags & kZeroLabel) != 0;
  const int wpr = (sx + 31) >> 5;
  uint32_t in_row = 0u;                              // the nibbles of the lane's voxels inside the row
#pragma unroll
  for (int b = 0; b < K; ++b)
    if ((b << 7) + (lane << 2) < sx) in_row |= 15u << (4 * b);
  unsigned int nstarts = 0;                          // label changes along x seen by this lane

  int slot = 0;                                      // the slot and phase parity of the item's stage i
  unsigned phase = 0u;
  for (int64_t j = blockIdx.x; j < items; j += gridDim.x) {
    const MarchSource me = march_source<W, Planes>(j, warp + 1, nz, sy, depth, nchunks);
    const bool zfirst = Planes == 2 && me.z % depth == 0;       // the warp's slice starts a volume
    const int ylast = me.ok ? me.yb : -2;                       // the last row it processes
    uint32_t ystart = 0u;                            // y-runs that start at row y (the previous ynext)
    mbar_wait(bar + slot, phase);
    for (int i = 0; i < nst; ++i) {
      const int next_slot = slot + 1 == S ? 0 : slot + 1;
      const unsigned next_phase = next_slot == 0 ? phase ^ 1u : phase;
      const int y = me.ya - 1 + i;
      if (i + 1 < nst) {
        mbar_wait(bar + next_slot, next_phase);
        if (y <= ylast) {
          const LT* cur = ring + slot * stage_labels + (warp + 1) * sx;
          const LT* next = ring + next_slot * stage_labels + (warp + 1) * sx;
          // row y's labels, read from the stage once for all three compares and the distances
          WT v[K][4];
          load_vec_row<Bytes, K>([&](int q0, WT* r) { load4_shared<Bytes>(cur + q0, r); }, sx, lane, v);
          // ---- y-runs that start at row y + 1, 4 bits per block (the line end counts; row -1 stands
          // for the line's start, so row 0 gets all bits) ----
          uint32_t ynext = in_row;
          if (y >= 0 && y + 1 < sy) {
            ynext = 0u;
#pragma unroll
            for (int b = 0; b < K; ++b) {
              const int q0 = (b << 7) + (lane << 2);
              if (q0 >= sx) continue;
              WT u[4];
              load4_shared<Bytes>(next + q0, u);
              ynext |= label_changes<WT>(v[b], u) << (4 * b);
            }
          }
          if (y >= me.ya) {                          // not the leading row: this row's outputs
            const int64_t line = (int64_t)me.z * sy + y;
            // ---- z-runs that start at row y: compare with the stage's row of slice z - 1 (a first slice
            // of a volume: all start) ----
            uint32_t zstart = in_row;
            if (Planes == 2 && !zfirst) {
              const LT* below = cur - sx;
              zstart = 0u;
#pragma unroll
              for (int b = 0; b < K; ++b) {
                const int q0 = (b << 7) + (lane << 2);
                if (q0 >= sx) continue;
                WT u[4];
                load4_shared<Bytes>(below + q0, u);
                zstart |= label_changes<WT>(u, v[b]) << (4 * b);
              }
            }
            const uint32_t one_row = sy > 1 ? (ystart & ynext) : 0u;   // lines of one row have no border term
            uint32_t set_y = 0xffffffffu, set_z = 0xffffffffu;
            first_axis_vec_row<Bytes, K, Plain, true, true>(v, out + line * sx, sx, table_s, border, flags,
                                                            keep_background, lane, lt_mask, gt_mask, nstarts,
                                                            planes.ty, planes.tz, &set_y, &set_z, one_row);
            // ---- settled planes: segment 4 b + w of the row is lanes 8 w .. 8 w + 7 of block b.  The lane's
            // unsettled blocks (y in bits 0 .. 3, z in 4 .. 7) go to bits 4 b + w (y) and 16 + 4 b + w (z);
            // one OR over the warp gives the segments that hold an unsettled voxel ----
            const uint32_t open = ~(set_y & 15u | (set_z & 15u) << 4) & 0xffu;
            const uint32_t open_seg = __reduce_or_sync(full, spread_nibble_bits(open) << (lane >> 3));
            if (lane == 0) {
              planes.settled_y[line] = ~open_seg | 0xffff0000u;
              if (Planes == 2) planes.settled_z[line] = ~(open_seg >> 16);
            }
            // ---- run-start planes: the y nibbles from ystart, the z ones from zstart -> the row's wpr
            // words, word c in lane c, stored by one instruction per plane ----
            uint32_t word_y, word_z;
            gather_plane_words(ystart | zstart << 16, lane, word_y, word_z);
            if (lane < wpr) {
              planes.y[line * wpr + lane] = word_y;
              if (Planes == 2) planes.z[line * wpr + lane] = word_z;
            }
          }
          ystart = ynext;
        }
      }
      __syncthreads();                               // stage i is read by no one any more
      if (warp == 0 && issue_j < items) issue_next();    // the stage S later, into its slot
      slot = next_slot;
      phase = next_phase;
    }
  }
  if (stat.counter) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) nstarts += __shfl_xor_sync(full, nstarts, s);
  }
  publish_run_stat(stat, nstarts, lane);
}

// ---- lower-envelope machinery shared by the three stages of later_axis_tile_kernel ----
//
// hullw[pos >> 5][x] bit (pos & 31) says "pos is a vertex of the lower envelope of its run".
// All navigation is bounded by the run [a, b), because one word can hold bits of several runs.
// One line of the tile: shared addresses of fs[0][x] and hullw[0][x]; rows are ROW bytes apart.
template <int TX>
struct TileLine {
  static constexpr uint32_t ROW = TX * 4;
  uint32_t f;      // &fs[0][x]
  uint32_t hull;   // &hullw[0][x]
  __device__ __forceinline__ float fval(int pos) const { return lds_f32(f + (uint32_t)pos * ROW); }
  __device__ __forceinline__ uint32_t hword(int wi) const { return lds_u32_volatile(hull + (uint32_t)wi * ROW); }
  __device__ __forceinline__ void drop(int pos) const {      // atomic: two runs may share a word
    asm volatile("red.shared.and.b32 [%0], %1;" ::"r"(hull + (uint32_t)(pos >> 5) * ROW), "r"(~(1u << (pos & 31)))
                 : "memory");
  }
};

// Vertex m is hidden when the parabola of r overtakes it no later than m overtakes l:
// s(m,r) <= s(l,m), compared by cross-multiplication in double (the reference divides in
// double, src/edt.hpp:205-221; for integer-valued data both are exact).
__device__ __forceinline__ bool vertex_hidden(int l, float fl, int m, float fm, int r, float fr, double w2) {
  const double dml = (double)(m - l), drm = (double)(r - m);
  const double nml = ((double)fm - (double)fl) + w2 * (dml * (double)(m + l));
  const double nrm = ((double)fr - (double)fm) + w2 * (drm * (double)(r + m));
  return nrm * dml <= nml * drm;
}

// The same test in exact integer arithmetic, for passes whose samples are integer-valued and small
// enough (decided by the host, see launch_later): with g(v) = f[v] + w2 * v^2 < 2^31 the numerators
// are g differences, the denominators position differences, and each side of the cross
// multiplication is one 32 x 32 -> 64-bit product.  No FP64 operations, no conversions to double,
// and a third of the registers -- the envelope stages run at 40 registers per thread.
__device__ __forceinline__ int g_value(float f, int pos, int w2i) {
  return __float2int_rn(f) + w2i * (pos * pos);
}
__device__ __forceinline__ bool vertex_hidden_int(int l, float fl, int m, float fm, int r, float fr, int w2i) {
  const int gl = g_value(fl, l, w2i), gm = g_value(fm, m, w2i), gr = g_value(fr, r, w2i);
  return (long long)(gr - gm) * (long long)(m - l) <= (long long)(gm - gl) * (long long)(r - m);
}

// Largest vertex v with a <= v < pos, or -1.
template <int TX>
__device__ __forceinline__ int prev_vertex(const TileLine<TX> ln, int pos, int a) {
  if (pos <= a) return -1;
  const int wa = a >> 5;
  int wi = (pos - 1) >> 5;
  uint32_t m = ln.hword(wi) & (0xffffffffu >> (31 - ((pos - 1) & 31)));
  for (;;) {
    if (wi == wa) m &= 0xffffffffu << (a & 31);
    if (m) return (wi << 5) + 31 - __clz(m);
    if (wi == wa) return -1;
    --wi;
    m = ln.hword(wi);
  }
}

// Smallest vertex v with pos < v < b, or -1.
template <int TX>
__device__ __forceinline__ int next_vertex(const TileLine<TX> ln, int pos, int b) {
  if (pos + 1 >= b) return -1;
  const int wb = (b - 1) >> 5;
  int wi = (pos + 1) >> 5;
  uint32_t m = ln.hword(wi) & (0xffffffffu << ((pos + 1) & 31));
  for (;;) {
    if (wi == wb) m &= 0xffffffffu >> (31 - ((b - 1) & 31));
    if (m) return (wi << 5) + __ffs(m) - 1;
    if (wi == wb) return -1;
    ++wi;
    m = ln.hword(wi);
  }
}

// A run [a, b) that crosses chunk boundaries is constant if each of its chunk segments was found
// constant in stage 1 (flag bits, see the kernel) and all segments share one value.  Then no scan
// is needed at all: out = min(f, border terms).
template <int TX>
__device__ __forceinline__ bool run_is_constant(const TileLine<TX> ln, uint32_t cflagcol, int a, int b) {
  const int ca = a >> 5, cb = (b - 1) >> 5;
  const float f0 = ln.fval(a);
  if (!(lds_u8_volatile(cflagcol + (uint32_t)ca * TX) & 2u)) return false;      // segment leaving chunk ca
  for (int c = ca + 1; c <= cb; ++c) {
    if (!(lds_u8_volatile(cflagcol + (uint32_t)c * TX) & 1u)) return false;     // segment entering chunk c
    if (!(ln.fval(c << 5) == f0)) return false;
  }
  return true;
}

// Rows of the chunk (bit = row - i0) that belong to a NON-constant segment.  `starts` has a bit at
// the first row of every segment (bit 0 always), `breaks` a bit at every row whose sample differs
// from the row below it inside a segment.  Every break bit is spread over its whole segment: up to
// the segment's last row by letting a carry ripple through the ones of ~starts, and down to its
// first row by the same trick on the bit-reversed words.
__device__ __forceinline__ uint32_t nonconstant_rows(uint32_t starts, uint32_t breaks) {
  const uint32_t m = ~starts;
  const uint32_t up = (((m + breaks) ^ m) | breaks) & m;                  // break row .. last row of the segment
  const uint32_t mr = ~__brev((starts >> 1) | 0x80000000u);              // zeros at the segments' last rows
  const uint32_t br = __brev(breaks >> 1);                               // the row below each break
  const uint32_t down = (((mr + br) ^ mr) | br) & mr;                    // first row of the segment .. row below the break
  return up | __brev(down);
}

// Lower envelopes of all the segments marked in `todo` (bit = row - i0; whole segments, each one
// beginning at a bit of `starts`), as vertex bits added to `hb`.  One loop over the marked rows for
// every lane, whatever the number and the lengths of the segments in its chunk: the vertex stack
// simply restarts where a segment starts.  Classic stack scan with the stack kept as bits: top
// vertex q, the one below it p, and (num, den) = numerator / denominator of s(p,q) so that each
// test is a cross-multiplication in double; samples of +inf are not sites.
template <int TX>
__device__ __forceinline__ uint32_t build_hull_rows(const TileLine<TX> ln, int i0, uint32_t todo, uint32_t starts,
                                                    double w2d, uint32_t hb) {
  const float inf = __int_as_float(0x7f800000);
  int cnt = 0, q = 0, p = 0;                                  // rows relative to i0
  double qd = 0.0, fqd = 0.0, num = 0.0, den = 1.0;
  uint32_t segmask = 0xffffffffu;
  for (uint32_t rest = todo; rest; rest &= rest - 1u) {
    const int r = __ffs(rest) - 1;
    if ((starts >> r) & 1u) { cnt = 0; segmask = 0xffffffffu << r; }
    const float fr = ln.fval(i0 + r);
    if (!(fr < inf)) continue;                                // +inf: not a site
    const double frd = (double)fr, rd = (double)(i0 + r);
    double den_r = rd - qd;
    double num_r = (frd - fqd) + w2d * (den_r * (rd + qd));
    while (cnt >= 2 && num_r * den <= num * den_r) {          // s(q,r) <= s(p,q): q is hidden
      hb &= ~(1u << q);
      --cnt;
      q = p; qd = (double)(i0 + q); fqd = (double)ln.fval(i0 + q);
      if (cnt >= 2) {
        const uint32_t m = hb & segmask & ((1u << q) - 1u);
        p = 31 - __clz(m);
        const double pd = (double)(i0 + p);
        den = qd - pd;
        num = (fqd - (double)ln.fval(i0 + p)) + w2d * (den * (qd + pd));
      }
      den_r = rd - qd;
      num_r = (frd - fqd) + w2d * (den_r * (rd + qd));
    }
    hb |= 1u << r;
    ++cnt;
    p = q; num = num_r; den = den_r;
    q = r; qd = rd; fqd = frd;
  }
  return hb;
}

// build_hull_rows in exact integer arithmetic (see vertex_hidden_int): top vertex q with g(q),
// the vertex below it p with g(p); q is hidden by the newcomer r when
// (g(r) - g(q)) * (q - p) <= (g(q) - g(p)) * (r - q).
template <int TX>
__device__ __forceinline__ uint32_t build_hull_rows_int(const TileLine<TX> ln, int i0, uint32_t todo, uint32_t starts,
                                                        int w2i, uint32_t hb) {
  const float inf = __int_as_float(0x7f800000);
  int cnt = 0, q = 0, p = 0, gq = 0, gp = 0;                  // rows relative to i0
  uint32_t segmask = 0xffffffffu;
  for (uint32_t rest = todo; rest; rest &= rest - 1u) {
    const int r = __ffs(rest) - 1;
    if ((starts >> r) & 1u) { cnt = 0; segmask = 0xffffffffu << r; }
    const float fr = ln.fval(i0 + r);
    if (!(fr < inf)) continue;                                // +inf: not a site
    const int gr = g_value(fr, i0 + r, w2i);
    while (cnt >= 2 && (long long)(gr - gq) * (long long)(q - p) <= (long long)(gq - gp) * (long long)(r - q)) {
      hb &= ~(1u << q);                                       // q is hidden
      --cnt;
      q = p; gq = gp;
      if (cnt >= 2) {
        const uint32_t m = hb & segmask & ((1u << q) - 1u);
        p = 31 - __clz(m);
        gp = g_value(ln.fval(i0 + p), i0 + p, w2i);
      }
    }
    hb |= 1u << r;
    ++cnt;
    p = q; gp = gq;
    q = r; gq = gr;
  }
  return hb;
}

// Is candidate (d1, f1) not above candidate (d0, f0) in exact arithmetic?  Asked when their float32
// values tie: rounded, the candidates along the hull are only weakly unimodal, and a walk that
// steps on a rounded tie can pass the exact minimiser (and, walking up row by row, never come
// back).  w2 (d1^2 - d0^2) is exact in double and so is f1 - f0, because the host gives the tile
// kernels only passes whose every candidate sum is exact in double (launch_later); the sign of
// their double sum is therefore exact.  d0, d1 are integers below 4096, so d^2 is exact in float32.
__device__ __forceinline__ bool tie_not_above(float w2, float d1, float f1, float d0, float f0) {
  const float dd = __fsub_rn(__fmul_rn(d1, d1), __fmul_rn(d0, d0));
  return __dadd_rn(__dsub_rn((double)f1, (double)f0), __dmul_rn((double)w2, (double)dd)) <= 0.0;
}

// Outputs of the rows in `todo` (bit = row - i0): rows of runs that lie INSIDE the chunk (first
// row at a bit of `starts`, last row at a bit of `ends`).  One loop over the marked rows for every
// lane; a run's state is set up at its first row.  A run whose rows are not marked in `noncst` is
// constant: every row is its own best site.  Otherwise the hull bits of the run in `hb` are walked
// (candidate values along the hull are unimodal at a fixed row) and each candidate is evaluated
// with one fused multiply-add, the correctly rounded w2*d^2 + f[v] of src/edt.hpp:225-230.
template <int TX, bool Epilogue>
__device__ __forceinline__ void read_out_rows_local(const TileLine<TX> ln, int i0, uint32_t todo, uint32_t starts,
                                                    uint32_t ends, uint32_t noncst, uint32_t hb, uint32_t wzero,
                                                    int n, float w2f, bool border_lo, bool border_hi, uint32_t sq,
                                                    char* __restrict__ line0, size_t pitch, int flags) {
  constexpr uint32_t ROW = TileLine<TX>::ROW;
  const float inf = __int_as_float(0x7f800000);
  int v = -1, v1 = -1;
  bool lo_b = false, hi_b = false, cst = true, bg = false;
  uint32_t left = 0u;
  float fv = inf, fv1 = inf, dv = 0.0f, dv1 = 0.0f;
  // running addresses of the row at hand (the rows of a run are consecutive): its sample, its two
  // border terms sq[i - a + 1] / sq[b - i], its output
  uint32_t f_at = ln.f, sq_lo = sq, sq_hi = sq;
  char* dst = line0;
  for (uint32_t rest = todo; rest; rest &= rest - 1u) {
    const int r = __ffs(rest) - 1;
    if ((starts >> r) & 1u) {                                 // first row of a run
      const int e = __ffs(ends & (0xffffffffu << r)) - 1;     // its last row
      const int a = i0 + r, b = i0 + e + 1;
      lo_b = a > 0 || border_lo; hi_b = b < n || border_hi;
      cst = !((noncst >> r) & 1u);
      bg = (wzero >> r) & 1u;
      f_at = ln.f + (uint32_t)a * ROW;
      sq_lo = sq + 4u;
      sq_hi = sq + (uint32_t)(b - a) * 4u;
      dst = line0 + (size_t)a * pitch;
      v = v1 = -1; fv = fv1 = inf;
      if (!cst) {
        left = hb & (0xffffffffu << r) & (0xffffffffu >> (31 - e));
        if (left) {
          v = __ffs(left) - 1; left &= left - 1u;
          fv = ln.fval(i0 + v); dv = (float)(r - v);
          if (left) { v1 = __ffs(left) - 1; left &= left - 1u; fv1 = ln.fval(i0 + v1); dv1 = (float)(r - v1); }
        }
      }
    }
    float best = inf;
    if (cst) {
      best = lds_f32(f_at);
    } else if (v >= 0) {
      best = __fmaf_rn(w2f, __fmul_rn(dv, dv), fv);
      while (v1 >= 0) {
        const float cand = __fmaf_rn(w2f, __fmul_rn(dv1, dv1), fv1);
        if (!(cand <= best)) break;
        if (cand == best && !tie_not_above(w2f, dv1, fv1, dv, fv)) break;
        best = cand; v = v1; fv = fv1; dv = dv1;
        if (left) { v1 = __ffs(left) - 1; left &= left - 1u; fv1 = ln.fval(i0 + v1); dv1 = (float)(r - v1); }
        else v1 = -1;
      }
      dv += 1.0f; dv1 += 1.0f;
    }
    if (lo_b) best = fminf(best, lds_f32(sq_lo));
    if (hi_b) best = fminf(best, lds_f32(sq_hi));
    if (Epilogue) best = finish_value(best, bg, flags);       // a run has one label
    *reinterpret_cast<float*>(dst) = best;
    f_at += ROW; sq_lo += 4u; sq_hi -= 4u; dst += pitch;
  }
}

// State of the walk along the final hull of a run [a, b) that crosses chunk boundaries, for the
// rows of one chunk: current vertex v, next vertex v1, and an iterator over the vertices above v1
// (`rem` = the not yet visited vertex bits of hull word `wi`, clipped to the run in its last word).
struct HullWalk {
  int b, v, v1, wi;
  uint32_t rem;
  float fv, fv1, dv, dv1;
};

// v1 <- the next vertex of the run above the current v1 (or -1), and its sample.
template <int TX>
__device__ __forceinline__ void walk_advance(HullWalk& w, const TileLine<TX> ln, int row) {
  const int wb = (w.b - 1) >> 5;
  while (!w.rem) {
    if (w.wi >= wb) { w.v1 = -1; return; }
    ++w.wi;
    w.rem = ln.hword(w.wi);
    if (w.wi == wb) w.rem &= 0xffffffffu >> (31 - ((w.b - 1) & 31));
  }
  w.v1 = (w.wi << 5) + __ffs(w.rem) - 1;
  w.rem &= w.rem - 1u;
  w.fv1 = ln.fval(w.v1);
  w.dv1 = (float)(row - w.v1);
}

// Sets the walk up for row `lo` of the run [a, b): the vertex that dominates row lo is found by
// starting at the nearest vertex at or below lo (else the first one above) and descending along
// the hull -- at a fixed row the candidate values are unimodal.
template <int TX>
__device__ __forceinline__ void walk_begin(HullWalk& w, const TileLine<TX> ln, int lo, int a, int b, float w2f) {
  const float inf = __int_as_float(0x7f800000);
  w.b = b;
  w.v = w.v1 = -1; w.fv = w.fv1 = inf; w.dv = w.dv1 = 0.0f;
  w.wi = 0; w.rem = 0u;
  int v = prev_vertex<TX>(ln, lo + 1, a);
  if (v < 0) v = next_vertex<TX>(ln, lo, b);
  if (v >= 0) {
    float fv = ln.fval(v), dv = (float)(lo - v);
    float best = __fmaf_rn(w2f, __fmul_rn(dv, dv), fv);
    for (;;) {
      const int u = prev_vertex<TX>(ln, v, a);
      if (u < 0) break;
      const float fu = ln.fval(u);
      const float du = (float)(lo - u);
      const float cand = __fmaf_rn(w2f, __fmul_rn(du, du), fu);
      // rounded to float32 the candidates are only weakly unimodal: two adjacent vertices that
      // round to the same value may hide a lower one farther down, so ties are settled exactly
      if (!(cand <= best)) break;
      if (cand == best && !tie_not_above(w2f, du, fu, dv, fv)) break;
      best = cand; v = u; fv = fu; dv = du;
    }
    w.v = v; w.fv = fv; w.dv = dv;
    // iterator over the vertices above v
    const int wb = (b - 1) >> 5;
    w.wi = v >> 5;
    w.rem = ((v & 31) == 31) ? 0u : (ln.hword(w.wi) & (0xfffffffeu << (v & 31)));
    if (w.wi == wb) w.rem &= 0xffffffffu >> (31 - ((b - 1) & 31));
    walk_advance<TX>(w, ln, lo);
  }
}

// The Y pass's refresh of the Z pass's settled plane (RunBits::refresh) by a tile that ran, after all
// its stores: values only fall within a pass, so bits only go from clear to set.  Thread t takes row t
// (blockDim.x >= n: no wide tiles).  When at most 32 of the tile's rows have the bit clear, one warp
// per such row re-reads its values (L2-hot) and sets the bit if none exceeds refresh_t; with more,
// the bits stay clear, which is still correct.  Other tiles of the same rows own the words' other
// bits, hence the atomic.  Its first barrier orders the tile's stores before the re-reads.
__device__ __forceinline__ void refresh_settled(const RunBits& rb, const float* f, const LineGeom& g, int64_t outer,
                                                int64_t inner0, int n) {
  const int t = threadIdx.x, lane = t & 31;
  const uint32_t bit = 1u << (int)(inner0 >> 5);       // the tile is x-segment inner0 / 32 of its rows
  uint32_t* const words = rb.refresh + outer * rb.settled_outer;
  const bool clear = t < n && !(words[(int64_t)t * rb.settled_row] & bit);
  const int nclear = __syncthreads_count(clear);
  if (nclear == 0 || nclear > 32) return;
  const bool live = inner0 + lane < g.inner_count;     // padding lines count as settled
  const float* col = f + (outer * g.outer_stride + inner0 + lane);
  for (uint32_t m = __ballot_sync(0xffffffffu, clear); m; m &= m - 1u) {
    const int64_t i = (t & ~31) + __ffs(m) - 1;
    const float v = live ? col[i * g.line_stride] : 0.0f;
    if (__all_sync(0xffffffffu, v <= rb.refresh_t) && lane == 0) atomicOr(words + i * rb.settled_row, bit);
  }
}

// The settled check of the grouped tile kernel: bit k of the result is set when tile t0 + k (of the
// cnt tiles from t0) has a segment that is not settled -- the per-tile check of later_axis_tile_kernel
// over the whole group in one read of the plane.  Thread t takes row t and walks the tiles from t0
// without a division per tile: tile k covers the lines [j0, j0 + TX) of its outer, which reach rows
// q, q + 1, ... of the plane, cut at multiples of sx (r: j0's place in row q).  Consecutive tiles share
// their word (the x-segments of one row), which is loaded once.  The masks are OR-ed over the CTA
// through `slots` (one word per warp), so the result is CTA-uniform.
template <int TX>
__device__ __forceinline__ uint32_t unsettled_tiles(const RunBits& rb, const LineGeom& g, int64_t t0, int cnt, int n,
                                                    uint32_t* slots) {
  const int64_t outer0 = t0 / g.tiles_per_outer;
  const int64_t j00 = (t0 - outer0 * g.tiles_per_outer) * TX;
  const int64_t q00 = j00 / rb.sx;
  uint32_t m = 0u;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    int64_t outer = outer0, j0 = j00, q = q00, r = j00 - q00 * rb.sx;
    int64_t last = -1;                                 // the index of the word in w
    uint32_t w = 0u;
    for (int k = 0; k < cnt; ++k) {
      bool settled = true;
      int64_t left = min((int64_t)TX, g.inner_count - j0), qq = q, rr = r;
      while (left > 0) {
        const int64_t take = min(left, rb.sx - rr);   // lines [rr, rr + take) of row qq
        const int lo = (int)rr, hi = (int)(rr + take) - 1;
        const uint32_t need = (0xffffffffu >> (31 - (hi >> 5))) & (0xffffffffu << (lo >> 5));
        const int64_t at = outer * rb.settled_outer + qq + (int64_t)i * rb.settled_row;
        if (at != last) { w = __ldg(rb.settled + at); last = at; }
        settled = settled && (w & need) == need;
        left -= take; rr = 0; ++qq;
      }
      if (!settled) m |= 1u << k;
      j0 += TX;
      if (j0 >= g.inner_count) {                       // the next tile starts the next outer
        ++outer; j0 = 0; q = 0; r = 0;
      } else {
        for (r += TX; r >= rb.sx; r -= rb.sx) ++q;
      }
    }
  }
  m = __reduce_or_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0) slots[threadIdx.x >> 5] = m;
  __syncthreads();
  for (int wi = 0; wi < (int)(blockDim.x >> 5); ++wi) m |= slots[wi];
  return m;
}

// The grouped tile kernel's step to its next tile: false when none is left; otherwise the barrier
// that frees the shared memory of the tile that ended, and the parity of the next mbarrier phase.
__device__ __forceinline__ bool next_group_tile(uint32_t todo, uint32_t& phase) {
  if (!todo) return false;
  __syncthreads();
  phase ^= 1u;
  return true;
}

// MinCtas: CTAs of 512 threads per SM the kernel is compiled for.  3 (40 registers, a few spills)
// is what the envelope stages want -- they are latency-bound and the third CTA's warps hide it;
// 2 (60 registers, no spills) is faster when nearly every run is one row long (label noise), where
// only the streaming path runs.  The host picks per launch (edt_passes.cuh).
// IntHull: hull tests in exact integer arithmetic (the host guarantees integer-valued samples with
// f + w2 * n^2 < 2^31 and passes w2 as an integer in `w2i`); otherwise in double.
// Bits: stage 0 reads the pass's run-start plane (RunBits, written by the X pass) instead of the
// labels: 4 + 1/8 bytes per voxel instead of 4 + Bytes on label noise, where nothing is stored.  The
// plane is read only after griddepcontrol.wait: the Z pass may start while the X pass is still
// running (the Y pass lets its dependents start before it waits itself).  Compiled for the
// label-noise shape only (2 CTAs per SM, TMA, 32-wide tiles, no background bits: unsigned transforms).
// Grouped (skips_settled: Bits with IntHull and no epilogue, the only instance that skips settled
// tiles and refreshes the Z pass's settled plane): a CTA owns the
// rb.group consecutive tiles from blockIdx.x * rb.group.  It reads the settled words of the whole
// group once, then runs the tiles that are not settled one after another, with the border table and
// the mbarrier set up once: a pass that skips nearly every tile costs one read per CTA instead of a
// CTA launch and an L2 round trip per tile (DESIGN.md section 4.1).
template <int Bytes, int TX, bool Epilogue, bool UseTMA, bool Wide, int MinCtas, bool IntHull, bool Bits = false>
__global__ void __launch_bounds__(Wide ? 1024 : 512, Wide ? 1 : MinCtas)
later_axis_tile_kernel(const __grid_constant__ CUtensorMap fmap,
                       const typename LabelOf<Bytes>::type* __restrict__ labels, const RunBits rb,
                       float* __restrict__ f, LineGeom g, TileBoxes tb, float w2,
                       int border_lo, int border_hi, int flags, int w2i) {
  static_assert(!Bits || (UseTMA && !Wide), "the run-start plane is read by the TMA, non-wide variants only");
  using LT = typename LabelOf<Bytes>::type;
  extern __shared__ __align__(128) unsigned char smem_tile[];
  constexpr int SUBS = 32 / TX;                       // chunks handled side by side by one warp
  // Variants with registers to spare (2 CTAs per SM, or one wide CTA) step a 64-bit label pointer
  // and share one pass over the samples between (1a) and (1b); at 40 registers both cost spills.
  constexpr bool kRoomy = Wide || MinCtas == 2;
  // One CTA per SM (lines of more than 512 rows): nothing else on the SM hides the label-load
  // latency, so the warps are decoupled -- one early barrier, then every warp loads its labels,
  // waits for the float tile and finishes its chunks at its own pace.  With two or
  // three CTAs per SM the other CTAs hide it and the extra work per chunk only costs.
  constexpr bool kDecoupled = Wide;
  constexpr uint32_t ROW = TX * 4;                    // bytes between rows of fs / between words

  const int n = g.n;
  const int nchunks = (n + 31) >> 5;
  const int rows_alloc = UseTMA ? tb.box_rows * tb.nboxes : n;
  // shared-memory map (byte addresses in the shared window)
  const uint32_t fs_a = smem_addr(smem_tile);                           // float [rows_alloc][TX]
  const uint32_t startw_a = fs_a + (uint32_t)rows_alloc * ROW;          // u32   [nchunks][TX]
  const uint32_t zerow_a = startw_a + (uint32_t)nchunks * ROW;          // u32   [nchunks][TX]
  const uint32_t hullw_a = zerow_a + (uint32_t)nchunks * ROW;           // u32   [nchunks][TX]
  const uint32_t sq_a = hullw_a + (uint32_t)nchunks * ROW;              // float [n + 2]
  const uint32_t bar_a = sq_a + (uint32_t)((n + 2 + 1) & ~1) * 4u;      // mbarrier
  const uint32_t nz_a = bar_a + 16u;                                    // u32   [TX]: chunks holding a run start
  const uint32_t cflag_a = nz_a + TX * 4u;                              // u8    [nchunks][TX]
  const bool use_nz = nchunks <= 32;                                    // (one bit per chunk; longer lines search)
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_tile + (bar_a - fs_a));

  const int lane = threadIdx.x & 31;
  const int x = lane & (TX - 1);
  const int chunk0 = (threadIdx.x >> 5) * SUBS + (lane / TX);
  const int chunk_step = (blockDim.x >> 5) * SUBS;
  constexpr bool kGrouped = skips_settled(Bits, IntHull, Epilogue);

  // (kGrouped) bit k of `todo`: tile t0 + k is still to run.  The group's settled tiles are dropped
  // here, before the mbarrier, any tile load or the border table.  The hull words hold the check's
  // per-warp masks: they are first written in stage 1, behind the barrier that ends stage 0.
  int64_t t0 = 0;
  uint32_t todo = 0u, phase = 0u;      // phase: the parity of the mbarrier phase of the current tile
  if constexpr (kGrouped) {
    pdl_launch_dependents();
    t0 = (int64_t)blockIdx.x * rb.group;
    const int cnt = (int)min((int64_t)rb.group, (int64_t)g.tiles_per_outer * g.outer_count - t0);
    todo = cnt >= 32 ? 0xffffffffu : (1u << cnt) - 1u;
    if (rb.settled) {
      pdl_wait_for_previous_grid();    // the plane is complete (Z pass: and refreshed by the Y pass)
      todo &= unsettled_tiles<TX>(rb, g, t0, cnt, n, reinterpret_cast<uint32_t*>(smem_tile + (hullw_a - fs_a)));
    }
    if (!todo) return;
    for (int i = threadIdx.x; i < n + 2; i += blockDim.x) {
      const float e = (float)i;
      sts_f32(sq_a + (uint32_t)i * 4u, __fmul_rn(w2, __fmul_rn(e, e)));
    }
    if (threadIdx.x == 0) {
      pdl_wait_for_previous_grid();
      mbar_init(bar, 1);               // made visible by the barrier that ends stage 0
    }
  }
  // One tile per pass of this loop; only the grouped kernel takes a second pass (`continue` ends a tile).
  do {
    int64_t tile = blockIdx.x;
    if constexpr (kGrouped) {
      tile = t0 + __ffs(todo) - 1;
      todo &= todo - 1u;
    }
    const int64_t outer = tile / g.tiles_per_outer;
    const int64_t inner0 = (tile - outer * g.tiles_per_outer) * TX;
    const bool live = (inner0 + x) < g.inner_count;
    // CTA-uniform tile origin + 32-bit element offsets (the host guarantees n * line_stride < 2^32)
    const LT* __restrict__ tl = labels + (outer * g.outer_stride + inner0);
    float* __restrict__ tf = f + (outer * g.outer_stride + inner0);
    const uint32_t ls = (uint32_t)g.line_stride;
    const size_t pitch = (size_t)ls * sizeof(float);
    const float inf = __int_as_float(0x7f800000);
    const double w2d = (double)w2;

    if (!kGrouped) pdl_launch_dependents();  // the next pass may start staging its labels during our tail
    if (!UseTMA) pdl_wait_for_previous_grid();           // plain loads of f happen in the staging loop
    // Float tile by TMA, border-term table, chunk mask.  (kDecoupled) together with the mbarrier the
    // table and the mask are the only things a warp needs from other warps before the votes at the end
    // of stage 1, so the one barrier comes here, early, while no warp has loads in flight yet; the tile
    // is requested right behind it, together with the first label loads.
    if (UseTMA && threadIdx.x == 0) {
      if (!kGrouped) {
        if (!kDecoupled) pdl_wait_for_previous_grid();    // f is complete only when the previous pass has finished
        mbar_init(bar, 1);
      }
      if (!kDecoupled) {
        mbar_expect_tx(bar, (unsigned)rows_alloc * ROW);
        for (int bx = 0; bx < tb.nboxes; ++bx)
          tma_load_3d(smem_tile + (size_t)bx * tb.box_rows * ROW, &fmap, (int)inner0, bx * tb.box_rows, (int)outer, bar);
      }
    }
    if (threadIdx.x < TX) sts_u32(nz_a + threadIdx.x * 4u, 0u);
    for (int i = threadIdx.x; !kGrouped && i < n + 2; i += blockDim.x) {
      const float e = (float)i;
      sts_f32(sq_a + (uint32_t)i * 4u, __fmul_rn(w2, __fmul_rn(e, e)));
    }
    if (kDecoupled) {
      __syncthreads();
      if (UseTMA && threadIdx.x == 0) {
        pdl_wait_for_previous_grid();
        mbar_expect_tx(bar, (unsigned)rows_alloc * ROW);
        for (int bx = 0; bx < tb.nboxes; ++bx)
          tma_load_3d(smem_tile + (size_t)bx * tb.box_rows * ROW, &fmap, (int)inner0, bx * tb.box_rows, (int)outer, bar);
      }
    }

    // ============ stage 0 (Bits): run-start bits -> one word per (chunk, line) ============
    if constexpr (Bits) {
      pdl_wait_for_previous_grid();      // the plane is complete (written by the X pass)
      if (live) {
        const int64_t j = inner0 + x, q = j / rb.sx, rj = j - q * rb.sx;
        const uint32_t* bstart = rb.start + (outer * rb.outer_words + q * rb.wpr + (rj >> 5));
        const int bit = (int)(rj & 31);
        const size_t rw = (size_t)rb.row_words;
        for (int c = chunk0; c < nchunks; c += chunk_step) {
          const int i0 = c << 5;
          const uint32_t* sp = bstart + (size_t)i0 * rw;
          uint32_t wstart = 0;
          if (i0 + 32 <= n) {
  #pragma unroll
            for (int r = 0; r < 32; ++r) wstart |= ((__ldg(sp + r * rw) >> bit) & 1u) << r;
          } else {
            for (int r = 0; r < n - i0; ++r) wstart |= ((__ldg(sp + r * rw) >> bit) & 1u) << r;
            wstart |= 1u << (n - i0);        // pretend a run starts at row n (line end)
          }
          if (i0 == 0) wstart |= 1u;         // a run starts at row 0 by definition
          sts_u32(startw_a + (uint32_t)c * ROW + (uint32_t)x * 4u, wstart);
          if (Epilogue) sts_u32(zerow_a + (uint32_t)c * ROW + (uint32_t)x * 4u, 0u);   // no sign: not read
        }
      } else {
        for (int c = chunk0; c < nchunks; c += chunk_step) {
          sts_u32(startw_a + (uint32_t)c * ROW + (uint32_t)x * 4u, 0u);
          if (Epilogue) sts_u32(zerow_a + (uint32_t)c * ROW + (uint32_t)x * 4u, 0u);
        }
      }
    }

    // ============ stage 0: labels -> run-start / background words ============
    for (int c = chunk0; !Bits && c < nchunks; c += chunk_step) {
      const int i0 = c << 5;
      uint32_t wstart = 0, wzero = 0, ext = 1u;      // ext: a run starts at row i0 + 32 (or the line ends there)
      if (live) {
        uint32_t idx = (uint32_t)i0 * ls + (uint32_t)x;
        const LT* lp = tl + idx;               // (kRoomy) stepped by one line stride per row
        LT prev = (i0 > 0) ? tl[idx - ls] : (LT)0;
        uint32_t fdst = fs_a + (uint32_t)i0 * ROW + (uint32_t)x * 4u;
        if (i0 + 32 <= n) {
  #pragma unroll
          for (int r = 0; r < 32; ++r) {
            const LT here = kRoomy ? *lp : tl[idx];
            if (kRoomy) lp += ls;
            if (!UseTMA) sts_f32(fdst + r * ROW, tf[idx]);
            if (!UseTMA || !kRoomy) idx += ls;
            if (here != prev) wstart |= (1u << r);
            if (Epilogue && here == 0) wzero |= (1u << r);
            prev = here;
          }
          if (kDecoupled && i0 + 32 < n) ext = (kRoomy ? *lp : tl[idx]) != prev;
        } else {
          for (int r = 0; r < n - i0; ++r) {
            const LT here = kRoomy ? *lp : tl[idx];
            if (kRoomy) lp += ls;
            if (!UseTMA) sts_f32(fdst + r * ROW, tf[idx]);
            if (!UseTMA || !kRoomy) idx += ls;
            if (here != prev) wstart |= (1u << r);
            if (Epilogue && here == 0) wzero |= (1u << r);
            prev = here;
          }
          wstart |= 1u << (n - i0);          // pretend a run starts at row n (line end)
        }
        if (i0 == 0) wstart |= 1u;           // a run starts at row 0 by definition
      }
      sts_u32(startw_a + (uint32_t)c * ROW + (uint32_t)x * 4u, wstart);
      if (Epilogue) sts_u32(zerow_a + (uint32_t)c * ROW + (uint32_t)x * 4u, wzero);
      if (kDecoupled) sts_u8(cflag_a + (uint32_t)(c * TX + x), ext << 2);   // bit 2 of the chunk's flag byte, for stage 1
    }
    pdl_wait_for_previous_grid();        // nobody may store into f before the previous pass is done
    if (!UseTMA || !kDecoupled) __syncthreads();   // words, table (and plain-loaded tile) visible; orders the mbarrier init
    if (UseTMA) mbar_wait(bar, phase);   // float tile has landed

    // every shared address used from here on carries the token, so no (non-volatile) load of the
    // staged tile can be scheduled above the barrier / the TMA completion wait
    const uint32_t tok = smem_token();
    TileLine<TX> ln;
    ln.f = fs_a + (uint32_t)x * 4u + tok;
    ln.hull = hullw_a + (uint32_t)x * 4u + tok;
    const uint32_t startcol = startw_a + (uint32_t)x * 4u + tok;
    const uint32_t zerocol = zerow_a + (uint32_t)x * 4u + tok;
    const uint32_t sq_t = sq_a + tok;
    // per (chunk, line): bit 0 = the long-run segment entering from below is constant,
    //                    bit 1 = the long-run segment leaving above is constant
    const uint32_t cflagcol = cflag_a + (uint32_t)x;
    const uint32_t nzcol = nz_a + (uint32_t)x * 4u;
    char* const line0 = reinterpret_cast<char*>(tf + x);

    // ============ stage 1: everything that can be finished inside a chunk ============
    // Per chunk (32 rows of one line): the rows are cut into segments by the run starts; a segment
    // is LOCAL when its run lies inside the chunk and CROSSING when the run goes on in the chunk
    // below and / or above.
    //   (1a) runs of length one: min(f, w2), straight-line predicated code;
    //   (1b) which segments are constant (no scan needed), from one pass over the samples;
    //   (1c) hulls of all non-constant segments, ONE loop over their rows (build_hull_rows);
    //   (1d) outputs of the local runs, ONE loop over their rows (read_out_rows_local).
    // The hull bits of the crossing segments go to hullw for stages 2 and 3.
    int any_cross = 0;
    if (live) {
      for (int c = chunk0; c < nchunks; c += chunk_step) {
        const int i0 = c << 5;
        const int rows = min(32, n - i0);
        const uint32_t rowmask = rows == 32 ? 0xffffffffu : ((1u << rows) - 1u);
        const uint32_t wstart = lds_u32(startcol + (uint32_t)c * ROW);
        const uint32_t wzero = Epilogue ? lds_u32(zerocol + (uint32_t)c * ROW) : 0u;
        // bit r of `nextw`: a run starts at row i0 + r + 1 (the line end counts as a start)
        // ext: a run starts at row i0 + 32 (the line end counts as a start)
        uint32_t ext = 1u;
        if (kDecoupled) ext = (lds_u8_volatile(cflagcol + (uint32_t)c * TX) >> 2) & 1u;     // (this thread's own store)
        else if (i0 + 32 < n) ext = lds_u32(startcol + (uint32_t)(c + 1) * ROW) & 1u;
        const uint32_t nextw = (wstart >> 1) | (ext << 31);
        uint32_t single = wstart & nextw & rowmask;          // runs of length one
        if (!border_lo && c == 0) single &= ~1u;             // rows lacking a border term go the long way
        if (!border_hi && i0 + 32 >= n) single &= ~(1u << (n - 1 - i0));

        // (1a) runs of length one: out = min(f, w2).  The pass works in place, so a row that keeps its
        // value (f <= w2 -- with label noise nearly every row of the later passes) is not stored at
        // all: one pass over the chunk's samples marks the rows that change (`chg`) and, for (1b),
        // the rows whose sample differs from the row below (`breaks`).  The square root / sign of the
        // last pass rewrites every row.
        uint32_t breaks = 0u;
        bool have_breaks = false;
        const uint32_t multi = rowmask & ~single;
        {
          const uint32_t at = ln.f + (uint32_t)i0 * ROW;
          if (single && !Epilogue && kRoomy) {
            have_breaks = true;
            uint32_t chg = 0u;
            float prev = lds_f32(at);
            if (prev > w2) chg = 1u;
            if (rows == 32) {
  #pragma unroll
              for (int r = 1; r < 32; ++r) {
                const float cur = lds_f32(at + r * ROW);
                if (cur != prev) breaks |= 1u << r;
                if (cur > w2) chg |= 1u << r;
                prev = cur;
              }
            } else {
              for (int r = 1; r < rows; ++r) {
                const float cur = lds_f32(at + r * ROW);
                if (cur != prev) breaks |= 1u << r;
                if (cur > w2) chg |= 1u << r;
                prev = cur;
              }
            }
            for (chg &= single; chg; chg &= chg - 1u)
              *reinterpret_cast<float*>(line0 + (size_t)(i0 + __ffs(chg) - 1) * pitch) = w2;
          } else {
            if (single) {                     // value computed unconditionally, store predicated
              char* op = line0 + (size_t)i0 * pitch;
              if (rows == 32) {
  #pragma unroll
                for (int r = 0; r < 32; ++r) {
                  const float fv = lds_f32(at + r * ROW);
                  if (Epilogue) {
                    const float v = finish_value(fminf(fv, w2), (wzero >> r) & 1u, flags);
                    if (single & (1u << r)) *reinterpret_cast<float*>(op) = v;
                  } else {
                    if ((single & (1u << r)) && fv > w2) *reinterpret_cast<float*>(op) = w2;
                  }
                  op += pitch;
                }
              } else {
                for (int r = 0; r < rows; ++r) {
                  const float fv = lds_f32(at + r * ROW);
                  float v = fminf(fv, w2);
                  if (Epilogue) v = finish_value(v, (wzero >> r) & 1u, flags);
                  if ((single & (1u << r)) && (Epilogue || fv > w2)) *reinterpret_cast<float*>(op) = v;
                  op += pitch;
                }
              }
            }
          }
        }

        uint32_t hb = 0u;
        if (multi) {
          const uint32_t wreal = wstart & rowmask;
          const uint32_t starts = wreal | 1u;                // the segment entering from below starts at row 0
          const bool entering = !(wstart & 1u), leaving = !ext;
          const uint32_t ent_mask = entering ? (wreal ? ((1u << (__ffs(wreal) - 1)) - 1u) : rowmask) : 0u;
          const int s2 = 31 - __clz(starts);                 // first row of the last segment
          const uint32_t lea_mask = (leaving && wreal) ? (0xffffffffu << s2) : 0u;
          const uint32_t cross_mask = ent_mask | lea_mask;

          // (1b) rows whose sample differs from the row below, then the rows of non-constant segments
          if (!have_breaks) {
            const uint32_t at = ln.f + (uint32_t)i0 * ROW;
            float prev = lds_f32(at);
            if (rows == 32) {
  #pragma unroll
              for (int r = 1; r < 32; ++r) {
                const float cur = lds_f32(at + r * ROW);
                if (cur != prev) breaks |= 1u << r;
                prev = cur;
              }
            } else {
              for (int r = 1; r < rows; ++r) {
                const float cur = lds_f32(at + r * ROW);
                if (cur != prev) breaks |= 1u << r;
                prev = cur;
              }
            }
          }
          const uint32_t noncst = nonconstant_rows(starts, breaks & ~starts & rowmask) & multi;
          // a constant crossing segment is its own hull: equal heights never hide one another
          if (cross_mask) {
            uint32_t cflags = 0u;
            if (ent_mask && !(noncst & ent_mask)) { cflags |= 1u; if (ln.fval(i0) < inf) hb |= ent_mask; }
            if (lea_mask && !(noncst & lea_mask)) { cflags |= 2u; if (ln.fval(i0 + s2) < inf) hb |= lea_mask; }
            sts_u8(cflagcol + (uint32_t)c * TX, cflags);
            any_cross |= 1;
            // bit 1: a crossing run that is not constant here, or across the boundary below
            if ((noncst & cross_mask) || (entering && ln.fval(i0) != ln.fval(i0 - 1))) any_cross |= 2;
          }
          // (1c) hulls of the non-constant segments
          if (noncst) hb = IntHull ? build_hull_rows_int<TX>(ln, i0, noncst, starts, w2i, hb)
                                   : build_hull_rows<TX>(ln, i0, noncst, starts, w2d, hb);
          // (1d) the local runs are finished here
          const uint32_t local = multi & ~cross_mask;
          if (local)
            read_out_rows_local<TX, Epilogue>(ln, i0, local, starts, nextw, noncst, hb, wzero, n, w2, border_lo,
                                              border_hi, sq_t, line0, pitch, flags);
        }
        sts_u32(ln.hull + (uint32_t)c * ROW, hb);
      }
    }
    if (!__syncthreads_or(any_cross)) {                      // every run was finished inside its chunk
      if constexpr (kGrouped) {
        if (rb.refresh) refresh_settled(rb, f, g, outer, inner0, n);
      }
      continue;
    }
    // Tiles with crossing runs: one bit per chunk that holds a run start, per line, so that the ends
    // of a crossing run are two look-ups instead of a walk over the chunks (made visible by the vote below).
    if (live && use_nz) {
      for (int c = chunk0; c < nchunks; c += chunk_step) {
        const uint32_t rowmask = (n - (c << 5) >= 32) ? 0xffffffffu : ((1u << (n - (c << 5))) - 1u);
        if (lds_u32(startcol + (uint32_t)c * ROW) & rowmask) red_shared_or(nzcol, 1u << c);
      }
    }
    // every crossing run of the tile constant (blocky labels, solid objects along this axis)?  Then
    // nothing needs stitching and stage 3 writes min(f, border terms) without looking at any hull.
    const bool all_const = !__syncthreads_or(any_cross & 2);

    // ============ stage 2: stitch the hulls of runs that cross chunk boundaries ============
    // Divide and conquer over the chunk segments of every run: the boundaries of a run are numbered
    // j = 1, 2, ... from the chunk the run starts in; in the round with group size `half` every
    // boundary with j = half (mod 2 half) merges the `half` segments left of it with the (up to)
    // `half` segments right of it, all runs, boundaries and lines in parallel.  Left of a boundary
    // stands the finished hull of the run's rows in the left group (A), right of it the finished hull
    // of its rows in the right group (B).  All of A lies left of all of B, so the hull of the union
    // is a prefix of A plus a suffix of B: drop A's top while it is hidden by (the vertex below it,
    // B's first), drop B's first while it is hidden by (A's top, B's second), until neither applies.
    // Numbering the boundaries per run (not per line) keeps the number of rounds -- each ends in a
    // CTA-wide barrier -- at log2 of the longest run's chunk count instead of log2 of the line's:
    // two rounds for runs of up to 128 rows.  Boundaries of different runs may meet in one hull word,
    // so bits are dropped with an atomic AND.
    if (!all_const) {
      for (int half = 1; half < nchunks; half <<= 1) {
        int more = 0;
        if (live) {
          for (int c = chunk0; c < nchunks; c += chunk_step) {
            if (c == 0) continue;                              // no boundary below the first chunk
            const int i0 = c << 5;
            const uint32_t wc = lds_u32(startcol + (uint32_t)c * ROW);
            if (wc & 1u) continue;                             // a run starts exactly here: nothing crosses
            int a = 0;                                         // start of the run that crosses
            int b = n;                                         // its end (exclusive)
            if (use_nz) {
              const uint32_t nzw = lds_u32_volatile(nzcol);
              const uint32_t below = nzw & ((1u << c) - 1u), above = nzw & (0xffffffffu << c);
              if (below) {
                const int cc = 31 - __clz(below);
                a = (cc << 5) + 31 - __clz(lds_u32(startcol + (uint32_t)cc * ROW));
              }
              if (above) {
                const int cc = __ffs(above) - 1;
                b = min(n, (cc << 5) + __ffs(lds_u32(startcol + (uint32_t)cc * ROW)) - 1);
              }
            } else {
              for (int cc = c - 1; cc >= 0; --cc) {
                const uint32_t w = lds_u32(startcol + (uint32_t)cc * ROW);
                if (w) { a = (cc << 5) + 31 - __clz(w); break; }
              }
              for (int cc = c; cc < nchunks; ++cc) {
                const uint32_t w = lds_u32(startcol + (uint32_t)cc * ROW);
                if (w) { b = min(n, (cc << 5) + __ffs(w) - 1); break; }
              }
            }
            const int ca = a >> 5, cb = (b - 1) >> 5;          // the run has boundaries 1 .. cb - ca
            if (cb - ca >= 2 * half) more = 1;                 // some boundary of it waits for a later round
            if (((c - ca) & (2 * half - 1)) != half) continue; // not this boundary's round
            if (half == 1) {
              // (first round only: later rounds see hulls that earlier merges may have thinned out)
              // equal-height rows on both sides of the boundary cannot hide one another: when the two
              // adjacent chunk segments are constant and equal there is nothing to drop here
              const uint32_t fl_hi = lds_u8_volatile(cflagcol + (uint32_t)c * TX);
              const uint32_t fl_lo = lds_u8_volatile(cflagcol + (uint32_t)(c - 1) * TX);
              const bool lo_const = (a >= ((c - 1) << 5)) ? (fl_lo & 2u) != 0 : (fl_lo & 1u) != 0;
              if ((fl_hi & 1u) && lo_const && ln.fval(i0) == ln.fval(i0 - 1)) continue;
            }
            const int alo = max(a, (c - half) << 5);           // the run's rows inside the two groups
            const int bhi = min(b, min(n, (c + half) << 5));
            int av = prev_vertex<TX>(ln, i0, alo);
            int bv = next_vertex<TX>(ln, i0 - 1, bhi);
            if (av < 0 || bv < 0) continue;
            int ap = prev_vertex<TX>(ln, av, alo);
            int bn = next_vertex<TX>(ln, bv, bhi);
            float fa = ln.fval(av), fb = ln.fval(bv);
            float fap = ap >= 0 ? ln.fval(ap) : 0.0f, fbn = bn >= 0 ? ln.fval(bn) : 0.0f;
            for (;;) {
              if (ap >= 0 && (IntHull ? vertex_hidden_int(ap, fap, av, fa, bv, fb, w2i)
                                      : vertex_hidden(ap, fap, av, fa, bv, fb, w2d))) {   // A's top is hidden
                ln.drop(av);
                av = ap; fa = fap;
                ap = prev_vertex<TX>(ln, av, alo);
                if (ap >= 0) fap = ln.fval(ap);
                continue;
              }
              if (bn >= 0 && (IntHull ? vertex_hidden_int(av, fa, bv, fb, bn, fbn, w2i)
                                      : vertex_hidden(av, fa, bv, fb, bn, fbn, w2d))) {   // B's first is hidden
                ln.drop(bv);
                bv = bn; fb = fbn;
                bn = next_vertex<TX>(ln, bv, bhi);
                if (bn >= 0) fbn = ln.fval(bn);
                continue;
              }
              break;
            }
          }
        }
        if (!__syncthreads_or(more)) break;                    // (the barrier of the round)
      }
    }

    // ============ stage 3: outputs of the crossing segments, ONE loop over their rows per chunk ============
    if (live) {
      for (int c = chunk0; c < nchunks; c += chunk_step) {
        const int i0 = c << 5;
        const int rows = min(32, n - i0);
        const uint32_t rowmask = rows == 32 ? 0xffffffffu : ((1u << rows) - 1u);
        const uint32_t wstart = lds_u32(startcol + (uint32_t)c * ROW);
        const uint32_t wzero = Epilogue ? lds_u32(zerocol + (uint32_t)c * ROW) : 0u;
        const bool entering = !(wstart & 1u);                             // only possible for c > 0
        bool leaving = false;
        if (i0 + 32 < n) leaving = !(lds_u32(startcol + (uint32_t)(c + 1) * ROW) & 1u);
        if (!entering && !leaving) continue;
        const uint32_t wreal = wstart & rowmask;
        const int s2 = 31 - __clz(wreal | 1u);                            // first row of the last segment
        const uint32_t ent_mask = entering ? (wreal ? ((1u << (__ffs(wreal) - 1)) - 1u) : rowmask) : 0u;
        const uint32_t lea_mask = (leaving && wreal) ? (0xffffffffu << s2) : 0u;

        // the runs of the two segments: [a_ent, b_ent) came in from below, [i0 + s2, b_up) leaves above
        int a_ent = 0, b_up = n;
        if (use_nz) {                  // nearest chunks with a run start, from the line's chunk mask
          const uint32_t nzw = lds_u32_volatile(nzcol);
          const uint32_t below = entering ? (nzw & ((1u << c) - 1u)) : 0u;
          const uint32_t above = leaving ? (nzw & (0xfffffffeu << c)) : 0u;
          if (below) {
            const int cc = 31 - __clz(below);
            a_ent = (cc << 5) + 31 - __clz(lds_u32(startcol + (uint32_t)cc * ROW));
          }
          if (above) {
            const int cc = __ffs(above) - 1;
            b_up = min(n, (cc << 5) + __ffs(lds_u32(startcol + (uint32_t)cc * ROW)) - 1);
          }
        } else {
          if (entering) {
            for (int cc = c - 1; cc >= 0; --cc) {
              const uint32_t ws = lds_u32(startcol + (uint32_t)cc * ROW);
              if (ws) { a_ent = (cc << 5) + 31 - __clz(ws); break; }
            }
          }
          if (leaving) {
            for (int cc = c + 1; cc < nchunks; ++cc) {
              const uint32_t ws = lds_u32(startcol + (uint32_t)cc * ROW);
              if (ws) { b_up = min(n, (cc << 5) + __ffs(ws) - 1); break; }
            }
          }
        }
        const int b_ent = wreal ? (i0 + __ffs(wreal) - 1) : (leaving ? b_up : min(n, i0 + 32));
        const bool cst_ent = ent_mask && (all_const || run_is_constant<TX>(ln, cflagcol, a_ent, b_ent));
        const bool cst_lea = lea_mask && (all_const || run_is_constant<TX>(ln, cflagcol, i0 + s2, b_up));

        // one straight loop per crossing segment (the rows of a segment are adjacent), running addresses
        for (int seg = 0; seg < 2; ++seg) {
          const uint32_t mask = seg ? lea_mask : ent_mask;
          if (!mask) continue;
          const int rlo = __ffs(mask) - 1, rhi = 32 - __clz(mask);      // rows [rlo, rhi) of the chunk
          const int a = seg ? i0 + s2 : a_ent, b = seg ? b_up : b_ent;
          const bool cst = seg ? cst_lea : cst_ent;
          const bool lo_b = a > 0 || border_lo, hi_b = b < n || border_hi, bg = (wzero >> rlo) & 1u;
          uint32_t sq_lo = sq_t + (uint32_t)(i0 + rlo - a + 1) * 4u;   // sq[i - a + 1]
          uint32_t sq_hi = sq_t + (uint32_t)(b - i0 - rlo) * 4u;       // sq[b - i]
          char* dst = line0 + (size_t)(i0 + rlo) * pitch;
          if (cst) {
            // a constant run: out = min(f, border terms) (solid objects, blocky labels, background).
            // The run's one value against the smallest border terms these rows can see (those of the
            // rows nearest to a and to b): when it is not above them every row keeps its value, and as
            // the pass works in place nothing has to be stored at all
            uint32_t f_at = ln.f + (uint32_t)(i0 + rlo) * ROW;
            const float f0 = lds_f32(f_at);
            const float lo_min = lo_b ? lds_f32(sq_lo) : inf;
            const float hi_min = hi_b ? lds_f32(sq_t + (uint32_t)(b - i0 - rhi + 1) * 4u) : inf;
            if (f0 <= fminf(lo_min, hi_min)) {
              if (!Epilogue) continue;
              const float v = finish_value(f0, bg, flags);
              if (__float_as_uint(v) == __float_as_uint(f0)) continue;
              for (int r = rlo; r < rhi; ++r) { *reinterpret_cast<float*>(dst) = v; dst += pitch; }
              continue;
            }
  #pragma unroll 4
            for (int r = rlo; r < rhi; ++r) {
              float best = lds_f32(f_at);
              if (lo_b) best = fminf(best, lds_f32(sq_lo));
              if (hi_b) best = fminf(best, lds_f32(sq_hi));
              if (Epilogue) best = finish_value(best, bg, flags);
              *reinterpret_cast<float*>(dst) = best;
              f_at += ROW; sq_lo += 4u; sq_hi -= 4u; dst += pitch;
            }
            continue;
          }
          HullWalk w;
          walk_begin<TX>(w, ln, i0 + rlo, a, b, w2);
          for (int i = i0 + rlo; i < i0 + rhi; ++i) {
            float best = inf;
            if (w.v >= 0) {
              best = __fmaf_rn(w2, __fmul_rn(w.dv, w.dv), w.fv);
              while (w.v1 >= 0) {
                const float cand = __fmaf_rn(w2, __fmul_rn(w.dv1, w.dv1), w.fv1);
                if (!(cand <= best)) break;
                if (cand == best && !tie_not_above(w2, w.dv1, w.fv1, w.dv, w.fv)) break;
                best = cand; w.v = w.v1; w.fv = w.fv1; w.dv = w.dv1;
                walk_advance<TX>(w, ln, i);
              }
              w.dv += 1.0f; w.dv1 += 1.0f;
            }
            if (lo_b) best = fminf(best, lds_f32(sq_lo));
            if (hi_b) best = fminf(best, lds_f32(sq_hi));
            if (Epilogue) best = finish_value(best, bg, flags);             // a run has one label
            *reinterpret_cast<float*>(dst) = best;
            sq_lo += 4u; sq_hi -= 4u; dst += pitch;
          }
        }
      }
    }
    if constexpr (kGrouped) {
      if (rb.refresh) refresh_settled(rb, f, g, outer, inner0, n);
    }
    // (kGrouped) the next tile's TMA and stage 0 overwrite the tile, the words and the chunk mask: every
    // thread must be done with them
  } while (kGrouped && next_group_tile(todo, phase));
}

// ---------------------------------------------------------------------------------------
// Later-axis pass for lines too long for a shared-memory tile (more than 4096 voxels), and for
// passes whose candidate sums w2 * d^2 + f are not all exact in double (decided by the host).
// Same arithmetic as the tile kernel; distances from `dbl_from` on go through double: 4096, whose
// square is not exact in float32, or 0 for the inexact passes.  The double sum rounded once to
// float32 is the reference's evaluation (src/edt.hpp:232); the single fused multiply-add equals it
// only when the double sum is exact.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ float parabola_at(float w2, int d, float height, int dbl_from = 4096) {
  if (d < dbl_from) {
    const float e = (float)d;
    return __fmaf_rn(w2, __fmul_rn(e, e), height);
  }
  const double e = (double)d;
  return (float)__dadd_rn(__dmul_rn((double)w2, e * e), (double)height);
}

// One thread per line, lanes on adjacent lines (coalesced while the lanes stay in step).  Each
// run of equal labels gets the classic lower-envelope scan (build the hull, then read it out),
// O(n) per line, with the vertex stack in a global scratch volume `hull` laid out like f (entry
// k of the run that starts at row a lives at row a + k of the same line) and everything read
// through L1/L2.  Out of place (fin -> fout), so no synchronisation is needed.
// Sites: also write each voxel's site code (see kSiteNone) to `codes`, laid out like fout.
template <int Bytes, bool Sites = false>
__global__ void __launch_bounds__(128)
later_axis_long_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels,
                       const float* __restrict__ fin, float* __restrict__ fout, int* __restrict__ hull,
                       LineGeom g, float w2, int border_lo, int border_hi, int flags, int dbl_from,
                       int* __restrict__ codes) {
  using LT = typename LabelOf<Bytes>::type;
  const int64_t lines_per_outer = g.inner_count;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= lines_per_outer * g.outer_count) return;
  const int64_t outer = gid / lines_per_outer;
  const int64_t base = outer * g.outer_stride + (gid - outer * lines_per_outer);
  const int64_t ls = g.line_stride;
  const int n = g.n;
  const float inf = __int_as_float(0x7f800000);
  const double w2d = (double)w2;

  int a = 0;
  while (a < n) {
    const LT mine = labels[base + (int64_t)a * ls];
    int b = a + 1;
    while (b < n && labels[base + (int64_t)b * ls] == mine) ++b;
    const bool lo_border = a > 0 || border_lo;
    const bool hi_border = b < n || border_hi;

    // ---- build: hull[a + k] = position of the k-th vertex ----
    int top = -1, q = 0, p = 0;
    float fq = 0.0f, fp = 0.0f;
    for (int r = a; r < b; ++r) {
      const float fr = fin[base + (int64_t)r * ls];
      if (!(fr < inf)) continue;                         // +inf: not a site
      while (top >= 1 && vertex_hidden(p, fp, q, fq, r, fr, w2d)) {
        --top;
        q = p; fq = fp;
        if (top >= 1) {
          p = hull[base + (int64_t)(a + top - 1) * ls];
          fp = fin[base + (int64_t)p * ls];
        }
      }
      ++top;
      hull[base + (int64_t)(a + top) * ls] = r;
      p = q; fp = fq;
      q = r; fq = fr;
    }

    // ---- read out ----
    int k = 0, v = 0, v1 = 0;
    float fv = inf, fv1 = inf;
    if (top >= 0) { v = hull[base + (int64_t)a * ls]; fv = fin[base + (int64_t)v * ls]; }
    if (top >= 1) { v1 = hull[base + (int64_t)(a + 1) * ls]; fv1 = fin[base + (int64_t)v1 * ls]; }
    // The walk compares the candidates as double sums, not rounded to float32: rounded, they are
    // only weakly unimodal along the hull, and a step taken on a rounded tie can pass the
    // minimiser for good.  (Exact wherever w2 d^2 + f is, see launch_later.)
    for (int i = a; i < b; ++i) {
      float best = inf;
      if (top >= 0) {
        const double dv = (double)abs(i - v);
        double bestd = __dadd_rn(__dmul_rn(w2d, dv * dv), (double)fv);
        while (k < top) {
          const double d1 = (double)abs(i - v1);
          const double cand = __dadd_rn(__dmul_rn(w2d, d1 * d1), (double)fv1);
          if (!(cand <= bestd)) break;
          bestd = cand; ++k; v = v1; fv = fv1;
          if (k < top) { v1 = hull[base + (int64_t)(a + k + 1) * ls]; fv1 = fin[base + (int64_t)v1 * ls]; }
        }
        best = parabola_at(w2, abs(i - v), fv, dbl_from);
      }
      if constexpr (Sites) {
        // a border term is the distance to the voxel (or face) just outside the run, on this line
        int site = top >= 0 ? v : kSiteNone;
        if (lo_border) {
          const float c = parabola_at(w2, i - a + 1, 0.0f);
          if (c < best) { best = c; site = site_direct(a - 1); }
        }
        if (hi_border) {
          const float c = parabola_at(w2, b - i, 0.0f);
          if (c < best) { best = c; site = site_direct(b); }
        }
        codes[base + (int64_t)i * ls] = best < inf ? site : kSiteNone;
      } else {
        if (lo_border) best = fminf(best, parabola_at(w2, i - a + 1, 0.0f));
        if (hi_border) best = fminf(best, parabola_at(w2, b - i, 0.0f));
      }
      fout[base + (int64_t)i * ls] = finish_value(best, mine == 0, flags);
    }
    a = b;
  }
}

}  // namespace edtb200
