// edt_slab.cuh -- the Z-slab decomposition across GPUs (see distributed.py): every kernel that
// couples neighbouring slabs.
//
// Every rank owns a contiguous Z slab.  X and Y passes are slab-local.  The Z pass of a slab runs
// with its interior faces open, and the neighbours' rows of the runs that cross a face are folded
// in afterwards.  What a neighbour needs from this rank -- per face: the face plane of labels, the
// length of the face-touching run of every (x,y) line, and the first / last `halo` planes of the
// Y-pass distances -- reaches it by one of two paths.  Both compute the run lengths with
// face_run_length and fold a face into one line with fold_face, so they give the same result.
//
// NCCL path (one C call per launch; distributed.py moves the arrays between the ranks):
//   face_runs_kernel    one face: the run lengths, and a flag when a foreground run is longer than
//                       the halo;
//   face_fixup_kernel   one face: fold_face on every line, from the arrays the neighbour sent.
//                       The low face is launched before the high face.
//
// Fused step (host side: edtb200_slab_step, one call per step): the arrays are published in a
// staging buffer in CUDA symmetric memory that the neighbours map over NVLink:
//   slab_stage_kernel   ONE kernel after the Y pass copies all of that for both faces into this
//                       rank's staging set (own HBM), and its last CTA tells both neighbours that
//                       step k is ready by a release store of k into THEIR flag word (a remote
//                       NVLink write);
//   slab_fixup_kernel   ONE kernel after the Z pass, both faces: each CTA first waits (acquire
//                       loads of its own flag word, local HBM) until the neighbour behind its face
//                       has published step k, then reads the neighbour's staging set IN PLACE over
//                       NVLink -- only the few planes within reach of the face values.
// No host synchronisation and no collective call is involved; compute and the peer transfers are
// ordered by the flag words alone.  Two staging sets alternate by step parity: set p of step k is
// rewritten at step k+2, after this rank's step-(k+1) fix-up has seen the neighbours' step-(k+1)
// flags, which they raise only after their step-k fix-up (the last reader of set p) is done.
#pragma once
#include "edt_kernels.cuh"

namespace edtb200 {

// Byte layout of one rank's symmetric buffer; identical on every rank.
struct SlabStageLayout {
  size_t f_lo, f_hi, lab_lo, lab_hi, m_lo, m_hi;   // offsets inside one staging set
  size_t set_bytes;                                // size of one set (two sets alternate)
  size_t flag_from_lo, flag_from_hi, counter;      // offsets from the buffer start (after both sets)
  size_t total_bytes;
};

__host__ __device__ inline SlabStageLayout slab_stage_layout(int64_t plane, int label_bytes, int halo) {
  SlabStageLayout L;
  size_t off = 0;
  auto take = [&off](size_t bytes) { const size_t at = off; off += (bytes + 255) / 256 * 256; return at; };
  L.f_lo = take((size_t)halo * plane * 4);
  L.f_hi = take((size_t)halo * plane * 4);
  L.lab_lo = take((size_t)plane * label_bytes);
  L.lab_hi = take((size_t)plane * label_bytes);
  L.m_lo = take((size_t)plane);
  L.m_hi = take((size_t)plane);
  L.set_bytes = off;
  L.flag_from_lo = 2 * L.set_bytes;
  L.flag_from_hi = L.flag_from_lo + 64;
  L.counter = L.flag_from_hi + 64;
  L.total_bytes = L.counter + 64;
  return L;
}

__device__ __forceinline__ void st_release_sys_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// ---------------------------------------------------------------------------------------
// The fold.  The Z pass of a slab has no border term at an interior face; the voxels of the
// neighbouring slab are folded in afterwards as extra candidates for the runs that touch the face:
//   * neighbour label differs: the face is a run border -> one zero-height site at distance 1;
//   * neighbour label equal  : the neighbour's part of the run (m <= halo rows, it must end inside
//     the neighbour's slab) contributes its rows as sites, plus the zero-height site behind it.
// Every such site lies outside the slab, so against the slab-local envelope its parabola only
// gets worse (by at least 2*w2 per row) as rows move away from the face.  Every candidate is the
// double sum w2 * d^2 + f rounded once to float32, the reference's evaluation.  The walk along a
// column stops at the first row where the best outside candidate is STRICTLY above the row's
// value: rounding is monotone, so that row's exact outside minimum is above its exact inside one,
// and the gap only widens further on.  A rounded tie proves nothing (the exact difference may
// still be negative and round lower a row later), so the walk goes on over ties; it stores only
// values strictly below the current one.
// Values are compared after the pass's epilogue: sqrt is monotone and the sign of a run is
// fixed, so min() commutes with both.
// ---------------------------------------------------------------------------------------

// z of the face plane in this slab's own order
__device__ __forceinline__ int64_t face_row(int nz, int high_face) { return high_face ? (int64_t)(nz - 1) : 0; }

// Length of the run of equal labels that touches the face on line q, whose face label is lab0:
// 1..halo, or halo + 1 = "longer than the halo, or spanning the slab".
template <typename LT>
__device__ __forceinline__ int face_run_length(const LT* __restrict__ labels, int64_t plane, int64_t q, int nz,
                                               int high_face, int halo, LT lab0) {
  const int64_t row0 = face_row(nz, high_face);
  const int64_t dir = high_face ? -1 : 1;
  int m = 1;
  const int limit = min(nz, halo + 1);
  while (m < limit && labels[(row0 + dir * m) * plane + q] == lab0) ++m;
  return (m > halo || m >= nz) ? halo + 1 : m;
}

// Fold the neighbour's sites into the rows of line q that belong to the run touching the face.
//   nb_label : the neighbour's face plane of labels        nb_m : its face_run_length per line
//   nb_f     : `halo` planes of the neighbour's distances AFTER its second-axis pass, in the
//              neighbour's own z order (for the low face these are its LAST planes)
// When the neighbour's part of the run is longer than the halo (nb_m = halo + 1) its first halo
// rows are still folded in, and the sites behind them -- unseen, at distance >= j + 1 + halo from
// row j, so never cheaper than w2 * (j + 1 + halo)^2 -- are ruled out by VALUE: if the combined
// result of a row does not exceed that bound nothing unseen can beat it.  sqrt of the result is
// 1-Lipschitz along the run (in units of w), so the bound holding at the face row implies it for
// every deeper row; it is tested (with one row of slack against rounding) on every row the walk
// visits, and bit 0 of *verdict (which may be NULL) is raised when it fails -- the caller then
// needs a deeper halo or the exact fallback.
// The first SiteCap rows within reach are cached; rows past them are read again where needed, so
// the cache size changes the memory traffic, not the result.
template <int Bytes, int SiteCap>
__device__ __forceinline__ void
fold_face(const typename LabelOf<Bytes>::type* __restrict__ labels, float* __restrict__ f, int64_t plane, int64_t q,
          int nz, int halo, float w2, int high_face, const typename LabelOf<Bytes>::type* __restrict__ nb_label,
          const unsigned char* __restrict__ nb_m, const float* __restrict__ nb_f, int flags,
          int* __restrict__ verdict) {
  using LT = typename LabelOf<Bytes>::type;
  const int64_t row0 = face_row(nz, high_face);
  const int64_t dir = high_face ? -1 : 1;
  // row r of the run in the neighbour (r = 0 next to the face), in the neighbour's own z order
  auto nb_site = [&](int r) { return nb_f[(high_face ? (int64_t)r : (int64_t)(halo - 1 - r)) * plane + q]; };
  const LT lab0 = labels[row0 * plane + q];
  const bool background = lab0 == 0;
  if (background && !(flags & kZeroLabel)) return;            // plain EDT: background stays 0
  const bool same = nb_label[q] == lab0;
  const int m_raw = same ? (int)nb_m[q] : 0;
  const bool unseen = m_raw > halo;                           // the run goes on behind the halo
  const int m = min(m_raw, halo);                             // neighbour rows of this run that we hold
  const bool negative = (flags & kNegate) && background;
  // the neighbour's rows of this run, read ONCE (they may live in a peer GPU's memory): every row
  // of the walk below needs them again.  Only those within reach of the face row's value are
  // fetched: deeper rows of this slab reach no further into the neighbour (Lipschitz again).
  float sites[SiteCap];
  int held = 0;
  {
    const float cur0 = fabsf(f[row0 * plane + q]);
    const float reach0 = (flags & kSqrt) ? cur0 * cur0 * 1.000001f : cur0;
    while (held < min(m, SiteCap) && parabola_at(w2, 1 + held, 0.0f, 0) <= reach0) {
      sites[held] = nb_site(held);
      ++held;
    }
  }
  for (int j = 0; j < nz; ++j) {
    const int64_t at = (row0 + dir * j) * plane + q;
    if (j > 0 && labels[at] != lab0) break;                   // end of the run inside this slab
    const float cur = fabsf(f[at]);
    // a site at distance d costs at least w2 * d^2: strictly beyond the current value's reach it
    // is strictly above the row's exact value, and stays so on every later row
    const float reach = (flags & kSqrt) ? cur * cur * 1.000001f : cur;
    // best outside site for row j: neighbour rows r = 0..m-1 at distance j + 1 + r, then (if the
    // run ends there) the zero-height site behind them at distance j + 1 + m
    float best = unseen ? CUDART_INF_F : parabola_at(w2, j + 1 + m, 0.0f, 0);
    for (int r = 0; r < m; ++r) {
      if (parabola_at(w2, j + 1 + r, 0.0f, 0) > reach) break;
      const float height = r < held ? sites[r] : nb_site(r);
      best = fminf(best, parabola_at(w2, j + 1 + r, height, 0));
    }
    if (flags & kSqrt) best = __fsqrt_rn(best);
    if (unseen) {
      float bound = parabola_at(w2, j + halo, 0.0f, 0);
      if (flags & kSqrt) bound = __fsqrt_rn(bound);
      if (!(fminf(best, cur) <= bound) && verdict) atomicOr(verdict, 1);
    }
    if (best > cur) break;                                    // no outside site helps from here on
    if (best < cur) f[at] = negative ? -best : best;
  }
}

// ---- NCCL path: one launch per face ----

// m[q] = face_run_length of every line q of the sx*sy plane; *overflow is raised if any foreground
// run is longer than the halo.
template <int Bytes>
__global__ void __launch_bounds__(256)
face_runs_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, int64_t plane, int nz, int high_face,
                 int H, int zero_is_label, uint8_t* __restrict__ m_out, int* __restrict__ overflow) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= plane) return;
  const auto lab0 = labels[face_row(nz, high_face) * plane + q];
  const int m = face_run_length(labels, plane, q, nz, high_face, H, lab0);
  if (m > H && (lab0 != 0 || zero_is_label)) *overflow = 1;
  m_out[q] = (uint8_t)m;
}

// fold_face on every line q of the sx*sy plane, from the neighbour's arrays as received.
template <int Bytes>
__global__ void __launch_bounds__(256)
face_fixup_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, float* __restrict__ f,
                  int64_t plane, int nz, int high_face, int H, float w2,
                  const typename LabelOf<Bytes>::type* __restrict__ nb_label,
                  const uint8_t* __restrict__ nb_m, const float* __restrict__ nb_f, int flags,
                  int* __restrict__ inexact) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= plane) return;
  fold_face<Bytes, 128>(labels, f, plane, q, nz, H, w2, high_face, nb_label, nb_m, nb_f, flags, inexact);
}

// ---- fused step: both faces in one launch each ----

// blockIdx.y = face (0 low, 1 high; faces without a neighbour are skipped).  One thread per (x,y)
// line: `halo` planes of distances, the face label and its face_run_length.
template <int Bytes>
__global__ void __launch_bounds__(256)
slab_stage_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, const float* __restrict__ f,
                  int64_t plane, int nz, int halo, int has_lo, int has_hi, unsigned char* __restrict__ set,
                  SlabStageLayout L, unsigned long long step, unsigned long long* flag_in_lo_peer,
                  unsigned long long* flag_in_hi_peer, unsigned int* counter) {
  using LT = typename LabelOf<Bytes>::type;
  pdl_launch_dependents();                 // the Z pass may start staging its labels under this kernel
  const int face = blockIdx.y;
  const bool active = face == 0 ? has_lo != 0 : has_hi != 0;
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (active && q < plane) {
    float* fdst = reinterpret_cast<float*>(set + (face ? L.f_hi : L.f_lo));
    LT* ldst = reinterpret_cast<LT*>(set + (face ? L.lab_hi : L.lab_lo));
    unsigned char* mdst = set + (face ? L.m_hi : L.m_lo);
    const int64_t first = face ? (int64_t)(nz - halo) : 0;       // planes in this slab's own z order
    for (int h = 0; h < halo; ++h) fdst[(int64_t)h * plane + q] = f[(first + h) * plane + q];
    const LT lab0 = labels[face_row(nz, face) * plane + q];
    ldst[q] = lab0;
    mdst[q] = (unsigned char)face_run_length(labels, plane, q, nz, face, halo, lab0);
  }
  // the last CTA of the grid publishes the step to both neighbours
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int total = gridDim.x * gridDim.y;
    if (atomicAdd(counter, 1u) == total - 1u) {
      *counter = 0u;
      __threadfence_system();
      if (has_lo && flag_in_lo_peer) st_release_sys_u64(flag_in_lo_peer, step);
      if (has_hi && flag_in_hi_peer) st_release_sys_u64(flag_in_hi_peer, step);
    }
  }
}

// Both faces in one launch; waits for the neighbours' staging sets of `step` and then folds them
// in.  One thread per (x,y) line folds the low face and THEN the high face: a run that spans the
// slab is walked from both ends over the same rows, and the second walk must see the first one's
// stores (the NCCL path's two launches give the same order).
// *status: bit 0 = halo too shallow for this volume (see fold_face), bit 1 = a
// neighbour never published the step (time-out).
template <int Bytes>
__global__ void __launch_bounds__(256)
slab_fixup_kernel(const typename LabelOf<Bytes>::type* __restrict__ labels, float* __restrict__ f, int64_t plane,
                  int nz, int halo, float w2, int has_lo, int has_hi, const unsigned char* __restrict__ set_lo_peer,
                  const unsigned char* __restrict__ set_hi_peer, SlabStageLayout L, unsigned long long step,
                  const unsigned long long* flag_from_lo, const unsigned long long* flag_from_hi, int flags,
                  int* __restrict__ status) {
  if (!has_lo && !has_hi) return;
  // launched with programmatic stream serialization right behind the Z pass: the CTAs become
  // resident during its last wave, wait for the neighbours' flags, and only then for the Z pass
  __shared__ int ready;
  if (threadIdx.x == 0) {
    int ok = 1;
    for (int face = 0; face < 2 && ok; ++face) {
      if (face == 0 ? !has_lo : !has_hi) continue;
      const unsigned long long* flag = face ? flag_from_hi : flag_from_lo;
      ok = 0;
      for (long long spin = 0; spin < (1ll << 25); ++spin) {      // a few seconds, then give up
        if (ld_acquire_sys_u64(flag) >= step) { ok = 1; break; }
        __nanosleep(64);
      }
    }
    ready = ok;
  }
  __syncthreads();
  pdl_wait_for_previous_grid();            // f holds the Z pass's results from here on
  if (!ready) {
    if (threadIdx.x == 0) atomicOr(status, 2);
    return;
  }
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= plane) return;
  using LT = typename LabelOf<Bytes>::type;
  // the neighbour's set: for my low face its HIGH-face data, for my high face its LOW-face data.
  // The layout goes in by value on purpose: with L read straight from the kernel parameter, ptxas
  // (CUDA 12.9) spills more in slab_fixup_kernel<1>, <2> and <4>.
  auto fold = [&](int high_face, const unsigned char* nb, SlabStageLayout layout) {
    fold_face<Bytes, 32>(labels, f, plane, q, nz, halo, w2, high_face,
                         reinterpret_cast<const LT*>(nb + (high_face ? layout.lab_lo : layout.lab_hi)),
                         nb + (high_face ? layout.m_lo : layout.m_hi),
                         reinterpret_cast<const float*>(nb + (high_face ? layout.f_lo : layout.f_hi)), flags, status);
  };
  if (has_lo) fold(0, set_lo_peer, L);
  if (has_hi) fold(1, set_hi_peer, L);
}

// ---- Z slabs <-> Y slabs (the transposition fallback of the slab split) ----
// A rank's slab (zc, sy, row) is cut along y into `n` parts (part i = rows start[i] .. start[i+1]);
// packed, part i is one contiguous block (zc, c_i, row) -- what rank i receives in ONE message --
// and the blocks follow one another in rank order.  ONE launch moves the whole slab either way
// (Unpack = the inverse map, for the way back), 16 bytes per thread and access when the rows allow.
struct SlabParts {
  int n;
  long long start[65];       // start[n] = sy
};

template <bool Unpack>
__global__ void __launch_bounds__(256)
slab_pack_kernel(const unsigned char* __restrict__ src, unsigned char* __restrict__ dst, long long zc, long long sy,
                 long long rowbytes, int vec16, SlabParts parts) {
  const long long rows = zc * sy;
  for (long long row = blockIdx.x; row < rows; row += gridDim.x) {
    const long long z = row / sy, y = row - z * sy;
    int i = 0;
    while (i + 1 < parts.n && y >= parts.start[i + 1]) ++i;
    const long long s = parts.start[i], c = parts.start[i + 1] - s;
    const long long packed = (zc * s + z * c + (y - s)) * rowbytes, plain = row * rowbytes;
    const unsigned char* a = src + (Unpack ? packed : plain);
    unsigned char* b = dst + (Unpack ? plain : packed);
    if (vec16) {
      for (long long k = (long long)threadIdx.x * 16; k < rowbytes; k += (long long)blockDim.x * 16)
        *reinterpret_cast<uint4*>(b + k) = *reinterpret_cast<const uint4*>(a + k);
    } else {
      for (long long k = threadIdx.x; k < rowbytes; k += blockDim.x) b[k] = a[k];
    }
  }
}

}  // namespace edtb200
