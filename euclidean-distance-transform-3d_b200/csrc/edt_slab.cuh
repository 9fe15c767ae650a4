// Z-slab decomposition across GPUs, one call per step (host side: edtb200_slab_step).
//
// Every rank owns a contiguous Z slab.  X and Y passes are slab-local.  The Z pass of a slab runs
// with its interior faces open, and the neighbours' rows of the runs that cross a face are folded
// in afterwards by face_fixup_kernel (edt_kernels.cuh).  What a neighbour needs from this rank
// -- per face: the face plane of labels, the length of the face-touching run of every (x,y) line,
// and the first / last `halo` planes of the Y-pass distances -- is published in a staging buffer
// in CUDA symmetric memory that the neighbours map over NVLink:
//
//   slab_stage_kernel   ONE kernel after the Y pass copies all of that for both faces into this
//                       rank's staging set (own HBM), and its last CTA tells both neighbours that
//                       step k is ready by a release store of k into THEIR flag word (a remote
//                       NVLink write);
//   slab_fixup_kernel   ONE kernel after the Z pass, both faces: each CTA first waits (acquire
//                       loads of its own flag word, local HBM) until the neighbour behind its face
//                       has published step k, then reads the neighbour's staging set IN PLACE over
//                       NVLink -- only the few planes within reach of the face values.
//
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

// blockIdx.y = face (0 low, 1 high; faces without a neighbour are skipped).  One thread per (x,y)
// line: `halo` planes of distances, the face label and the length m of the face-touching run
// (capped at halo + 1 = "longer than the halo, or spanning the slab"), as face_runs_kernel.
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
    const int64_t row0 = face ? (int64_t)(nz - 1) : 0;
    const int64_t dir = face ? -1 : 1;
    const LT lab0 = labels[row0 * plane + q];
    ldst[q] = lab0;
    int m = 1;
    const int limit = min(nz, halo + 1);
    while (m < limit && labels[(row0 + dir * m) * plane + q] == lab0) ++m;
    if (m > halo || m >= nz) m = halo + 1;
    mdst[q] = (unsigned char)m;
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

// One face of line q, as face_fixup_kernel does it, reading the neighbour's set over NVLink.
template <int Bytes>
__device__ __forceinline__ void
slab_fold_face(const typename LabelOf<Bytes>::type* __restrict__ labels, float* __restrict__ f, int64_t plane,
               int64_t q, int nz, int halo, float w2, int high_face, const unsigned char* __restrict__ nb,
               SlabStageLayout L, int flags, int* __restrict__ status) {
  using LT = typename LabelOf<Bytes>::type;
  // the neighbour's set: for my low face its HIGH-face data, for my high face its LOW-face data
  const LT* nb_label = reinterpret_cast<const LT*>(nb + (high_face ? L.lab_lo : L.lab_hi));
  const unsigned char* nb_m = nb + (high_face ? L.m_lo : L.m_hi);
  const float* nb_f = reinterpret_cast<const float*>(nb + (high_face ? L.f_lo : L.f_hi));
  const int H = halo;

  const int64_t row0 = high_face ? (int64_t)(nz - 1) : 0;
  const int64_t dir = high_face ? -1 : 1;
  const LT lab0 = labels[row0 * plane + q];
  const bool background = lab0 == 0;
  if (background && !(flags & kZeroLabel)) return;            // plain EDT: background stays 0
  const bool same = nb_label[q] == lab0;
  const int m_raw = same ? (int)nb_m[q] : 0;
  const bool unseen = m_raw > H;                              // the run goes on behind the halo
  const int m = min(m_raw, H);                                // neighbour rows of this run that we hold
  const bool negative = (flags & kNegate) && background;
  // the neighbour's rows of this run, read ONCE over NVLink (every row of the walk below needs them
  // again), and only those within reach of the face row's value: deeper rows of this slab reach
  // no further into the neighbour (sqrt of the result is 1-Lipschitz along the run)
  constexpr int kSiteCap = 32;
  float sites[kSiteCap];
  int held = 0;
  {
    const float cur0 = fabsf(f[row0 * plane + q]);
    const float reach0 = (flags & kSqrt) ? cur0 * cur0 * 1.000001f : cur0;
    while (held < min(m, kSiteCap) && parabola_at(w2, 1 + held, 0.0f, 0) <= reach0) {
      sites[held] = nb_f[(high_face ? (int64_t)held : (int64_t)(H - 1 - held)) * plane + q];
      ++held;
    }
  }
  // candidates, stop rule and stores as in face_fixup_kernel (edt_kernels.cuh)
  for (int j = 0; j < nz; ++j) {
    const int64_t at = (row0 + dir * j) * plane + q;
    if (j > 0 && labels[at] != lab0) break;                   // end of the run inside this slab
    const float cur = fabsf(f[at]);
    // a site at distance d costs at least w2 * d^2: strictly beyond the current value's reach it
    // is strictly above the row's exact value, and stays so on every later row
    const float reach = (flags & kSqrt) ? cur * cur * 1.000001f : cur;
    float best = unseen ? CUDART_INF_F : parabola_at(w2, j + 1 + m, 0.0f, 0);
    for (int r = 0; r < m; ++r) {
      if (parabola_at(w2, j + 1 + r, 0.0f, 0) > reach) break;
      const float height = r < held ? sites[r] : nb_f[(high_face ? (int64_t)r : (int64_t)(H - 1 - r)) * plane + q];
      best = fminf(best, parabola_at(w2, j + 1 + r, height, 0));
    }
    if (flags & kSqrt) best = __fsqrt_rn(best);
    if (unseen) {
      float bound = parabola_at(w2, j + H, 0.0f, 0);
      if (flags & kSqrt) bound = __fsqrt_rn(bound);
      if (!(fminf(best, cur) <= bound)) atomicOr(status, 1);
    }
    if (best > cur) break;                                    // no outside site helps from here on
    if (best < cur) f[at] = negative ? -best : best;
  }
}

// Both faces in one launch; waits for the neighbours' staging sets of `step` and then folds them
// in.  One thread per (x,y) line folds the low face and THEN the high face: a run that spans the
// slab is walked from both ends over the same rows, and the second walk must see the first one's
// stores (the NCCL path's two launches give the same order).
// *status: bit 0 = halo too shallow for this volume (see face_fixup_kernel), bit 1 = a
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
  if (has_lo) slab_fold_face<Bytes>(labels, f, plane, q, nz, halo, w2, 0, set_lo_peer, L, flags, status);
  if (has_hi) slab_fold_face<Bytes>(labels, f, plane, q, nz, halo, w2, 1, set_hi_peer, L, flags, status);
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
