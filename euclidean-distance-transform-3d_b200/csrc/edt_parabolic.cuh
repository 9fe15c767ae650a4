// edt_parabolic.cuh -- parabolic erosion and dilation: the distance transform of a sampled function
// (edtb200_parabolic, include/edt_b200.h).
//
// One pass along an axis replaces every sample g(i) of a line by
//   min( g(i), min_{j != i} fl32(fl64(fl64(w2 * fl64((i-j)^2)) + g(j))) ),   w2 = fl32(w * w),
// the caller's samples read with NaN as +inf and -0.0 as +0.0 (negated first for a dilation, whose
// store negates back).  Rounding is monotone, so the minimum of the rounded candidates is the rounded
// value of the candidate whose REAL value w2 (i-j)^2 + g(j) is least -- wherever w2 (i-j)^2 is exact in
// double, which holds for every line of at most kParabolicExactN samples ((i-j)^2 < 2^29, w2 has 24
// significant bits).  Such lines take the lower envelope of those parabolas (Felzenszwalb-Huttenlocher)
// with exact predicates: a double evaluation with an error bound, and an exact sum of TwoSum /
// FMA-TwoProduct terms when the bound cannot decide the sign.  Longer lines take a brute-force minimum
// over every candidate formed exactly as the definition forms it.
//
// Kernels:
//   parabolic_tile_kernel<false, S>  Y / Z passes, lines of at most kParabolicTileN: a CTA of S warps
//       stages 32 adjacent lines (lanes along x, cp.async, coalesced), warp s the rows of segment s;
//       each lane builds its segment's hull in place over its staged column, and after a barrier reads
//       out its segment's rows as the minimum over the S segment hulls, row by row (coalesced).
//   parabolic_tile_kernel<true, S>   X pass, rows of at most kParabolicTileN: the CTA stages 32 whole
//       rows transposed into shared memory (pitch 33: no bank conflicts either way), segments as above,
//       and results leave through one 32 x 33 transpose buffer per warp, coalesced.
//       S = kParabolicWarps = 4 by default: at 512^3 it is 1.1-1.9x faster than one warp per CTA (one
//       or two warps per SM) and at 1024^3 2.6x (records/h100/parabolic_bench.txt).
//   parabolic_long_kernel          lines longer than kParabolicTileN, up to kParabolicExactN: one
//       thread per line, the hull in device scratch (8 bytes per sample of the lines in flight).
//   parabolic_brute_kernel         lines longer than kParabolicExactN: one thread per output sample.
//   parabolic_copy_kernel          a pass whose w2 overflows float32: every j != i candidate is +inf,
//       so the pass only folds NaN and -0.0 (and negates for a dilation).
// Each value is read once and written once per pass on the tile kernels, which need no device memory
// beyond their input and output; in place (in == out) every kernel but the brute-force one reads a
// line wholly before writing it, and that one reads a copy.
//
// Sites (edtb200_parabolic_sites): separate instances (Sites = true, and parabolic_copy_sites_kernel)
// also write every sample's winning row to a code plane, kSiteNone where the line has no candidate; the
// values are those of the other instances bit for bit.  On lines of at most kParabolicExactN samples the
// row is the least REAL minimiser: the read-out moves to the next hull vertex only when it is strictly
// lower (pb_below, exact), and the tile kernels merge their segments in order by the same exact test.
// Longer lines take the least j with the least double candidate.  The X tile kernel sends the codes
// through a second transpose buffer per warp, so its rows of 1009 to 1024 samples take 2 warps, not 4.
#pragma once
#include "edt_host.h"

#include <cuda_pipeline.h>

#include <cmath>
#include <cstdlib>

namespace edtb200 {

constexpr int kParabolicTileN = 1024;     // longest line of the tile kernels
constexpr int kParabolicExactN = 23170;   // longest line whose squared distances stay below 2^29
constexpr int kParabolicWarps = 4;        // warps per tile CTA (segments per line)

// A caller's sample as the passes see it, and a result as the caller sees it.
__device__ __forceinline__ float pb_in(float v, bool dilate) {
  const float x = dilate ? -v : v;
  if (x != x) return __int_as_float(0x7f800000);
  return x == 0.0f ? 0.0f : x;
}
__device__ __forceinline__ float pb_out(float r, bool dilate) {
  const float x = dilate ? -r : r;
  return x == 0.0f ? 0.0f : x;
}

__device__ __forceinline__ void pb_two_sum(double a, double b, double& s, double& e) {
  s = __dadd_rn(a, b);
  const double bb = __dsub_rn(s, a);
  e = __dadd_rn(__dsub_rn(a, __dsub_rn(s, bb)), __dsub_rn(b, bb));
}

// Sign of the exact sum of M doubles: Shewchuk's grow-expansion, whose last non-zero component
// carries the sign.  No term here can overflow (every term is below 2^200).
template <int M>
__device__ __noinline__ int pb_exact_sign(const double (&t)[M]) {
  double h[M];
  int n = 0;
  for (int m = 0; m < M; ++m) {
    double q = t[m];
    for (int i = 0; i < n; ++i) {
      double s, e;
      pb_two_sum(q, h[i], s, e);
      h[i] = e;
      q = s;
    }
    h[n++] = q;
  }
  for (int i = n - 1; i >= 0; --i)
    if (h[i] != 0.0) return h[i] > 0.0 ? 1 : -1;
  return 0;
}

// Whether hull vertex k is hidden by its neighbours j < k < l: with F_m = f_m + w2 m^2, the point
// (k, F_k) lies on or above the chord from (j, F_j) to (l, F_l), i.e. with A = k - j, B = l - k
//   E = (A+B) f_k - B f_j - A f_l - w2 A B (A+B) >= 0.
// (A+B) f_k, B f_j and A f_l are exact in double (15 + 24 bits), as is x = w2 A B (52 bits);
// x (A+B) = p + e exactly by an FMA.
__device__ __forceinline__ bool pb_hidden(float fj, int j, float fk, int k, float fl, int l, double w2) {
  const double A = (double)(k - j), B = (double)(l - k), S = A + B;
  const double t1 = __dmul_rn(S, (double)fk), t2 = -__dmul_rn(B, (double)fj), t3 = -__dmul_rn(A, (double)fl);
  const double x = __dmul_rn(w2, __dmul_rn(A, B));
  const double p = __dmul_rn(x, S);
  const double e = __fma_rn(x, S, -p);
  const double s = __dsub_rn(__dadd_rn(__dadd_rn(t1, t2), t3), p);
  // three roundings of at most 2^-53 of the magnitudes each, and the term e left out
  const double bound = __dadd_rn(__dmul_rn(fabs(t1) + fabs(t2) + fabs(t3) + fabs(p), 0x1p-50), fabs(e));
  if (s > bound) return true;
  if (s < -bound) return false;
  const double t[5] = {t1, t2, t3, -p, -e};
  return pb_exact_sign<5>(t) >= 0;
}

// Whether vertex b > a is at least as low as a at row i:
//   f_b + w2 (i-b)^2 <= f_a + w2 (i-a)^2  <=>  f_b - f_a - w2 D <= 0,  D = (i-a)^2 - (i-b)^2,
// |D| < 2^29, so w2 D is exact in double.
__device__ __forceinline__ bool pb_not_above(float fa, int a, float fb, int b, int i, double w2) {
  const double q = __dmul_rn(w2, (double)(b - a) * (double)(2 * i - a - b));
  const double s = __dsub_rn(__dsub_rn((double)fb, (double)fa), q);
  const double bound = __dmul_rn(fabs((double)fa) + fabs((double)fb) + fabs(q), 0x1p-50);
  if (s < -bound) return true;
  if (s > bound) return false;
  const double t[3] = {(double)fb, -(double)fa, -q};
  return pb_exact_sign<3>(t) <= 0;
}

// Whether vertex b is strictly lower than vertex a at row i (any a, b): pb_not_above without the tie,
// so that a read-out or a merge that moves only on it keeps the least minimiser.
__device__ __forceinline__ bool pb_below(float fa, int a, float fb, int b, int i, double w2) {
  const double q = __dmul_rn(w2, (double)(b - a) * (double)(2 * i - a - b));
  const double s = __dsub_rn(__dsub_rn((double)fb, (double)fa), q);
  const double bound = __dmul_rn(fabs((double)fa) + fabs((double)fb) + fabs(q), 0x1p-50);
  if (s < -bound) return true;
  if (s > bound) return false;
  const double t[3] = {(double)fb, -(double)fa, -q};
  return pb_exact_sign<3>(t) < 0;
}

// The candidate of vertex (f, v) at row i, rounded as the definition rounds it (d^2 w2 exact).
__device__ __forceinline__ float pb_value(float f, int v, int i, double w2) {
  const int d = i - v;
  return __double2float_rn(__dadd_rn(__dmul_rn(w2, (double)(d * d)), (double)f));
}

// The lower envelope of one line: push() takes the samples (already through pb_in) onto a stack of
// (height, position) whose slot m lives at sf[m * fs] / si[m * is] -- slot m never runs ahead of the
// sample being read, so the stack may overwrite the samples it was staged over -- and at(i) reads the
// minimum at row i, for i = 0, 1, ... in order.
template <class Index>
struct PbHull {
  float* sf;
  Index* si;
  int fs, is;
  double w2;
  int top = -1;
  bool neg = false;
  int k = 0, a = 0, b = 0;
  float fa = 0.0f, fb = 0.0f;

  __device__ void push(float f, int j) {
    if (f == __int_as_float(0x7f800000)) return;            // +inf (and NaN): not a site
    if (f == -__int_as_float(0x7f800000)) { neg = true; return; }
    while (top >= 1 && pb_hidden(sf[(top - 1) * fs], (int)si[(top - 1) * is], sf[top * fs], (int)si[top * is], f, j, w2))
      --top;
    ++top;
    sf[top * fs] = f;
    si[top * is] = (Index)j;
  }
  __device__ void start() {
    if (top < 0) return;
    fa = sf[0];
    a = (int)si[0];
    if (top > 0) { fb = sf[fs]; b = (int)si[is]; }
  }
  __device__ float at(int i) {
    if (neg) return -__int_as_float(0x7f800000);             // a -inf sample: the whole line is -inf
    if (top < 0) return __int_as_float(0x7f800000);           // no site
    while (k < top && pb_not_above(fa, a, fb, b, i, w2)) {
      ++k;
      fa = fb;
      a = b;
      if (k < top) { fb = sf[(k + 1) * fs]; b = (int)si[(k + 1) * is]; }
    }
    return pb_value(fa, a, i, w2);
  }
  // at(i) with its site: the read-out stays on a vertex that ties with the next one, so the site is the
  // least minimiser (the hull never drops it: a vertex hidden at E = 0 ties with a lower position).
  // first_neg: the first -inf position pushed (kSiteNone: none), the site of a -inf line.
  __device__ float at_site(int i, int first_neg, int* site) {
    if (neg) { *site = first_neg; return -__int_as_float(0x7f800000); }
    if (top < 0) { *site = kSiteNone; return __int_as_float(0x7f800000); }
    while (k < top && pb_below(fa, a, fb, b, i, w2)) {
      ++k;
      fa = fb;
      a = b;
      if (k < top) { fb = sf[(k + 1) * fs]; b = (int)si[(k + 1) * is]; }
    }
    *site = a;
    return pb_value(fa, a, i, w2);
  }
};

// The site-tracking read-out of a tile: the minimum at row i over the S segment hulls and its site.
// Segments are merged in order and a later one wins only when its REAL candidate is strictly lower
// (fminf of the rounded minima could not tell two different reals that round alike), so the site is
// the least minimiser of the line; an earlier -inf segment keeps its first -inf position.
template <int S>
__device__ __forceinline__ float pb_merge_sites(PbHull<uint16_t> (&r)[S], const int (&first_neg)[S], int i,
                                                double w2, int* site) {
  float v = r[0].at_site(i, first_neg[0], site);
  float bf = r[0].fa;                 // the winning vertex, when it is one (not -inf, not none)
  for (int q = 1; q < S; ++q) {
    int sq;
    const float vq = r[q].at_site(i, first_neg[q], &sq);
    if (sq == kSiteNone || v == -__int_as_float(0x7f800000)) continue;
    if (vq == -__int_as_float(0x7f800000) || *site == kSiteNone || pb_below(bf, *site, r[q].fa, sq, i, w2)) {
      v = vq;
      *site = sq;
      bf = r[q].fa;
    }
  }
  return v;
}

// Shared memory of one tile CTA of S warps: the staged samples / stack heights, the stack positions,
// each segment's stack top and -inf flag and, for the X pass, one 32 x 33 transpose buffer per warp.
// With sites, the X pass has a second transpose buffer per warp for the site codes.
__host__ __device__ constexpr size_t pb_tile_smem(int n, bool rows, int S, bool sites = false) {
  return (size_t)n * (rows ? 33 : 32) * 4 + (size_t)n * 32 * 2 + (size_t)S * 32 * 8 +
         (rows ? (size_t)S * 32 * 33 * 4 * (sites ? 2 : 1) : 0);
}

// rows = false: lines of g (Y / Z pass), a tile = 32 adjacent lines of one outer index.
// rows = true:  rows of n contiguous samples, outer_count of them outer_stride apart (X pass); a
//               tile = 32 consecutive rows.
// S warps per CTA: warp s stages segment s of every line (rows [s*seg, (s+1)*seg), seg = ceil(n / S))
// and its lane builds that segment's hull in place; after a barrier each lane reads out the rows of its
// own segment as the minimum over the S segment hulls.  The minimum of the rounded minima of the
// segments is the rounded minimum of the line, so the result does not depend on S; S trades a shorter
// serial hull build (n / S per lane) and S times the warps per SM for S candidates per output row.
// Sites: also write every sample's site code (its winning row, or kSiteNone) to `codes`, laid out like
// `out`: each segment's read-out keeps its least minimiser and pb_merge_sites merges them exactly.
template <bool Rows, int S, bool Sites = false>
__global__ void __launch_bounds__(32 * S)
parabolic_tile_kernel(const float* in, float* out, LineGeom g, double w2, bool dilate, int64_t tiles, int* codes) {
  extern __shared__ __align__(16) unsigned char pb_smem[];
  constexpr int fp = Rows ? 33 : 32;
  const int n = g.n, lane = threadIdx.x & 31, s = threadIdx.x >> 5;
  const int seg = (n + S - 1) / S, lo = min(n, s * seg), hi = min(n, lo + seg);
  float* sf = reinterpret_cast<float*>(pb_smem);
  uint16_t* si = reinterpret_cast<uint16_t*>(pb_smem + (size_t)n * fp * 4);
  int* tops = reinterpret_cast<int*>(pb_smem + (size_t)n * fp * 4 + (size_t)n * 64);
  int* negs = tops + S * 32;
  float* ob = reinterpret_cast<float*>(negs + S * 32) + s * 32 * 33;
  int* oc = reinterpret_cast<int*>(negs + S * 32) + (S + s) * 32 * 33;     // Sites, X pass: the codes' buffer
  const int64_t tpo = (g.inner_count + 31) >> 5;
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    int64_t base;
    bool on;
    if (Rows) {
      const int64_t r0 = t * 32;
      for (int r = 0; r < 32 && r0 + r < g.outer_count; ++r) {
        const float* row = in + (r0 + r) * g.outer_stride;
        for (int c = lo + lane; c < hi; c += 32) __pipeline_memcpy_async(&sf[c * 33 + r], row + c, 4);
      }
      on = r0 + lane < g.outer_count;
      base = (r0 + lane) * g.outer_stride;
    } else {
      const int64_t o = t / tpo, j = (t - o * tpo) * 32 + lane;
      on = j < g.inner_count;
      base = o * g.outer_stride + j;
      if (on)
        for (int i = lo; i < hi; ++i) __pipeline_memcpy_async(&sf[i * 32 + lane], in + base + i * g.line_stride, 4);
    }
    __pipeline_commit();
    __pipeline_wait_prior(0);
    __syncwarp();                     // the warp's lanes staged each other's columns of its segment
    PbHull<uint16_t> h{sf + lo * fp + lane, si + lo * 32 + lane, fp, 32, w2};
    int first_neg = kSiteNone;        // Sites: the segment's first -inf position
    if (on)
      for (int j = lo; j < hi; ++j) {
        const float v = pb_in(sf[j * fp + lane], dilate);
        if constexpr (Sites)
          if (first_neg == kSiteNone && v == -__int_as_float(0x7f800000)) first_neg = j;
        h.push(v, j);
      }
    tops[s * 32 + lane] = h.top;
    if constexpr (Sites) negs[s * 32 + lane] = first_neg;
    else negs[s * 32 + lane] = h.neg;
    __syncthreads();                  // every segment's hull is built
    PbHull<uint16_t> r[S];
    int rneg[S];
    for (int q = 0; q < S; ++q) {
      const int qlo = min(n, q * seg);
      r[q] = PbHull<uint16_t>{sf + qlo * fp + lane, si + qlo * 32 + lane, fp, 32, w2};
      r[q].top = tops[q * 32 + lane];
      if constexpr (Sites) {
        rneg[q] = negs[q * 32 + lane];
        r[q].neg = rneg[q] != kSiteNone;
      } else {
        r[q].neg = negs[q * 32 + lane] != 0;
      }
      r[q].start();
    }
    auto at = [&](int i) {
      float v = r[0].at(i);
      for (int q = 1; q < S; ++q) v = fminf(v, r[q].at(i));
      return pb_out(v, dilate);
    };
    if (Rows) {
      const int64_t r0 = t * 32;
      for (int c = lo; c < hi; c += 32) {
        for (int q = 0; q < 32 && c + q < hi; ++q) {
          if constexpr (Sites) {
            int site;
            ob[q * 33 + lane] = pb_out(pb_merge_sites<S>(r, rneg, c + q, w2, &site), dilate);
            oc[q * 33 + lane] = site;
          } else {
            ob[q * 33 + lane] = at(c + q);
          }
        }
        __syncwarp();
        if (c + lane < hi)
          for (int rr = 0; rr < 32 && r0 + rr < g.outer_count; ++rr) {
            out[(r0 + rr) * g.outer_stride + c + lane] = ob[lane * 33 + rr];
            if constexpr (Sites) codes[(r0 + rr) * g.outer_stride + c + lane] = oc[lane * 33 + rr];
          }
        __syncwarp();
      }
    } else if (on) {
      for (int i = lo; i < hi; ++i) {
        if constexpr (Sites) {
          int site;
          out[base + i * g.line_stride] = pb_out(pb_merge_sites<S>(r, rneg, i, w2, &site), dilate);
          codes[base + i * g.line_stride] = site;
        } else {
          out[base + i * g.line_stride] = at(i);
        }
      }
    }
    __syncthreads();                  // the next tile's staging overwrites every segment's hull
  }
}

// One thread per line of at most kParabolicExactN samples; stack slot m of thread `tid` at
// [m * threads + tid] of sf / si (coalesced across threads).  Lines: outer_count x inner_count.
// Sites: also the site codes, as parabolic_tile_kernel writes them.
template <bool Sites = false>
__global__ void __launch_bounds__(128)
parabolic_long_kernel(const float* in, float* out, LineGeom g, double w2, bool dilate, float* sf, int* si, int* codes) {
  const int64_t threads = (int64_t)gridDim.x * blockDim.x, tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t lines = g.outer_count * g.inner_count;
  for (int64_t l = tid; l < lines; l += threads) {
    const int64_t o = l / g.inner_count, base = o * g.outer_stride + (l - o * g.inner_count);
    PbHull<int> h{sf + tid, si + tid, (int)threads, (int)threads, w2};
    int first_neg = kSiteNone;
    for (int j = 0; j < g.n; ++j) {
      const float v = pb_in(in[base + j * g.line_stride], dilate);
      if constexpr (Sites)
        if (first_neg == kSiteNone && v == -__int_as_float(0x7f800000)) first_neg = j;
      h.push(v, j);
    }
    h.start();
    for (int i = 0; i < g.n; ++i) {
      if constexpr (Sites) {
        int site;
        out[base + i * g.line_stride] = pb_out(h.at_site(i, first_neg, &site), dilate);
        codes[base + i * g.line_stride] = site;
      } else {
        out[base + i * g.line_stride] = pb_out(h.at(i), dilate);
      }
    }
  }
}

// One thread per output sample of lines longer than kParabolicExactN: every candidate, formed as the
// definition forms it (fl64 of (i-j)^2, of its product with w2 and of the sum).  `in` is not `out`.
// Sites: the least j with the least double candidate (j == i: the sample itself), which rounds to the
// minimum of the rounded candidates; +inf samples are never sites.
template <bool Sites = false>
__global__ void __launch_bounds__(256)
parabolic_brute_kernel(const float* __restrict__ in, float* __restrict__ out, LineGeom g, double w2, bool dilate,
                       int* __restrict__ codes) {
  const int64_t total = g.outer_count * g.inner_count * (int64_t)g.n;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < total; v += (int64_t)gridDim.x * blockDim.x) {
    const int64_t l = v / g.n, i = v - l * g.n;
    const int64_t o = l / g.inner_count, base = o * g.outer_stride + (l - o * g.inner_count);
    if constexpr (Sites) {
      double best = __int_as_float(0x7f800000);
      int site = kSiteNone;
      for (int64_t j = 0; j < g.n; ++j) {
        const float f = pb_in(in[base + j * g.line_stride], dilate);
        if (f == __int_as_float(0x7f800000)) continue;
        const double d = (double)(i - j);
        const double c = j == i ? (double)f : __dadd_rn(__dmul_rn(w2, __dmul_rn(d, d)), (double)f);
        if (site == kSiteNone || c < best) {
          best = c;
          site = (int)j;
        }
      }
      out[base + i * g.line_stride] = pb_out(__double2float_rn(best), dilate);
      codes[base + i * g.line_stride] = site;
    } else {
      float best = pb_in(in[base + i * g.line_stride], dilate);
      for (int64_t j = 0; j < g.n; ++j) {
        if (j == i) continue;
        const double d = (double)(i - j);
        const float c = __double2float_rn(__dadd_rn(__dmul_rn(w2, __dmul_rn(d, d)),
                                                    (double)pb_in(in[base + j * g.line_stride], dilate)));
        best = fminf(best, c);
      }
      out[base + i * g.line_stride] = pb_out(best, dilate);
    }
  }
}

__global__ void __launch_bounds__(256)
parabolic_copy_kernel(const float* in, float* out, int64_t total, bool dilate) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = pb_out(pb_in(in[i], dilate), dilate);
}

// parabolic_copy_kernel with the site codes: every sample is its own site (its row, (i / stride) % n
// along lines of n samples `stride` apart), but +inf, which has none.
__global__ void __launch_bounds__(256)
parabolic_copy_sites_kernel(const float* in, float* out, int* codes, int64_t total, int64_t stride, int n,
                            bool dilate) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = pb_in(in[i], dilate);
    out[i] = pb_out(v, dilate);
    codes[i] = v == __int_as_float(0x7f800000) ? kSiteNone : (int)((i / stride) % n);
  }
}

namespace host {

// Lines in flight of parabolic_long_kernel: enough threads to fill the GPU, at most 1 GiB of stack.
inline int64_t pb_long_threads(int64_t lines, int n) {
  int64_t t = ((int64_t)1 << 30) / (8 * (int64_t)n);
  if (t < 4096) t = 4096;
  return t < lines ? t : lines;
}

int launch_parabolic_pass(const float* in, float* out, const LineGeom& g, bool rows, float w, bool dilate,
                          DeviceCache& dc, cudaStream_t stream, int* kernel, int* codes) {
  const float w2f = w * w;                     // rounded to float, as the definition rounds it
  const double w2 = (double)w2f;
  const int64_t lines = g.outer_count * g.inner_count, total = lines * (int64_t)g.n;
  if (total == 0) return 0;
  auto blocks_for = [&](int64_t work, int per) {
    int64_t b = (work + per - 1) / per;
    const int64_t cap = (int64_t)dc.sm_count * 16;
    return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
  };
  if (std::isinf(w2f)) {
    *kernel = 3;
    // lines are whole and cover the volume, so the pass is elementwise over it
    if (codes) {
      const int64_t stride = rows ? 1 : g.line_stride;       // the row of sample i is (i / stride) % n
      parabolic_copy_sites_kernel<<<blocks_for(total, 256), 256, 0, stream>>>(in, out, codes, total, stride, g.n,
                                                                              dilate);
    } else {
      parabolic_copy_kernel<<<blocks_for(total, 256), 256, 0, stream>>>(in, out, total, dilate);
    }
    CUDA_TRY(cudaGetLastError());
    return 0;
  }
  if (g.n <= kParabolicTileN) {
    *kernel = 0;
    // warps per CTA (segments per line): the default from records/h100/parabolic_bench.txt, or
    // EDTB200_PARABOLIC_WARPS = 1, 2 or 4 (an A/B switch for measurements); fewer where the shared
    // memory of S transpose buffers does not fit (with sites, X rows of more than 1008 samples take 2)
    int S = kParabolicWarps;
    if (const char* env = getenv("EDTB200_PARABOLIC_WARPS")) S = atoi(env);
    if (S != 1 && S != 2 && S != 4) return fail(EDTB200_EINVAL, "EDTB200_PARABOLIC_WARPS must be 1, 2 or 4 (got %d)", S);
    const bool sites = codes != nullptr;
    while (S > 1 && pb_tile_smem(g.n, rows, S, sites) > (size_t)dc.max_smem_optin) S >>= 1;
    const size_t smem = pb_tile_smem(g.n, rows, S, sites);
    if (smem > (size_t)dc.max_smem_optin) return fail(EDTB200_ELIMIT, "a parabolic tile of %d rows exceeds the shared memory", g.n);
    const int64_t tiles = rows ? (g.outer_count + 31) >> 5 : ((g.inner_count + 31) >> 5) * g.outer_count;
    const unsigned blocks = (unsigned)(tiles < ((int64_t)1 << 30) ? tiles : ((int64_t)1 << 30));
    auto go = [&](auto kern) {
      CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      kern<<<blocks, 32 * S, smem, stream>>>(in, out, g, w2, dilate, tiles, codes);
      CUDA_TRY(cudaGetLastError());
      return 0;
    };
    auto pick = [&](auto with_sites) {
      constexpr bool St = decltype(with_sites)::value;
      if (rows) return S == 1 ? go(parabolic_tile_kernel<true, 1, St>) : S == 2 ? go(parabolic_tile_kernel<true, 2, St>)
                                                                       : go(parabolic_tile_kernel<true, 4, St>);
      return S == 1 ? go(parabolic_tile_kernel<false, 1, St>) : S == 2 ? go(parabolic_tile_kernel<false, 2, St>)
                                                              : go(parabolic_tile_kernel<false, 4, St>);
    };
    return sites ? pick(std::true_type{}) : pick(std::false_type{});
  }
  if (g.n <= kParabolicExactN) {
    *kernel = 1;
    const int64_t threads = pb_long_threads(lines, g.n);
    const int64_t blocks = (threads + 127) / 128, slots = blocks * 128;
    Scratch stack;
    if (const int rc = stack.take(dc, (size_t)slots * (size_t)g.n * 8, stream, "the long lines' hull stacks")) return rc;
    float* sf = stack.get<float>();
    int* si = reinterpret_cast<int*>(sf + slots * (int64_t)g.n);
    if (codes) parabolic_long_kernel<true><<<(unsigned)blocks, 128, 0, stream>>>(in, out, g, w2, dilate, sf, si, codes);
    else parabolic_long_kernel<false><<<(unsigned)blocks, 128, 0, stream>>>(in, out, g, w2, dilate, sf, si, nullptr);
    CUDA_TRY(cudaGetLastError());
    return 0;
  }
  *kernel = 2;
  Scratch copy;
  const float* src = in;
  if (in == out) {
    // lines cover the volume from its first sample to its last
    const int64_t span = (g.outer_count - 1) * g.outer_stride + (g.inner_count - 1) + (int64_t)(g.n - 1) * g.line_stride + 1;
    if (const int rc = copy.take(dc, sizeof(float) * (size_t)span, stream, "the copy of the long lines")) return rc;
    CUDA_TRY(cudaMemcpyAsync(copy.get(), in, sizeof(float) * (size_t)span, cudaMemcpyDeviceToDevice, stream));
    src = copy.get<float>();
  }
  if (codes) parabolic_brute_kernel<true><<<blocks_for(total, 256), 256, 0, stream>>>(src, out, g, w2, dilate, codes);
  else parabolic_brute_kernel<false><<<blocks_for(total, 256), 256, 0, stream>>>(src, out, g, w2, dilate, nullptr);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace host
}  // namespace edtb200
