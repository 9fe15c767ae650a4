"""The window kernel of the bounded transforms (later_axis_window_kernel, edt_bounded.cuh) restated on the
CPU, for tests of one pass at a time (edtb200_pass_window), and adversarial lines for it.

  plan(w, d)     B and R of one later pass, in exact rational arithmetic: B is the largest float32 whose
                 value is at most the double d*d (the largest finite float32 when there is none above),
                 B+ the float32 after it, w2 = fl32(w * w), and R the largest r >= 0 with w2 r^2 < B+
                 exactly (capped at 2^62, which also stands for "no bound").
  window_pass    one pass by definition: for every row the least, over the WHOLE run of its label (not
                 just the window), of the rounded candidates fl32(fl64(w2) delta^2 + fl64(f_v)) and the
                 border terms fl32(w2 delta^2) where the run ends inside the line (at a face only with
                 border_lo / border_hi); +inf above B; then the epilogue (correctly rounded sqrt, the
                 sign of sdf on label 0).  A radius too small shows here as a difference.
  check_codes    the site codes the kernel writes, as the feature transform reads them: the winning
                 row, site_direct(row) = -2 - row for a border term, kSiteNone for +inf; where rounded
                 candidates tie any tied site is accepted.

Arrays are C-ordered (z, y, x) like oracle.pass_later takes them; a pass along axis 1 runs down y,
along axis 2 down z.  Every label is an ordinary label (background runs too), compared by all its bits.
"""
import math
from fractions import Fraction

import numpy as np

CAP = 1 << 62
SITE_NONE = -(1 << 31)
SQRT, SIGNED = 1, 2
WINDOW_ROWS = 64                       # kWindowRows: rows of a window tile
RADIUS_LIMIT = 128                     # kWindowRadiusLimit
F32_MAX_BITS = 0x7F7FFFFF


def f32_bits(k):
  return np.array([k], np.uint32).view(np.float32)[0]


def site_direct(row):
  return -2 - row


def plan(w, d):
  """(B as np.float32, R) of a later pass with weight w under max_distance d >= 0."""
  lim = d * d                                       # the double the library squares d into
  if lim >= float(f32_bits(F32_MAX_BITS)):
    bits = F32_MAX_BITS
  else:                                             # the largest float32 bits whose value is <= lim
    exact = Fraction(lim)
    lo, hi = 0, F32_MAX_BITS
    while lo < hi:
      mid = (lo + hi + 1) // 2
      if Fraction(float(f32_bits(mid))) <= exact:
        lo = mid
      else:
        hi = mid - 1
    bits = lo
  b = f32_bits(bits)
  with np.errstate(over="ignore"):
    w2 = np.float32(np.float32(w) * np.float32(w))
  if np.isinf(w2):
    return b, 0                                     # only r = 0 has w2 r^2 (= 0) below B+, even +inf
  if bits == F32_MAX_BITS or w2 == 0:
    return b, CAP                                   # B+ = +inf, or w2 = 0: every r qualifies
  above = Fraction(float(f32_bits(bits + 1)))
  q = above / Fraction(float(w2))                   # r^2 < q  <=>  r^2 <= floor((p - 1) / s)
  return b, min(CAP, math.isqrt((q.numerator - 1) // q.denominator))


def distance_for(w, radius):
  """A max_distance whose plan has exactly R = radius for weight w, and its B: d^2 = w2 radius^2 rounded
  to a float32 from above, so that a winner exactly R rows away lands on B."""
  w2 = float(np.float32(np.float32(w) * np.float32(w)))
  target = np.float32(w2 * radius * radius)
  if float(target) < w2 * radius * radius:
    target = np.nextafter(target, np.float32(np.inf))
  d = math.sqrt(float(target))
  for _ in range(8):                                # the double whose square is the target or just above
    if plan(w, d)[0] >= target:
      break
    d = math.nextafter(d, math.inf)
  b, r = plan(w, d)
  assert r == radius, (w, radius, d, r)
  return d, b


def _lines(a, axis):
  """(n, lines) view of a (z, y, x) array with the pass axis first."""
  along = 0 if axis == 2 else 1
  moved = np.moveaxis(np.asarray(a), along, 0)
  return np.ascontiguousarray(moved).reshape(moved.shape[0], -1)


def _unlines(lines, shape, axis):
  along = 0 if axis == 2 else 1
  moved_shape = (shape[along],) + tuple(s for i, s in enumerate(shape) if i != along)
  return np.ascontiguousarray(np.moveaxis(lines.reshape(moved_shape), 0, along))


def _runs(lab):
  """Per (row, line): the first row a of its run and the row b after it."""
  n = lab.shape[0]
  rows = np.arange(n).reshape(-1, 1)
  start = np.ones(lab.shape, bool)
  start[1:] = lab[1:] != lab[:-1]
  a = np.maximum.accumulate(np.where(start, rows, 0), axis=0)
  end = np.ones(lab.shape, bool)
  end[:-1] = lab[1:] != lab[:-1]
  b = np.minimum.accumulate(np.where(end, rows + 1, n)[::-1], axis=0)[::-1]
  return a, b


def _candidates(lab, f, w2, radius=None):
  """(n, n, lines): fl32(fl64(w2) (i - v)^2 + fl64(f_v)) for row i and sample v of i's run (and within
  `radius` rows of i, when given), else +inf."""
  n = lab.shape[0]
  a, b = _runs(lab)
  i = np.arange(n).reshape(-1, 1, 1)
  v = np.arange(n).reshape(1, -1, 1)
  same = (v >= a[:, None, :]) & (v < b[:, None, :])
  if radius is not None:
    same &= np.abs(i - v) <= radius
  with np.errstate(over="ignore", invalid="ignore"):
    c = (w2 * ((i - v) ** 2).astype(np.float64) + f.astype(np.float64)[None, :, :]).astype(np.float32)
  return np.where(same & ~np.isnan(c), c, np.float32(np.inf))


def _borders(lab, w2, lo, hi, radius=None):
  """(low term, high term) per (row, line): fl32(w2 delta^2) to the row just outside the run, +inf where
  the run reaches a face that is not a border (or, when `radius` is given, lies farther away)."""
  n = lab.shape[0]
  a, b = _runs(lab)
  i = np.arange(n).reshape(-1, 1)
  with np.errstate(over="ignore"):
    low = (w2 * ((i - a + 1) ** 2).astype(np.float64)).astype(np.float32)
    high = (w2 * ((b - i) ** 2).astype(np.float64)).astype(np.float32)
  low = np.where((a > 0) | bool(lo), low, np.float32(np.inf))
  high = np.where((b < n) | bool(hi), high, np.float32(np.inf))
  if radius is not None:
    low = np.where(i - a + 1 <= radius, low, np.float32(np.inf))
    high = np.where(b - i <= radius, high, np.float32(np.inf))
  return low, high


def _w2(w):
  with np.errstate(over="ignore"):
    return float(np.float32(np.float32(w) * np.float32(w)))


def pass_values(lab, f, axis, w, d, lo, hi, radius=None):
  """The pass before its epilogue: the least candidate or border term, +inf above B.  radius: only what
  lies within that many rows (a window; None: the whole run, the definition)."""
  lab_l, f_l = _lines(lab, axis), _lines(np.asarray(f, np.float32), axis)
  w2 = _w2(w)
  best = _candidates(lab_l, f_l, w2, radius).min(axis=1) if lab_l.size else np.zeros(lab_l.shape, np.float32)
  low, high = _borders(lab_l, w2, lo, hi, radius)
  best = np.minimum(best, np.minimum(low, high))
  b, _ = plan(w, d)
  best = np.where(best <= b, best, np.float32(np.inf)).astype(np.float32)
  return _unlines(best, np.shape(lab), axis)


def epilogue(values, lab, flags):
  out = np.asarray(values, np.float32).copy()
  if flags & SQRT:
    out = np.sqrt(out)
  if flags & SIGNED:
    out = np.where(np.asarray(lab) == 0, -out, out).astype(np.float32)
  return out


def window_pass(lab, f, axis, w, d, lo, hi, flags=0):
  """What edtb200_pass_window must write to fout (see the module's docstring)."""
  return epilogue(pass_values(lab, f, axis, w, d, lo, hi), lab, flags)


def check_codes(lab, f, axis, w, d, lo, hi, codes):
  """Assert the site codes of a pass: kSiteNone exactly where the pass is +inf, elsewhere a site of the
  row's own run (a sample row, or site_direct of the row just outside the run, a face only with the
  border flag) whose own candidate equals the pass value bit for bit."""
  values = _lines(pass_values(lab, f, axis, w, d, lo, hi), axis)
  lab_l, f_l, c = _lines(lab, axis), _lines(np.asarray(f, np.float32), axis), _lines(np.asarray(codes), axis)
  n = lab_l.shape[0]
  w2 = _w2(w)
  a, b = _runs(lab_l)
  rows = np.arange(n).reshape(-1, 1)
  none = c == SITE_NONE
  inf = np.isinf(values)
  assert np.array_equal(none, inf), "kSiteNone at %d rows, +inf at %d" % (none.sum(), inf.sum())
  direct = (c < 0) & ~none
  site = np.where(direct, -2 - c.astype(np.int64), c.astype(np.int64))
  in_run = (site >= a) & (site < b)
  sample_ok = ~direct & in_run
  border_ok = direct & (((site == a - 1) & ((a > 0) | bool(lo))) | ((site == b) & ((b < n) | bool(hi))))
  ok = none | sample_ok | border_ok
  assert ok.all(), "a site outside its run at (row, line) %s: code %d" % (
    tuple(np.argwhere(~ok)[0]), int(c[~ok][0]))
  delta2 = ((rows - site) ** 2).astype(np.float64)
  fs = np.take_along_axis(f_l, np.clip(site, 0, n - 1), axis=0).astype(np.float64)
  with np.errstate(over="ignore", invalid="ignore"):
    got = np.where(direct, w2 * delta2, w2 * delta2 + fs).astype(np.float32)
  bad = ~none & (got.view(np.uint32) != values.view(np.uint32))
  assert not bad.any(), "the site's candidate is not the pass value at (row, line) %s: %r vs %r (%d rows)" % (
    tuple(np.argwhere(bad)[0]), float(got[bad][0]), float(values[bad][0]), int(bad.sum()))


# ---- adversarial lines ---------------------------------------------------------------------------------

def labels(rng, kind, shape, axis, dtype):
  """Labels whose runs along `axis` are: the whole line, random lengths, single rows among long runs,
  or (8-byte labels) two values that differ only in their high 32 bits, alternating in runs."""
  n = shape[0] if axis == 2 else shape[1]
  if kind == "one_run":
    run = np.zeros(n, np.int64)
  elif kind == "runs":
    cuts = np.cumsum(rng.geometric(1.0 / max(2, n // 4), n))
    run = np.searchsorted(cuts, np.arange(n), side="right")
  elif kind == "specks":
    run = np.where(rng.random(n) < 0.08, 1 + np.arange(n) % 2, 0)
  else:
    raise ValueError(kind)
  along = run.reshape((-1, 1, 1) if axis == 2 else (1, -1, 1))
  offset = rng.integers(0, 2, tuple(1 if i == (0 if axis == 2 else 1) else s for i, s in enumerate(shape)))
  lab = np.broadcast_to((along + offset) % 3, shape).astype(np.uint64)
  if np.dtype(dtype).itemsize == 8:
    lab = np.where(lab == 2, np.uint64(1) | np.uint64(1 << 40), lab)     # 1 and 1 + 2^40: same low bits
  return np.ascontiguousarray(lab.astype(dtype))


PROFILES = ("sparse", "at_bound", "tile_edges", "border_ties", "real", "tiny")


def profile(rng, kind, shape, axis, w, radius, b):
  """float32 samples for a pass with weight w, radius R and bound B:
    sparse      mostly +inf, a few zero-height sites (one alone on a quarter of the lines): winners at every
                distance, R and R + 1 among them
    at_bound    heights B, the float32s either side of it, and +inf, over a few sites
    tile_edges  a zero-height site exactly R and R + 1 rows beyond the first and last row of every
                window tile, where the staged halo ends
    border_ties integer heights w2 (k^2 - j^2) that tie a sample at j rows with a border term at k rows
    real        real heights in [0, B]: inexact candidate sums
    tiny        a height of 2^-52 among real ones: candidate sums inexact in double"""
  n = shape[0] if axis == 2 else shape[1]
  along = 0 if axis == 2 else 1
  other = tuple(s for i, s in enumerate(shape) if i != along)
  lines = int(np.prod(other))
  w2 = _w2(w)
  f = np.full((n, lines), np.inf, np.float32)
  bf = float(b)
  if kind == "sparse":
    f[rng.random(f.shape) < max(0.02, 1.0 / max(1, 2 * radius + 1))] = 0.0
    alone = rng.random(lines) < 0.25                # lines with one site: rows exactly R and R + 1 from it
    f[:, alone] = np.inf
    f[rng.integers(0, max(1, n - radius), lines)[alone], np.flatnonzero(alone)] = 0.0
  elif kind == "at_bound":
    near = [bf, float(np.nextafter(b, np.float32(np.inf))), float(np.nextafter(b, np.float32(0)))]
    pick = rng.integers(0, 4, f.shape)
    f = np.where(pick < 3, np.array(near, np.float32)[np.minimum(pick, 2)], np.float32(np.inf))
    f[rng.random(f.shape) < 0.05] = 0.0
  elif kind == "tile_edges":
    for t0 in range(0, n, WINDOW_ROWS):
      for edge, step in ((t0, -1), (min(t0 + WINDOW_ROWS, n) - 1, 1)):
        for dist in (radius, radius + 1):
          r = edge + step * dist
          if 0 <= r < n:
            f[r, rng.random(lines) < 0.5] = 0.0
  elif kind == "border_ties":
    k = rng.integers(1, radius + 2, f.shape)
    j = rng.integers(0, 1 + np.maximum(k - 1, 0))
    f = (w2 * (k.astype(np.float64) ** 2 - j.astype(np.float64) ** 2)).astype(np.float32)
    f[rng.random(f.shape) < 0.3] = np.inf
  elif kind == "real":
    f = (rng.random(f.shape) * (bf if math.isfinite(bf) and bf > 0 else 1.0)).astype(np.float32)
    f[rng.random(f.shape) < 0.5] = np.inf
  elif kind == "tiny":
    f = (rng.random(f.shape) * 50.0).astype(np.float32)
    f[rng.random(f.shape) < 0.1] = 2.0 ** -52
    f[rng.random(f.shape) < 0.4] = np.inf
  else:
    raise ValueError(kind)
  moved_shape = (n,) + other
  return np.ascontiguousarray(np.moveaxis(f.reshape(moved_shape), 0, along))
