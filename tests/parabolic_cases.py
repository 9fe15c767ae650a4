"""Parabolic erosion and dilation (edt_b200.parabolic_erode / _dilate, include/edt_b200.h) restated in numpy.

Each pass is a brute-force O(n^2) minimum per line: every candidate w2 * (i-j)^2 + g(j) formed in
float64 (w2 = float32(w * w), the square (i-j)^2 converted to float64), rounded once to float32, and the
sample itself for j == i.  Passes run along x, y, z -- x being the last numpy axis of a C-ordered array and
the first of an F-ordered one, as for edt().  NaN is read as +inf (never a site), -0.0 as +0.0; dilation
is -erosion(-f) with the same rules, and every zero result is +0.0.

`defect` plants one mistake so that the tests can show their comparisons notice it: "w2_double" (w2
rounded in float64 instead of float32) and "negzero" (-0.0 kept as it is).

The value generators make the families the GPU tests run: integers, uniform floats, floats of random sign
over exponents 2^-40 .. 2^40, values above 2^24, +-inf / NaN / -0.0, lines of +inf only and single -inf
samples, and near-tie lines whose two lowest candidates straddle a float32 rounding midpoint by a few
float64 ulps (near_tie_line).
"""
import numpy as np

INF = np.float32(np.inf)


def _w2(w, defect=None):
  if defect == "w2_double":
    return np.float64(w) * np.float64(w)
  with np.errstate(over="ignore"):
    return np.float64(np.float32(w) * np.float32(w))


def _load(g, defect=None):
  g = np.array(g, dtype=np.float32)
  g[np.isnan(g)] = INF
  if defect != "negzero":
    g[g == 0] = np.float32(0.0)
  return g


def line_pass(lines, w, defect=None):
  """One pass over the rows of a 2-D float32 array (lines along the last axis)."""
  lines = np.asarray(lines, np.float32)
  L, n = lines.shape
  w2 = _w2(w, defect)
  if not np.isfinite(w2) or n <= 1 or L == 0:
    return lines.copy()
  d = np.arange(n, dtype=np.int64)
  out = np.empty_like(lines)
  rows = max(1, min(n, (1 << 22) // n))                 # output rows i per block
  for i0 in range(0, n, rows):
    i = d[i0:i0 + rows]
    P = w2 * ((i[:, None] - d[None, :]) ** 2).astype(np.float64)  # P[i, j]
    step = max(1, (1 << 23) // P.size)
    for s in range(0, L, step):
      c = (P[None, :, :] + lines[s:s + step, None, :].astype(np.float64)).astype(np.float32)   # c[l, i, j]
      c[:, i - i0, i] = lines[s:s + step, i0:i0 + rows]
      out[s:s + step, i0:i0 + rows] = c.min(axis=2)
  return out


def _axis_pass(g, axis, w, defect):
  moved = np.moveaxis(g, axis, -1)
  shape = moved.shape
  res = line_pass(moved.reshape(-1, shape[-1]), w, defect).reshape(shape)
  return np.moveaxis(res, -1, axis)


def erode(f, anisotropy=None, order="C", defect=None, stacked=False):
  """The erosion of f (any real dtype) whose memory order is `order`: passes along the x-fastest axes.
  stacked: the slowest axis in memory indexes volumes and takes no pass."""
  g = _load(f, defect)
  nd = g.ndim
  axes = list(range(nd))
  if stacked:
    axes = axes[1:] if order == "C" else axes[:-1]
  w = (1.0,) * len(axes) if anisotropy is None else tuple(np.atleast_1d(np.asarray(anisotropy, np.float64)))
  assert len(w) == len(axes)
  weight = dict(zip(axes, w))
  for axis in (reversed(axes) if order == "C" else axes):
    g = _axis_pass(g, axis, weight[axis], defect)
  return g


def dilate(f, anisotropy=None, order="C", defect=None, stacked=False):
  neg = -np.asarray(f, np.float32)
  g = -erode(neg, anisotropy, order, defect, stacked)
  if defect != "negzero":
    g[g == 0] = np.float32(0.0)
  return g


def restate(op, f, anisotropy=None, order="C", defect=None, stacked=False):
  return (erode if op == "erode" else dilate)(f, anisotropy, order, defect, stacked)


def same_bits(a, b):
  a = np.asarray(a, np.float32)
  b = np.asarray(b, np.float32)
  return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ---- value families -------------------------------------------------------------------------------------

FAMILIES = ("integers", "uniform", "wide", "big", "special", "empty_lines", "neg_inf", "near_tie")

# Lines on which a double evaluation of the hull predicates gets the sign wrong, so that only the exact
# fallback gives the right result.  At CANCEL_W = 2^30 (w2 = 2^60 exactly):
#   read-out  [-2^60, 1] -> [-2^60, +0]: at row 1, f_b - f_a - w2 D = 1 + 2^60 - 2^60 = 1 > 0 keeps the
#             vertex at 0 (candidate 0), but 1 + 2^60 rounds to 2^60 in double, which reads as a tie and
#             moves to the vertex at 1 (candidate 1.0)
#   hull      [-2^60, -1, -2^60] stays as it is: E = 2 (-1) + 2^60 + 2^60 - 2^60 * 2 = -2 < 0 keeps the
#             middle vertex, but in double the -2 is lost and E reads 0, which drops it (row 1 would be 0)
CANCEL_W = 2.0 ** 30
CANCEL_CASES = (([-2.0 ** 60, 1.0], [-2.0 ** 60, 0.0]), ([-2.0 ** 60, -1.0, -2.0 ** 60], [-2.0 ** 60, -1.0, -2.0 ** 60]))


def cancel_line(n, case, at):
  """A line of n samples, +inf but for CANCEL_CASES[case]'s samples from `at`."""
  src = CANCEL_CASES[case][0]
  f = np.full(n, np.inf, np.float32)
  f[at:at + len(src)] = src
  return f


NEAR_TIE_W = 8.0


def near_tie_line(n, rng):
  """A line for the weight NEAR_TIE_W = 8 (w2 = 64) where, at some row i, the site p = 33 rows away has
  the candidate M = 64 * 513^2 + 1, a float32 rounding midpoint that rounds down (to even), and the site
  q = 513 rows away has M + 2^-23, just above it, which rounds up: only the true minimiser gives the right
  float32.  Lines too short for that get a pair of sites one float32 ulp apart around a row instead."""
  f = np.full(n, np.float32(2.0 ** 40))
  p, q = 33, 513
  M = 64 * q * q + 1
  if n > q + p + 1:
    i = int(rng.integers(p, n - q))
    f[i - p] = np.float32(M - 64 * p * p)                 # 16773121 < 2^24: an exact float32
    f[i + q] = np.float32(1.0 + 2.0 ** -23)
    assert float(f[i - p]) == M - 64 * p * p
    assert float(f[i - p]) + 64 * p * p == M and float(f[i + q]) + 64 * q * q == M + 2.0 ** -23
    return f
  j = int(rng.integers(0, n)) if n else 0
  if 0 < j < n - 1:
    f[j - 1] = np.float32(1.0)
    f[j + 1] = np.nextafter(np.float32(1.0), np.float32(2.0))
  return f


def values(family, shape, rng):
  size = int(np.prod(shape))
  if family == "integers":
    v = rng.integers(-50, 200, size).astype(np.float32)
  elif family == "uniform":
    v = rng.uniform(-3.0, 5.0, size).astype(np.float32)
  elif family == "wide":
    v = (rng.choice([-1.0, 1.0], size) * 2.0 ** rng.uniform(-40, 40, size)).astype(np.float32)
  elif family == "big":
    v = (2.0 ** 24 + rng.integers(0, 1 << 20, size) * rng.choice([1.0, 3.0, 7.0], size)).astype(np.float32)
  elif family == "special":
    v = rng.uniform(-10, 10, size).astype(np.float32)
    pick = rng.random(size)
    v[pick < 0.1] = np.inf
    v[(pick >= 0.1) & (pick < 0.15)] = np.nan
    v[(pick >= 0.15) & (pick < 0.25)] = -0.0
    v[(pick >= 0.25) & (pick < 0.3)] = 0.0
    v[(pick >= 0.3) & (pick < 0.31)] = -np.inf
  elif family == "empty_lines":
    v = np.full(size, np.inf, np.float32)
    v[rng.random(size) < 0.01] = rng.uniform(0, 100)
  elif family == "neg_inf":
    v = rng.uniform(0, 100, size).astype(np.float32)
    v[int(rng.integers(0, size))] = -np.inf
  elif family == "near_tie":
    n = int(shape[-1])
    v = np.concatenate([near_tie_line(n, rng) for _ in range(size // n)]) if n else np.zeros(0, np.float32)
  else:
    raise ValueError(family)
  return v.reshape(shape)
