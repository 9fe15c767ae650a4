"""The sites of parabolic erosion and dilation (parabolic_erode / _dilate with return_indices=True,
edtb200_parabolic_sites in include/edt_b200.h) restated in numpy, on the values of parabolic_cases.py.

Each pass picks a site on every line among the candidates of the values' definition (j = i included, with
the sample itself):
  - lines of at most EXACT_N samples: the least j among the REAL minimisers of w2 (i-j)^2 + g(j).  The
    rounded candidates narrow the choice to the j whose rounded candidate is the minimum (rounding is
    monotone, so the real minimisers are among them); those few are compared exactly with Fraction.
  - longer lines: the least j among the minimisers of the float64 candidate, before its float32 rounding.
  - +inf (and NaN, read as +inf) is never a site; a line holding -inf takes its least -inf position;
    with w2 = +inf every sample is its own site; a voxel whose line has no candidate has none.
The sites compose as the feature transform's resolver composes them: q_z from the Z pass at p, q_y from
the Y pass at (p_x, p_y, q_z), q_x from the X pass at (p_x, q_y, q_z); no site is -1 in every coordinate.

`defect` plants one mistake so that the tests can show their comparisons notice it: "last" (the greatest
index among tied minimisers) and "rounded" (the least j among the rounded minima, with no exact
comparison).
"""
from fractions import Fraction

import numpy as np

import parabolic_cases as pc

EXACT_N = 23170          # longest line decided on real values (kParabolicExactN)
INF = np.float32(np.inf)


def _w2(w):
  return pc._w2(w)


def line_sites(lines, w, defect=None):
  """(values, sites) of one pass over the rows of a 2-D float32 array of loaded samples (no NaN, no
  -0.0; lines along the last axis).  The values are parabolic_cases.line_pass's."""
  lines = np.asarray(lines, np.float32)
  L, n = lines.shape
  w2 = _w2(w)
  real = lines != INF
  if L == 0 or n == 0 or not np.isfinite(w2):
    return lines.copy(), np.where(real, np.arange(n)[None, :], -1)
  values = np.empty_like(lines)
  sites = np.full((L, n), -1, np.int64)
  d = np.arange(n, dtype=np.int64)
  rows = max(1, min(n, (1 << 21) // n))
  for i0 in range(0, n, rows):
    i = d[i0:i0 + rows]
    P = w2 * ((i[:, None] - d[None, :]) ** 2).astype(np.float64)
    step = max(1, (1 << 22) // P.size)
    for s in range(0, L, step):
      g = lines[s:s + step]
      c64 = P[None, :, :] + g[:, None, :].astype(np.float64)            # c64[l, i, j]
      c64[:, i - i0, i] = g[:, i0:i0 + rows]
      c = c64.astype(np.float32)
      m = c.min(axis=2)
      values[s:s + step, i0:i0 + rows] = m
      ok = real[s:s + step, None, :]
      if n > EXACT_N:                                                    # the float64 candidates
        c64 = np.where(ok, c64, np.inf)
        best = c64.min(axis=2)
        tie = (c64 == best[..., None]) & ok
      else:
        tie = (c == m[..., None]) & ok
      has = tie.any(axis=2)
      first = np.argmax(tie, axis=2)
      last = n - 1 - np.argmax(tie[:, :, ::-1], axis=2)
      pick = last if defect == "last" else first
      if n <= EXACT_N and defect != "rounded":
        many = has & (first != last) & (m != -INF)
        for l, r in zip(*np.nonzero(many)):
          ii = i0 + int(r)
          js = np.flatnonzero(tie[l, r])
          gl = g[l]
          exact = [Fraction(float(w2)) * (ii - int(j)) ** 2 + Fraction(float(gl[j])) for j in js]
          low = min(exact)
          win = [int(j) for j, e in zip(js, exact) if e == low]
          pick[l, r] = win[-1] if defect == "last" else win[0]
      sites[s:s + step, i0:i0 + rows] = np.where(has, pick, -1)
  return values, sites


def _pass_axes(nd, order, stacked):
  """The array axes that take a pass, x first."""
  axes = list(range(nd))
  if stacked:
    axes = axes[1:] if order == "C" else axes[:-1]
  return axes[::-1] if order == "C" else axes


def _weights(nd, anisotropy, order, stacked):
  axes = list(range(nd))
  if stacked:
    axes = axes[1:] if order == "C" else axes[:-1]
  w = (1.0,) * len(axes) if anisotropy is None else tuple(np.atleast_1d(np.asarray(anisotropy, np.float64)))
  assert len(w) == len(axes)
  return dict(zip(axes, w))


def _loaded(op, f):
  return pc._load(-np.asarray(f, np.float32) if op == "dilate" else f)


def compose(shape, plane_of, order_axes, vol_axes):
  """indices (len(vol_axes),) + shape from the per-pass site planes plane_of[axis] (x pass first in
  order_axes), as the resolver follows them; -1 everywhere without a site."""
  P = np.indices(shape)
  q = {}
  none = np.zeros(shape, bool)
  for k in range(len(order_axes) - 1, -1, -1):
    a = order_axes[k]
    at = [P[b] for b in range(len(shape))]
    for later in order_axes[k + 1:]:
      at[later] = np.where(none, 0, q[later])
    got = plane_of[a][tuple(at)]
    none |= got < 0
    q[a] = got
  out = np.stack([np.where(none, -1, q[a]) for a in vol_axes]) if vol_axes else np.zeros((0,) + shape, np.int64)
  return out.astype(np.int32)


def restate(op, f, anisotropy=None, order="C", defect=None, stacked=False, line=line_sites):
  """(values, indices) of parabolic_erode / _dilate(f, anisotropy, return_indices=True) for an array of
  memory order `order`; `line(lines, w, defect)` gives one pass's (values, sites)."""
  g = _loaded(op, f)
  nd = g.ndim
  weight = _weights(nd, anisotropy, order, stacked)
  axes = _pass_axes(nd, order, stacked)
  planes = {}
  for a in axes:
    moved = np.moveaxis(g, a, -1)
    shp = moved.shape
    vals, s = line(moved.reshape(-1, shp[-1]), weight[a], defect)
    g = np.moveaxis(vals.reshape(shp), -1, a)
    planes[a] = np.moveaxis(s.reshape(shp), -1, a)
  if op == "dilate":
    g = -g
    g[g == 0] = np.float32(0.0)
  vol_axes = sorted(weight)
  return g, compose(g.shape, planes, axes, vol_axes)


def chain(op, f, indices, anisotropy=None, order="C", stacked=False):
  """The value at every p formed from f(q), q = indices[:, p]: the X pass's rounded candidate, then the
  Y pass's, then the Z pass's; +inf (-inf for dilation) where there is no site."""
  g = _loaded(op, f)
  nd = g.ndim
  weight = _weights(nd, anisotropy, order, stacked)
  vol_axes = sorted(weight)
  shape = g.shape
  idx = np.asarray(indices).astype(np.int64)
  none = idx[0] < 0 if len(vol_axes) else np.zeros(shape, bool)
  P = np.indices(shape)
  at = [P[b] for b in range(nd)]
  for k, a in enumerate(vol_axes):
    at[a] = np.where(none, 0, idx[k])
  v = g[tuple(at)].astype(np.float32)
  for a in _pass_axes(nd, order, stacked):
    dist = P[a] - at[a]
    w2 = _w2(weight[a])
    with np.errstate(invalid="ignore", over="ignore"):
      c = (w2 * (dist * dist).astype(np.float64) + v.astype(np.float64)).astype(np.float32)
    v = np.where(dist == 0, v, c)
  v = np.where(none, INF, v)
  if op == "dilate":
    v = -v
    v[v == 0] = np.float32(0.0)
  return v


def brute_line(lines, w, defect=None):
  """line_sites by the definition alone, one voxel at a time with Fraction (lines of at most EXACT_N)."""
  lines = np.asarray(lines, np.float32)
  L, n = lines.shape
  w2 = _w2(w)
  values = lines.copy()
  sites = np.full((L, n), -1, np.int64)
  for l in range(L):
    g = [float(x) for x in lines[l]]
    for i in range(n):
      cands = [j for j in range(n) if g[j] != np.inf]
      if not np.isfinite(w2):
        sites[l, i] = i if g[i] != np.inf else -1
        continue
      if not cands:
        continue
      negs = [j for j in cands if g[j] == -np.inf]
      if negs:
        sites[l, i], values[l, i] = negs[0], -INF
        continue
      exact = {j: Fraction(float(w2)) * (i - j) ** 2 + Fraction(g[j]) for j in cands}
      low = min(exact.values())
      j = min(j for j in cands if exact[j] == low)
      sites[l, i] = j
      values[l, i] = np.float32(g[i]) if j == i else np.float32(np.float64(w2) * np.float64((i - j) ** 2) + g[j])
  return values, sites
