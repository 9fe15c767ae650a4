"""CPU tests of the window-kernel restatement (tests/window_cases.py): its plan against
edtb200_bounded_plan (pure host logic, no device), its pass against the oracle's envelope pass when
nothing is cut, and the window it implies against the whole run it takes the minimum over.
"""
import ctypes
import math
from fractions import Fraction

import numpy as np
import pytest

import envelope_cases as ec
import window_cases as wc

WINDOW_MAX = 2           # EDTB200_BOUNDED_WINDOW_MAX
SITES_WINDOW_MAX = 32    # EDTB200_BOUNDED_SITES_WINDOW_MAX
F32_MAX = float(np.finfo(np.float32).max)

WEIGHTS = [1.0, 3.0, 30.0,                                        # integer
           0.7, 1.3, 2.9, 0.1, 1.333549976348877,                  # real
           0.5, 0.25, 1.5, 0.125, 2.5,                             # dyadic
           2.0 ** -26, 1e20]                                       # tiny (w2 = 2^-52) and huge (w2 = +inf)


def f32(x):
  return np.float32(x)


def around(x):
  """x and the doubles either side of it."""
  return [x, math.nextafter(x, 0.0), math.nextafter(x, math.inf)]


def distances():
  """d = 0, subnormal, the roots of squares and of their float32 neighbours, values near sqrt(FLT_MAX)
  and FLT_MAX, +inf."""
  out = [0.0, 5e-324, 1e-300, math.sqrt(1e-45), 1e-20]
  for k in (1, 2, 3, 7, 31, 32, 33, 64, 127, 128, 129, 4097):
    sq = f32(k * k)
    for b in (sq, np.nextafter(sq, f32(0)), np.nextafter(sq, f32(np.inf))):
      out += around(math.sqrt(float(b)))
  out += around(math.sqrt(F32_MAX)) + around(float(np.nextafter(f32(F32_MAX), f32(0)))) + around(F32_MAX)
  out += [1e19, 1e20, 1e200, math.inf]
  return out


def on_b_plus():
  """(w, d, r): distances whose B+ (the float32 after B) is exactly w2 r^2, so that r is just out of reach."""
  out = []
  for w in (1.0, 1.5, 0.5, 0.7, 2.9, 2.0 ** -26, 3.0):
    w2 = f32(f32(w) * f32(w))
    for r in (1, 2, 3, 4, 8, 16, 32, 64, 128, 1024):
      t = w2 * f32(r * r)
      if float(t) != float(w2) * r * r:
        continue                                   # w2 r^2 is not a float32
      b = np.nextafter(t, f32(0))
      d = math.sqrt(float(b))
      while wc.plan(w, d)[0] < b:
        d = math.nextafter(d, math.inf)
      while wc.plan(w, d)[0] > b:
        d = math.nextafter(d, 0.0)
      if wc.plan(w, d)[0] == b:
        out.append((w, d, r))
  return out


def library_plan(edt, w, d):
  r = (ctypes.c_int64 * 3)()
  win = (ctypes.c_int * 3)()
  assert edt._lib().edtb200_bounded_plan(3, 8, 8, 8, w[0], w[1], w[2], d, r, win) == 0
  return list(r), list(win)


def windowed_bits(k, r):
  return int(k >= 1 and r <= WINDOW_MAX) | int(k >= 1 and r <= SITES_WINDOW_MAX) << 1


@pytest.fixture
def default_limits(monkeypatch):
  monkeypatch.delenv("EDTB200_BOUNDED_RMAX", raising=False)


def double_test_is_exact(w, r):
  """Whether the library's test of r and r + 1, (double)w2 * r * r in double arithmetic, is exact."""
  with np.errstate(over="ignore"):
    w2 = float(f32(f32(w) * f32(w)))
  if not math.isfinite(w2):
    return True
  return all(Fraction(w2 * float(x) * float(x)) == Fraction(w2) * x * x for x in (r, r + 1))


def test_plan_is_the_exact_restatement(edt, default_limits):
  """Every radius equals the exact one wherever the library's double products are exact (every radius
  up to 2^14 whatever the weight, and far beyond for dyadic weights); beyond that, where only a
  product that rounds can tell r from r + 1, the two agree to double precision."""
  exact = 0
  for i, w in enumerate(WEIGHTS):
    ws = (w, WEIGHTS[(i + 3) % len(WEIGHTS)], WEIGHTS[(i + 7) % len(WEIGHTS)])
    for d in distances():
      radius, windowed = library_plan(edt, ws, d)
      want = [wc.plan(x, d)[1] for x in ws]
      for x, got, r in zip(ws, radius, want):
        if r == wc.CAP or double_test_is_exact(x, r):
          assert got == r, (ws, d, radius, want)
          exact += r < (1 << 14)
        else:
          assert r > (1 << 14) and abs(got - r) <= r * 2.0 ** -50, (ws, d, radius, want)
      assert windowed == [windowed_bits(k, r) for k, r in enumerate(want)], (ws, d, windowed)
  assert exact > 500, exact


def test_plan_on_b_plus(edt, default_limits):
  """Where w2 r^2 is exactly B+, r is out of reach: R = r - 1, in the restatement and the library."""
  cases = on_b_plus()
  assert len(cases) >= 30
  for w, d, r in cases:
    assert wc.plan(w, d)[1] == r - 1, (w, d, r)
    assert wc.plan(w, math.nextafter(d, math.inf))[1] >= r - 1
    assert library_plan(edt, (w, w, w), d)[0] == [r - 1] * 3, (w, d, r)


def test_plan_edges():
  assert wc.plan(1.0, 0.0) == (0.0, 0)
  assert wc.plan(1.0, 3.0) == (9.0, 3)
  assert wc.plan(1.0, float(np.nextafter(f32(3.0), f32(0))))[1] == 2
  assert wc.plan(1.0, math.inf) == (f32(F32_MAX), wc.CAP)
  assert wc.plan(1e20, 5.0) == (25.0, 0)                 # w2 = +inf: only the row itself
  assert wc.plan(2.0 ** -26, 1.0)[1] == (1 << 26) + 3     # w2 = 2^-52: r^2 < 2^52 + 2^29
  b, r = wc.plan(1.0, 5e-324)                            # a subnormal d squares to 0
  assert b == 0.0 and r == 0
  for w in (1.0, 0.7, 2.5):
    for r in (0, 1, 2, 3, 31, 32, 33, 63, 64, 65, 127, 128):
      d, b = wc.distance_for(w, r)
      assert wc.plan(w, d) == (b, r)
      assert float(b) >= float(f32(f32(w) * f32(w))) * r * r


def pass_cases():
  rng = np.random.default_rng(41)
  k = 0
  for n in (1, 2, 5, 33, 64, 65, 130):
    for shape, axis in (((n, 3, 5), 2), ((2, n, 7), 1)):
      for kind in ec.PROFILES:
        k += 1
        lab = ec.labels(rng, ec.LABELINGS[k % len(ec.LABELINGS)], shape, axis, np.uint16)
        f = ec.profile(rng, kind, shape)
        w = (1.0, 3.0, 0.7, 1.333549976348877)[k % 4] if kind not in ("int_ties", "zeros", "above_2_24") else \
            (1.0, 3.0)[k % 2]
        yield lab, f, axis, w, k % 2, (k // 2) % 2, kind


def test_unbounded_pass_is_the_oracle_pass(oracle):
  """With d = +inf nothing is cut, and the pass is the reference's envelope pass, except at the
  read-out exception (DESIGN.md section 8): there the reference keeps an earlier hull vertex on a row
  where a later one is lower by less than the rounding of their intersection.  Such a row is counted,
  and the restatement must be the brute force of the definition there (envelope_cases.brute_pass)."""
  exceptions = 0
  for lab, f, axis, w, lo, hi, kind in pass_cases():
    got = wc.window_pass(lab, f, axis, w, math.inf, lo, hi)
    want = ec.expected_pass(oracle, lab, f, axis, w, lo, hi)
    diff = got.view(np.uint32) != want.view(np.uint32)
    if diff.any():
      assert kind in ("real", "tiny"), (kind, axis, w, int(diff.sum()))
      brute = ec.brute_pass(lab, f, axis, w, lo, hi)
      assert np.array_equal(got[diff], brute[diff]) and (got[diff] < want[diff]).all(), (kind, w)
      exceptions += int(diff.sum())
    assert np.array_equal(got[~diff], want[~diff])
  assert exceptions <= 4, exceptions


@pytest.mark.parametrize("w", [1.0, 0.7, 2.5])
def test_window_of_radius_r_is_the_whole_run(w):
  """DESIGN.md section 5: within R rows is all a pass under bound B needs, so the window of R rows gives
  the whole-run pass bit for bit; R - 1 rows does not, on the lines built to tell them apart."""
  rng = np.random.default_rng(int(w * 10))
  for r in (1, 2, 3, 31, 32, 33, 63, 64, 65, 127, 128):
    d, b = wc.distance_for(w, r)
    for kind in ("sparse", "tile_edges", "at_bound", "border_ties"):
      for lo, hi in ((0, 0), (1, 1)):
        shape = (300, 3, 4)
        lab = wc.labels(rng, "one_run" if kind in ("sparse", "tile_edges") else "runs", shape, 2, np.uint32)
        f = wc.profile(rng, kind, shape, 2, w, r, b)
        whole = wc.pass_values(lab, f, 2, w, d, lo, hi)
        assert np.array_equal(wc.pass_values(lab, f, 2, w, d, lo, hi, radius=r), whole), (w, r, kind)
        assert np.array_equal(wc.pass_values(lab, f, 2, w, d, lo, hi, radius=r + 5), whole), (w, r, kind)
        if kind == "sparse" and not lo and not hi:
          short = wc.pass_values(lab, f, 2, w, d, lo, hi, radius=r - 1)
          assert not np.array_equal(short, whole), (w, r, kind)


def test_codes_check_rejects_wrong_codes():
  """check_codes notices a border term's code written as the plain row, a sample code moved one row,
  and a kSiteNone missing or misplaced."""
  rng = np.random.default_rng(5)
  shape, w, r = (70, 2, 3), 1.0, 4
  d, b = wc.distance_for(w, r)
  lab = wc.labels(rng, "runs", shape, 2, np.uint8)
  f = wc.profile(rng, "border_ties", shape, 2, w, r, b)
  codes = brute_codes(lab, f, 2, w, d, 1, 1)
  wc.check_codes(lab, f, 2, w, d, 1, 1, codes)
  direct = (codes < 0) & (codes != wc.SITE_NONE)
  assert direct.any() and (codes >= 0).any() and (codes == wc.SITE_NONE).any()
  plain = np.where(direct, -2 - codes, codes)
  with pytest.raises(AssertionError):
    wc.check_codes(lab, f, 2, w, d, 1, 1, plain)
  moved = np.where(codes >= 0, codes + 1, codes)
  with pytest.raises(AssertionError):
    wc.check_codes(lab, f, 2, w, d, 1, 1, moved)
  with pytest.raises(AssertionError):
    wc.check_codes(lab, f, 2, w, d, 1, 1, np.where(codes == wc.SITE_NONE, 0, codes))


def brute_codes(lab, f, axis, w, d, lo, hi):
  """Codes of one pass, row by row, as the window kernel picks them: its own row, then d = 1, 2, ... below
  before above, the first strictly lower candidate winning."""
  assert axis == 2
  w2 = float(np.float32(np.float32(w) * np.float32(w)))
  b, r = wc.plan(w, d)
  n = lab.shape[0]
  out = np.empty(lab.shape, np.int64)
  for j in np.ndindex(lab.shape[1:]):
    l, v = lab[(slice(None),) + j], f[(slice(None),) + j].astype(np.float64)
    for i in range(n):
      best, site = np.float32(v[i]), i
      down = up = True
      for dd in range(1, r + 1):
        wall = np.float32(w2 * dd * dd)
        for p, go in ((i - dd, down), (i + dd, up)):
          if not go:
            continue
          if p < 0 or p >= n or l[p] != l[i]:
            if p < i:
              down = False
            else:
              up = False
            if (0 <= p < n or (lo if p < 0 else hi)) and wall < best:
              best, site = wall, -2 - p
          else:
            c = np.float32(w2 * dd * dd + v[p])
            if c < best:
              best, site = c, p
      out[(i,) + j] = site if best <= b else wc.SITE_NONE
  return out.astype(np.int32)
