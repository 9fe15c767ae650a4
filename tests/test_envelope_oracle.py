"""CPU tests of the per-pass envelope inputs: the sample generators, the brute force of one
later-axis pass against the oracle's, the float32 rounding edges the GPU tests rely on, and the
oracle against the compiled reference's rounding-edge fixtures (tests/golden/rounding_edges.npz).
"""
import os
from fractions import Fraction

import numpy as np
import pytest

import envelope_cases as ec

EDGES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rounding_edges.npz")

TIE_ANISO = (2.0 ** -26, float(np.float32(1.333549976348877)))


def tie_image():
  img = np.ones((2, 4), dtype=np.uint8, order="F")
  img[0, 0] = 0
  return img


def test_generators_are_deterministic():
  for kind in ec.PROFILES:
    a = ec.profile(np.random.default_rng(5), kind, (3, 40, 7))
    b = ec.profile(np.random.default_rng(5), kind, (3, 40, 7))
    assert a.dtype == np.float32 and np.array_equal(a, b, equal_nan=True), kind
  for kind in ec.LABELINGS:
    for axis in (1, 2):
      a = ec.labels(np.random.default_rng(6), kind, (40, 33, 7), axis, np.uint16)
      b = ec.labels(np.random.default_rng(6), kind, (40, 33, 7), axis, np.uint16)
      assert a.dtype == np.uint16 and np.array_equal(a, b), (kind, axis)
  f = ec.profile(np.random.default_rng(1), "inf_rich", (2, 30, 5))
  assert np.all(np.isinf(f[..., 1]))
  assert np.all(ec.profile(np.random.default_rng(1), "above_2_24", (2, 30, 5)) >= 2 ** 24)


@pytest.mark.parametrize("axis", [1, 2])
@pytest.mark.parametrize("kind", ec.PROFILES)
def test_brute_force_matches_oracle_pass(oracle, axis, kind):
  rng = np.random.default_rng(hash((axis, kind)) % 2 ** 32)
  for n in (1, 2, 31, 33, 65):
    shape = (n, 3, 4) if axis == 2 else (2, n, 5)
    f = ec.profile(rng, kind, shape)
    for labeling in ec.LABELINGS:
      lab = ec.labels(rng, labeling, shape, axis, np.uint8)
      for w in (1.0, 3.0, 0.7, 1.333549976348877):
        for lo, hi in ((0, 0), (1, 0), (0, 1), (1, 1)):
          want = ec.brute_pass(lab, f, axis, w, lo, hi)
          got = ec.expected_pass(oracle, lab, f, axis, w, lo, hi)
          assert np.array_equal(got, want), (n, labeling, w, lo, hi, np.argwhere(got != want)[:3])


def test_double_rounding_tie_exists(oracle, reference):
  """w2 * 9 + 2^-52 at [1, 3] of the tie image: the reference forms the sum in double (one
  rounding) and rounds that to float32 (a second); a fused multiply-add rounds the exact sum once,
  one ulp higher.  Kernels that use the fused form must not be given this pass."""
  w2 = Fraction(float(np.float32(np.float32(TIE_ANISO[1]) ** 2)))
  exact = w2 * 9 + Fraction(2) ** -52
  twice = np.float32(float(exact))               # float(Fraction) rounds correctly to double
  near = np.float32(float(exact))
  cands = (np.nextafter(near, np.float32(-np.inf)), near, np.nextafter(near, np.float32(np.inf)))
  once = min(cands, key=lambda c: (abs(Fraction(float(c)) - exact), int(c.view(np.uint32)) & 1))
  assert float(twice) == 16.005199432373047 and float(once) == 16.00520133972168
  got = oracle.edtsq(tie_image(), anisotropy=TIE_ANISO, black_border=False)
  assert float(got[1, 3]) == float(twice)
  if reference is not None:
    assert np.array_equal(reference.edtsq(tie_image(), anisotropy=TIE_ANISO, black_border=False), got)


def strict_walk(f, row, w2=1.0):
  """walk_begin of the tile kernel restated with float32 candidates: start at the nearest vertex
  at or below `row`, step down while the next vertex is STRICTLY lower."""
  sites = [p for p in range(len(f)) if np.isfinite(f[p])]
  cand = {p: np.float32(w2 * (row - p) ** 2 + float(f[p])) for p in sites}
  below = [p for p in sites if p <= row]
  v = below[-1]
  for u in reversed(below[:-1]):
    if not cand[u] < cand[v]:
      break
    v = u
  return cand[v]


@pytest.mark.parametrize("m", [8, 9, 40])
def test_plateau_trap_is_a_trap(oracle, m):
  f, K, pos = ec.plateau_trap(m=m)
  lab = np.ones((len(f), 1, 1), np.uint8)
  vol = f.reshape(-1, 1, 1)
  want = ec.brute_pass(lab, vol, 2, 1.0, 0, 0)
  assert np.array_equal(ec.expected_pass(oracle, lab, vol, 2, 1.0, 0, 0), want)
  assert float(want[64, 0, 0]) == K - 128                      # the farthest vertex wins
  assert float(strict_walk(f, 64)) == K                         # a strict descent stops on the plateau
  # each of the three sites is the exact minimum at some row: all are vertices of the envelope
  owners = {min(pos, key=lambda p: (r - p) ** 2 + float(f[p])) for r in range(len(f))}
  assert owners == set(pos)


def test_oracle_pins_rounding_edge_fixtures(oracle):
  z = np.load(EDGES)
  names = [str(s) for s in z["names"]]
  assert len(names) >= 10
  for name in names:
    lab = z[name + "_labels"]
    an = tuple(float(a) for a in z[name + "_aniso"])
    bb = bool(z[name + "_border"])
    got = oracle.edtsq(lab, anisotropy=an, black_border=bb)
    want = z[name + "_edtsq"]
    assert got.shape == want.shape and np.array_equal(got, want, equal_nan=True), name
  tie = z["tie2d_edtsq"]
  assert float(tie[1, 3]) == 16.005199432373047
