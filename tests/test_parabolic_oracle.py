"""CPU tests: the restatement of parabolic erosion and dilation in parabolic_cases.py against
scipy.ndimage's grey_erosion / grey_dilation with the full-size non-flat structure -sum_a (w_a q_a)^2
(where every sum is exact: integer samples and weights), against the CPU oracle's edtsq on masks, and
the planted defects each noticed."""
import numpy as np
import pytest
from scipy import ndimage

import parabolic_cases as pc

SHAPES = [(9,), (7, 6), (5, 4, 6)]
WEIGHTS = {1: [(1.0,), (3.0,)], 2: [(1.0, 1.0), (2.0, 1.0)], 3: [(1.0, 1.0, 1.0), (1.0, 2.0, 3.0)]}


def _structure(shape, w):
  grids = np.meshgrid(*[np.arange(-(n - 1), n) for n in shape], indexing="ij")
  return -sum((wa * g.astype(np.float64)) ** 2 for wa, g in zip(w, grids))


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%dd" % len(s))
@pytest.mark.parametrize("op", ["erode", "dilate"])
def test_restatement_equals_scipy_grey_morphology(op, shape):
  rng = np.random.default_rng(len(shape) + (10 if op == "dilate" else 0))
  for w in WEIGHTS[len(shape)]:
    for trial in range(3):
      f = rng.integers(-40, 60, shape).astype(np.float64)
      if trial == 2:
        f[rng.random(shape) < 0.5] = np.inf if op == "erode" else -np.inf
      s = _structure(shape, w)
      if op == "erode":
        want = ndimage.grey_erosion(f, structure=s, mode="constant", cval=np.inf)
      else:
        want = ndimage.grey_dilation(f, structure=s, mode="constant", cval=-np.inf)
      got = pc.restate(op, f, w)
      assert np.array_equal(got.astype(np.float64), want), (op, w, trial)


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("w", [(1.0, 1.0, 1.0), (6.0, 6.0, 30.0), (2.0, 3.0, 5.0)])
def test_restatement_of_a_mask_equals_the_oracle_edtsq(oracle, w, order):
  rng = np.random.default_rng(7)
  mask = rng.random((9, 11, 13)) < 0.85
  mask = np.asfortranarray(mask) if order == "F" else mask
  f = np.where(mask, np.float32(np.inf), np.float32(0))
  ww = w if order == "C" else tuple(reversed(w))
  m = mask if order == "C" else np.ascontiguousarray(mask.T)
  want = oracle.edtsq(m.astype(np.uint8), ww if order == "F" else w)
  got = pc.erode(f, w, order=order)
  assert pc.same_bits(got if order == "C" else np.ascontiguousarray(got.T), want)


def test_c_and_f_order_of_the_same_data_agree():
  rng = np.random.default_rng(3)
  f = pc.values("wide", (6, 7, 8), rng)
  w = (0.7, 1.3, 2.9)
  c = pc.erode(f, w, order="C")
  fo = pc.erode(f.T, tuple(reversed(w)), order="F")
  assert pc.same_bits(c.T, fo)


def test_stack_is_the_stack_of_volumes():
  rng = np.random.default_rng(4)
  f = pc.values("uniform", (3, 5, 6), rng)
  got = pc.dilate(f, (1.5, 0.5), stacked=True)
  assert pc.same_bits(got, np.stack([pc.dilate(v, (1.5, 0.5)) for v in f]))


def test_special_values():
  inf, nan = np.float32(np.inf), np.float32(np.nan)
  line = np.array([inf, nan, inf], np.float32)
  assert pc.same_bits(pc.erode(line), [inf, inf, inf])
  assert pc.same_bits(pc.dilate(line), [inf, inf, inf])         # +inf is -(-inf): one -inf line
  assert pc.same_bits(pc.dilate(np.array([nan, nan], np.float32)), [-inf, -inf])
  assert pc.same_bits(pc.erode(np.array([5, -inf, 7], np.float32)), [-inf, -inf, -inf])
  assert pc.same_bits(pc.erode(np.array([-0.0, 2.0], np.float32)), [0.0, 1.0])
  assert pc.same_bits(pc.dilate(np.array([-0.0, 0.0], np.float32)), [0.0, 0.0])
  # w^2 overflows float32: the pass leaves its samples as they are (NaN and -0.0 folded)
  assert pc.same_bits(pc.erode(np.array([3.0, nan, -0.0, 1.0], np.float32), 1e20), [3.0, inf, 0.0, 1.0])


def test_near_tie_needs_the_true_minimiser():
  rng = np.random.default_rng(5)
  f = pc.near_tie_line(700, rng)
  i = int(np.flatnonzero(f == np.float32(16773121))[0]) + 33
  got = pc.line_pass(f[None], pc.NEAR_TIE_W)[0]
  assert got[i] == np.float32(64 * 513 * 513)             # the midpoint rounds down; the other site up
  assert np.float32(np.float64(f[i + 513]) + 64.0 * 513 * 513) == np.float32(64 * 513 * 513 + 2)


@pytest.mark.parametrize("defect", ["w2_double", "negzero"])
def test_each_defect_is_noticed(oracle, defect):
  rng = np.random.default_rng(6)
  mask = rng.random((9, 11, 13)) < 0.85
  w = (1.3, 2.9, 1.0)                   # w^2 rounds differently in float32 and float64 along y and z
  f = np.where(mask, np.float32(np.inf), np.float32(-0.0))
  want = oracle.edtsq(mask.astype(np.uint8), w)
  assert pc.same_bits(pc.erode(f, w), want)
  assert not pc.same_bits(pc.erode(f, w, defect=defect), want)
