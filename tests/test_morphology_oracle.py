"""CPU tests: the two restatements of the spherical morphology in morphology_cases.py -- the threshold
rule on the CPU oracle's transforms and scipy.ndimage per label -- agree wherever the arithmetic is
exact (integer and dyadic weights, radii with exact ties such as r = 2 and the 3-4-5 triangle at
r = 5), and each of them notices a planted defect."""
import numpy as np
import pytest

import morphology_cases as mc

SHAPES = [(41,), (23, 19), (14, 12, 11)]
# exact: integer and dyadic weights, squares exact in float32 and float64
WEIGHTS = {1: [(1.0,), (2.0,), (0.5,)], 2: [(1.0, 1.0), (1.0, 2.0), (0.75, 1.25)],
           3: [(1.0, 1.0, 1.0), (1.0, 2.0, 1.0), (0.5, 1.0, 1.5)]}
RADII = [0.0, 1.0, 1.5, 2.0, 3.0, 5.0]


@pytest.mark.parametrize("op", mc.OPS)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%dd" % len(s))
@pytest.mark.parametrize("kind", mc.KINDS)
def test_restatements_agree(oracle, op, shape, kind):
  rng = np.random.default_rng(100 * mc.OPS.index(op) + 10 * len(shape) + mc.KINDS.index(kind))
  arr = mc.seeded(rng, kind, shape, np.uint16)
  for w in WEIGHTS[len(shape)]:
    for r in RADII:
      for bb in (False, True):
        want = mc.per_label(op, arr, r, w, bb)
        got = mc.threshold(op, arr, r, w, bb)
        assert got.dtype == want.dtype and np.array_equal(got, want), (op, kind, w, r, bb)


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("dtype", [np.uint8, np.int32, np.uint64, np.float32, np.float64, np.bool_])
def test_restatements_agree_on_dtypes(oracle, dtype, order):
  rng = np.random.default_rng(11)
  arr = mc.seeded(rng, "touching", (13, 11, 9), np.int32)
  arr = (arr != 0) if dtype == np.bool_ else arr.astype(dtype)
  arr = np.asfortranarray(arr) if order == "F" else np.ascontiguousarray(arr)
  if arr.dtype.kind == "f":
    arr[arr == 0] = -0.0                     # background by value
  for op in mc.OPS:
    for r in (1.0, 2.0):
      got, want = mc.threshold(op, arr, r, (1.0, 1.0, 2.0), True), mc.per_label(op, arr, r, (1.0, 1.0, 2.0), True)
      assert got.dtype == (np.bool_ if op in ("dilate", "close") else arr.dtype)
      assert np.array_equal(mc._raw(got), mc._raw(want)), (op, r)
      if op in ("erode", "open"):
        assert not np.signbit(got[got == 0]).any() if got.dtype.kind == "f" else True


def test_three_four_five_tie(oracle):
  """A voxel at (3, 4) from the nearest other label is at exactly r = 5: within, so it is eroded."""
  arr = np.ones((9, 11), np.uint8)
  arr[0, 0] = 0
  got = mc.threshold("erode", arr, 5.0)
  assert got[3, 4] == 0 and got[3, 5] == 1
  assert np.array_equal(got, mc.per_label("erode", arr, 5.0))


def test_one_label_without_black_border_has_no_site(oracle):
  arr = np.full((6, 7), 3, np.int16)
  for op in ("erode", "open"):
    assert np.array_equal(mc.threshold(op, arr, 4.0), arr)
    assert np.array_equal(mc.per_label(op, arr, 4.0), arr)
  assert not mc.threshold("erode", arr, 4.0, black_border=True).any()


DEFECT_CASES = [
  ("lt", "erode", 2.0, False),
  ("lt", "dilate", 2.0, False),
  ("border", "erode", 2.0, False),
  ("border", "close", 2.0, True),
  ("open_border", "open", 3.0, False),
]


@pytest.mark.parametrize("defect,op,r,bb", DEFECT_CASES, ids=[c[0] + "_" + c[1] for c in DEFECT_CASES])
def test_each_restatement_notices_a_planted_defect(oracle, defect, op, r, bb):
  rng = np.random.default_rng(5)
  arr = mc.balls(rng, (24, 22, 20), 6, 7.0, np.uint8) if op in ("dilate", "close") else mc.voronoi(rng, (24, 22, 20), 5)
  good_t, good_s = mc.threshold(op, arr, r, None, bb), mc.per_label(op, arr, r, None, bb)
  assert np.array_equal(good_t, good_s)
  assert not np.array_equal(mc.threshold(op, arr, r, None, bb, defect=defect), good_s)
  assert not np.array_equal(mc.per_label(op, arr, r, None, bb, defect=defect), good_t)
