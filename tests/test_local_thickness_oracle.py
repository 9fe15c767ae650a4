"""CPU tests of the local thickness restatements (local_thickness_cases): the threshold restatement on the
oracle's edtsq equals the seed/voxel brute force on tiny multi-label volumes, the known answers hold, the
default levels keep their promises, and each planted defect is caught."""
import numpy as np
import pytest

import local_thickness_cases as lt
import morphology_cases as mc

# integer and dyadic weights: every squared distance is exact in float32 and float64 alike
WEIGHTS = {1: [None, (2.0,), (0.5,)], 2: [None, (1.0, 2.0), (0.5, 1.5)], 3: [None, (1.0, 2.0, 0.5), (1.5, 1.0, 1.0)]}
SHAPES = {1: (23,), 2: (9, 11), 3: (6, 5, 7)}
LEVELS = [0.0, 0.5, 1.0, 1.5, 2.0, 2.5, 3.0, 4.5]


@pytest.mark.parametrize("nd", [1, 2, 3])
@pytest.mark.parametrize("kind", mc.KINDS)
def test_threshold_equals_brute_force(oracle, nd, kind):
  rng = np.random.default_rng(nd * 10 + mc.KINDS.index(kind))
  arr = mc.seeded(rng, kind, SHAPES[nd], np.uint16)
  for w in WEIGHTS[nd]:
    for bb in (False, True):
      want = lt.brute(arr, LEVELS, w, bb)
      assert np.array_equal(lt.threshold(arr, LEVELS, w, bb), want), (w, bb)
      levels = lt.default_levels(arr, 7, w, bb)
      assert np.array_equal(lt.threshold(arr, levels, w, bb), lt.brute(arr, levels, w, bb)), (w, bb)


def test_float_labels_fold_minus_zero(oracle):
  arr = np.array([[0.0, -0.0, 2.5, 2.5, 2.5], [-0.0, 2.5, 2.5, 2.5, -1.0], [0.0, 2.5, 2.5, -1.0, -1.0]], np.float32)
  for bb in (False, True):
    assert np.array_equal(lt.threshold(arr, LEVELS, None, bb), lt.brute(arr, LEVELS, None, bb))
  assert not lt.threshold(arr, LEVELS)[arr == 0].any()


def test_order_and_repeats_of_levels_do_not_matter(oracle):
  arr = lt.rod_between_balls()[0]
  a = lt.threshold(arr, [4.0, 1.0, 2.0, 0.5])
  assert np.array_equal(a, lt.threshold(arr, [0.5, 1.0, 1.0, 2.0, 4.0, 4.0]))


def test_run_of_seven_takes_the_top_default_level(oracle):
  arr = lt.run_of_seven()
  levels = lt.default_levels(arr, 25)
  assert 3.5 < levels[0] < 4.0 and levels[-1] == 0.5
  got = lt.threshold(arr, levels)
  assert np.all(got[1:-1] == np.float32(levels[0])) and got[0] == 0 and got[-1] == 0
  assert np.array_equal(got, lt.brute(arr, levels))
  # the same run with the volume's faces as background
  ones = np.ones(7, np.uint8)
  assert np.all(lt.threshold(ones, lt.default_levels(ones, 25, None, True), None, True) == np.float32(levels[0]))


@pytest.mark.parametrize("t", [3, 4, 5, 6, 7])
def test_slab_is_uniform(oracle, t):
  arr = lt.slab(t)
  sizes = [0.5, 1.0, 1.5, 2.0, 2.5, 3.0, 3.5, 4.0]
  got = lt.threshold(arr, sizes)
  inside = got[arr != 0]
  assert np.all(inside == inside[0]) and not got[arr == 0].any()
  # the largest size whose erosion is not empty: below the slab's R = ceil(t / 2)
  assert inside[0] == max(s for s in sizes if s < (t + 1) // 2)


def test_rod_between_balls_takes_the_rods_level(oracle):
  arr, mid = lt.rod_between_balls()
  got = lt.threshold(arr, [0.5, 1.0, 2.0, 4.0])
  assert got[mid] == 1.0
  assert got[arr.shape[0] // 2, 7] == 4.0                      # a disc centre
  assert np.array_equal(got, lt.brute(arr, [0.5, 1.0, 2.0, 4.0]))


def test_thin_line_takes_half_a_voxel(oracle):
  arr = lt.thin_line()
  got = lt.threshold(arr, (0.5, 1.0, 2.0))
  assert np.all(got[arr != 0] == 0.5) and not got[arr == 0].any()


def test_default_levels_promises(oracle):
  rng = np.random.default_rng(3)
  for w in (None, (1.0, 2.0), (0.7, 1.3)):
    arr = mc.voronoi(rng, (15, 13), 5, np.uint8)
    levels = lt.default_levels(arr, 12, w, True)
    h = lt.least_weight(lt.weights(arr, w))
    assert np.all(np.diff(levels) < 0) and levels[-1] == h / 2
    got = lt.threshold(arr, levels, w, True)
    assert np.all(got[arr != 0] >= np.float32(h / 2))
    d2 = lt.threshold(arr, levels[:1], w, True)
    assert d2.any()                                             # the top level keeps seeds
  one = np.full((6, 5), 4, np.uint8)                            # one label, no black border: R = h/2
  assert np.all(lt.default_levels(one, 5, (2.0, 3.0)) == 1.0)
  assert np.all(lt.threshold(one, lt.default_levels(one, 5, (2.0, 3.0)), (2.0, 3.0)) == 1.0)
  empty = np.zeros((4, 4), np.uint8)
  assert np.all(lt.default_levels(empty, 3) == 0.5) and not lt.threshold(empty, [0.5]).any()


@pytest.mark.parametrize("defect", lt.DEFECTS)
def test_every_defect_is_caught(oracle, defect):
  caught = False
  for arr in (lt.rod_between_balls()[0], lt.slab(6), mc.bridges((12, 9), np.uint8)):
    for bb in (False, True):
      sizes = [0.5, 1.0, 2.0, 2.5, 3.0, 4.0]
      caught |= not np.array_equal(lt.threshold(arr, sizes, None, bb, defect), lt.brute(arr, sizes, None, bb))
  assert caught, defect
