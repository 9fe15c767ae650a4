"""CPU tests: the medial axis restated (medial_axis_cases.py) against the brute-force lexicographic rule, the
guarantees the docstring states (the reconstruction, each site in its voxel's label, a medial voxel in every
label), the worked examples, and that each planted defect is noticed."""
import numpy as np
import pytest

import medial_axis_cases as mac

WEIGHTS = {1: [(1.0,), (2.0,), (3.0,)], 2: [(1.0, 1.0), (1.0, 2.0), (3.0, 1.0)],
           3: [(1.0, 1.0, 1.0), (1.0, 2.0, 3.0), (2.0, 1.0, 1.0)]}
SHAPES = {1: [(17,), (30,)], 2: [(9, 11), (12, 7)], 3: [(5, 6, 7), (7, 5, 4)]}


def _volumes(nd, seed):
  rng = np.random.default_rng(seed)
  for shape in SHAPES[nd]:
    for kind in mac.KINDS:
      yield kind, mac.seeded(rng, kind, shape, np.uint16)
    yield "noise", rng.integers(0, 3, shape).astype(np.uint8)


@pytest.mark.parametrize("border", [False, True])
@pytest.mark.parametrize("nd", [1, 2, 3])
def test_restatement_is_the_lexicographic_rule(nd, border):
  for w in WEIGHTS[nd]:
    for kind, labels in _volumes(nd, nd):
      got = mac.restate(labels, w, border)[0]
      assert np.array_equal(got, mac.brute(labels, w, border)), (kind, w, labels.shape)


@pytest.mark.parametrize("border", [False, True])
@pytest.mark.parametrize("nd", [1, 2, 3])
def test_reconstruction_and_labels(nd, border):
  for w in WEIGHTS[nd]:
    for kind, labels in _volumes(nd, 10 + nd):
      medial, d2, values, idx = mac.restate(labels, w, border)
      rec = mac.reconstruct(medial, d2, w)
      fg = labels != 0
      assert np.array_equal(rec[fg], values[fg]) and np.all(rec[fg] > 0), (kind, w)
      assert np.array_equal(rec > 0, fg), (kind, w)                     # integer weights: exactly the labels
      assert not np.any(medial & ~fg)
      site = labels[tuple(idx)]
      assert np.array_equal(site[fg], labels[fg]), (kind, w)             # q(p) carries L(p)
      for m in np.unique(labels[fg]):                                    # per label: its balls rebuild it
        own = labels == m
        assert medial[own].any()
        assert np.array_equal(mac.reconstruct(medial & own, d2, w) > 0, own), (kind, w, m)


def test_the_reconstruction_holds_for_other_weights():
  rng = np.random.default_rng(5)
  for w in [(0.7, 1.3), (1.1, 2.9), (0.3, 0.3)]:
    for kind in mac.KINDS:
      labels = mac.seeded(rng, kind, (10, 13), np.int32)
      for border in (False, True):
        medial, d2, values, _ = mac.restate(labels, w, border)
        fg = labels != 0
        rec = mac.reconstruct(medial, d2, w)
        assert np.array_equal(rec[fg], values[fg]) and np.all(rec[fg] > 0), (kind, w, border)


def test_worked_examples():
  five = np.array([0, 1, 1, 1, 1, 1, 0], np.uint8)
  medial, d2, _, _ = mac.restate(five)
  assert d2[1:6].tolist() == [1, 4, 9, 4, 1] and np.flatnonzero(medial).tolist() == [3]
  four = np.array([0, 1, 1, 1, 1, 0], np.uint8)
  medial, d2, _, _ = mac.restate(four)
  assert d2[1:5].tolist() == [1, 4, 4, 1] and np.flatnonzero(medial).tolist() == [2, 3]
  for labels in (np.full(9, 3, np.uint8), np.full((4, 5), 2, np.int32), np.full((3, 4, 2), 7, np.uint16)):
    medial, d2, _, _ = mac.restate(labels)
    assert np.all(np.isinf(d2)) and np.flatnonzero(medial).tolist() == [0]
    assert np.array_equal(medial, mac.brute(labels, (1.0,) * labels.ndim))
    medial, d2, _, _ = mac.restate(labels, black_border=True)              # with a border: finite balls
    assert np.all(np.isfinite(d2)) and np.array_equal(mac.reconstruct(medial, d2) > 0, labels != 0)


def test_stacks_are_the_per_volume_calls():
  rng = np.random.default_rng(3)
  for order in ("C", "F"):
    for shape in ((4, 9), (3, 6, 7), (2, 4, 5, 3)):
      labels = rng.integers(0, 3, shape).astype(np.uint8)
      labels = np.asfortranarray(labels) if order == "F" else labels
      w = (1.0, 2.0, 1.0)[:len(shape) - 1]
      got = mac.restate(labels, w, True, order, stacked=True)[0]
      axis = 0 if order == "C" else len(shape) - 1
      want = np.stack([mac.restate(np.take(labels, i, axis), w, True, order)[0] for i in range(shape[axis])], axis)
      assert np.array_equal(got, want), (order, shape)


def test_planted_defects_are_noticed():
  rng = np.random.default_rng(8)
  caught = {"background": 0, "greatest": 0}
  for nd in (1, 2, 3):
    for w in WEIGHTS[nd]:
      for kind, labels in _volumes(nd, 20 + nd):
        for border in (False, True):
          want = mac.brute(labels, w, border)
          for defect in caught:
            caught[defect] += not np.array_equal(mac.restate(labels, w, border, defect=defect)[0], want)
  assert all(n > 0 for n in caught.values()), caught
