"""CPU tests: the restatements of fill_holes and dust in holes_cases.py agree with each other on seeded volumes,
a bool mask gives scipy.ndimage.binary_fill_holes at every ndim and connectivity, the docstring examples hold,
and each planted defect is caught by the case generators."""
import numpy as np
import pytest
import scipy.ndimage as ndi

import holes_cases as hc

SHAPES = {1: (60,), 2: (17, 19), 3: (9, 10, 11)}


@pytest.mark.parametrize("nd", [1, 2, 3])
def test_the_two_fill_restatements_agree(nd):
  rng = np.random.default_rng(nd)
  for conn in range(1, nd + 1):
    for order in ("C", "F"):
      for trial in range(4):
        lab = hc.random_labels(rng, SHAPES[nd], nlabels=1 + trial % 3)
        lab = np.asfortranarray(lab) if order == "F" else lab
        for max_size in (None, 0, 2, 5):
          a = hc.restate_fill(lab, conn, max_size, order, "scipy")
          b = hc.restate_fill(lab, conn, max_size, order, "flood")
          assert np.array_equal(a[0], b[0]) and a[1] == b[1], (conn, order, max_size)


@pytest.mark.parametrize("nd", [1, 2, 3])
def test_the_two_dust_restatements_agree(nd):
  rng = np.random.default_rng(10 + nd)
  for conn in range(1, nd + 1):
    lab = hc.random_labels(rng, SHAPES[nd], nlabels=3, p=0.4)
    for threshold in (0, 1, 2, 3, 8):
      for invert in (False, True):
        assert np.array_equal(hc.restate_dust(lab, threshold, conn, invert, how="scipy"),
                              hc.restate_dust(lab, threshold, conn, invert, how="cc"))


@pytest.mark.parametrize("nd", [1, 2, 3])
def test_a_bool_mask_is_binary_fill_holes(nd):
  rng = np.random.default_rng(20 + nd)
  for conn in range(1, nd + 1):
    for _ in range(10):
      mask = hc.random_mask(rng, SHAPES[nd])
      want = ndi.binary_fill_holes(mask, hc.structure(nd, conn))
      for how in ("scipy", "flood"):
        got, n = hc.restate_fill(mask, conn, how=how)
        assert got.dtype == np.bool_ and np.array_equal(got, want) and n == int((want & ~mask).sum())


def test_the_docstring_examples(edt):
  assert "fill_holes(np.array([1, 0, 0, 1, 0]))" in edt.fill_holes.__doc__
  f = lambda a, **k: hc.restate_fill(np.array(a), **k)[0].tolist()
  assert f([1, 0, 0, 1, 0]) == [1, 1, 1, 1, 0]
  assert f([2, 0, 1, 0, 1]) == [2, 0, 1, 1, 1]
  ring = [[0, 1, 0], [1, 0, 1], [0, 1, 0]]
  assert f(ring) == [[0, 1, 0], [1, 1, 1], [0, 1, 0]]
  assert f(ring, connectivity=2) == ring
  assert f([1, 0, 0, 1], max_size=1) == [1, 0, 0, 1]
  d = lambda a, t, **k: hc.restate_dust(np.array(a), t, **k).tolist()
  assert d([1, 1, 0, 2, 0, 1], 2) == [1, 1, 0, 0, 0, 0]
  assert d([1, 1, 0, 2, 0, 1], 2, invert=True) == [0, 0, 0, 2, 0, 1]
  assert d([[1, 0], [0, 1]], 2) == [[0, 0], [0, 0]]
  assert d([[1, 0], [0, 1]], 2, connectivity=2) == [[1, 0], [0, 1]]


def test_the_case_volumes_have_the_answers_they_claim():
  for nd in (2, 3):
    lab, want = hc.cell_with_nucleus(nd)
    for conn in range(1, nd + 1):
      assert np.array_equal(hc.restate_fill(lab, conn)[0], want)
  lab = hc.diagonal_touch()
  assert hc.restate_fill(lab, 1)[0][2, 2] == 1 and hc.restate_fill(lab, 2)[0][2, 2] == 0
  for name, lab, conn in hc.crossing_holes():
    a, b = hc.restate_fill(lab, conn), hc.restate_fill(lab, conn, how="flood")
    assert np.array_equal(a[0], b[0]) and a[1] == b[1]
    assert (a[1] == 0) == name.startswith("open_"), name
  assert hc.restate_fill(hc.stacked_slabs(), stacked=True)[1].tolist() == [8, 0]


def _caught_fill(defect):
  """The generators that catch a fill_holes defect: the answer with the defect differs on some case."""
  cases = [(hc.diagonal_touch(), 2, None, False), (hc.cell_with_nucleus(2)[0], 1, None, False),
           (hc.sized_hole(7), 1, 7, False), (hc.stacked_slabs(), 1, None, True)]
  cases += [(lab, conn, None, False) for _, lab, conn in hc.crossing_holes()]
  rng = np.random.default_rng(0)
  cases += [(hc.random_labels(rng, SHAPES[3], nlabels=2), 3, None, False) for _ in range(3)]
  for how in ("scipy", "flood"):
    if not any(not np.array_equal(hc.restate_fill(lab, conn, m, how=how, stacked=st)[0],
                                  hc.restate_fill(lab, conn, m, how=how, defect=defect, stacked=st)[0])
               for lab, conn, m, st in cases):
      return False
  return True


@pytest.mark.parametrize("defect", [d for d in hc.DEFECTS if d != "threshold_off_by_one"])
def test_each_fill_defect_is_caught(defect):
  assert _caught_fill(defect), defect


def test_the_dust_defect_is_caught():
  comp = (hc.sized_hole(7) == 0).astype(np.uint8)
  for how in ("scipy", "cc"):
    assert not np.array_equal(hc.restate_dust(comp, 7, how=how),
                              hc.restate_dust(comp, 7, how=how, defect="threshold_off_by_one"))
