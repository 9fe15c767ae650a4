"""CPU tests: the restatements of connected_components and extended_maxima in components_cases.py agree with
each other on seeded volumes, give the worked examples of the docstrings and the header, and each planted
defect is caught by at least one volume here."""
import numpy as np
import pytest

import components_cases as cc


@pytest.mark.parametrize("nd", [1, 2, 3])
def test_the_three_component_restatements_agree(nd):
  rng = np.random.default_rng(nd)
  shape = {1: (200,), 2: (23, 31), 3: (9, 11, 13)}[nd]
  for conn in range(1, nd + 1):
    for order in ("C", "F"):
      lab = cc.random_labels(rng, shape)
      lab = np.asfortranarray(lab) if order == "F" else lab
      want = cc.restate_cc(lab, conn, order, "csgraph")
      assert np.array_equal(cc.restate_cc(lab, conn, order, "scipy"), want)
      assert np.array_equal(cc.restate_cc(lab, conn, order, "bfs"), want)


def test_c_order_is_scipy_label_numbering_for_one_label():
  import scipy.ndimage
  rng = np.random.default_rng(1)
  mask = rng.random((17, 19, 21)) < 0.4
  for conn in (1, 2, 3):
    want, _ = scipy.ndimage.label(mask, scipy.ndimage.generate_binary_structure(3, conn))
    assert np.array_equal(cc.restate_cc(mask, conn), want)
    # F order: scipy's numbering of a.T, transposed back
    f = np.asfortranarray(mask)
    want_f = scipy.ndimage.label(f.T, scipy.ndimage.generate_binary_structure(3, conn))[0].T
    assert np.array_equal(cc.restate_cc(f, conn, "F"), want_f)


@pytest.mark.parametrize("nd", [1, 2, 3])
def test_the_three_reconstructions_agree(nd):
  rng = np.random.default_rng(10 + nd)
  shape = {1: (40,), 2: (7, 9), 3: (4, 5, 6)}[nd]
  for conn in range(1, nd + 1):
    for h in (0.0, 0.25, 1.0, 2.5):
      img = cc.random_image(rng, shape, levels=6)
      img.reshape(-1)[rng.integers(0, img.size, 3)] = [np.nan, -0.0, np.inf]
      lab = cc.random_labels(rng, shape, nlabels=2, block=2)
      for labels in (None, lab):
        nodes, keys = cc._nodes_keys(labels, shape)
        f = cc.image_f(img)
        m = cc.start_m(f, h)
        R = cc.r_relax(f, m, nodes, keys, conn)
        assert np.array_equal(cc.r_flood(f, m, nodes, keys, conn).view(np.uint32), R.view(np.uint32))
        assert np.array_equal(cc.r_brute(f, m, nodes, keys, conn).view(np.uint32), R.view(np.uint32))
        want = cc.restate_em(img, h, labels, conn)
        for recon, how in (("flood", "bfs"), ("brute", "scipy")):
          assert np.array_equal(cc.restate_em(img, h, labels, conn, recon=recon, how=how), want)


def test_worked_examples():
  a = np.array([[1, 1, 0, 2], [0, 1, 0, 2], [3, 0, 0, 1]])
  assert cc.restate_cc(a).tolist() == [[1, 1, 0, 2], [0, 1, 0, 2], [3, 0, 0, 4]]
  assert cc.restate_cc(np.array([[1, 0], [0, 1]]), 1).tolist() == [[1, 0], [0, 2]]
  assert cc.restate_cc(np.array([[1, 0], [0, 1]]), 2).tolist() == [[1, 0], [0, 1]]
  x = np.array([0, 3, 1, 5, 2, 0], np.float32)
  for h in (0.0, 1.9):
    assert cc.restate_em(x, h).tolist() == [0, 1, 0, 2, 0, 0]
  assert cc.restate_em(x, 2.0).tolist() == [0, 0, 0, 1, 0, 0]
  y = np.array([0, 4, 3.5, 4, 0], np.float32)
  for h in (0.0, 0.4):
    assert cc.restate_em(y, h).tolist() == [0, 1, 0, 2, 0]
  for h in (0.5, 1.0):
    assert cc.restate_em(y, h).tolist() == [0, 1, 1, 1, 0]


def test_the_dynamic_rule():
  """With f - h exact, a peak survives exactly when its dynamic exceeds h: the peak of 3 behind a pass of 1
  on the way to 5 has dynamic 2."""
  x = np.array([0, 3, 1, 5, 2, 0], np.float32)
  for h, n in ((1.75, 2), (2.0, 1), (2.25, 1), (4.75, 1), (5.0, 1)):
    assert cc.restate_em(x, h).max() == n, h
  # the highest peak of each label survives every h, marked by the plateau of R at its top: with h above
  # the label's whole range of f that plateau is the label
  lab = np.array([1, 1, 1, 2, 2, 2], np.uint8)
  assert cc.restate_em(x, 0.5, lab).tolist() == [0, 1, 0, 2, 0, 0]
  assert cc.restate_em(x, 100.0, lab).tolist() == [1, 1, 1, 2, 2, 2]


def _defect_volumes():
  """(defect, function of (defect) -> output): one volume per defect on which it shows."""
  diag = np.array([[1, 0], [0, 1]], np.uint8)
  line = np.array([[1, 1, 0, 1]], np.uint8)
  nz = np.array([-1, -0.0, 0.0, -1], np.float32)                       # one plateau of -0.0 and +0.0
  nan = np.array([0, 1, np.nan, 2, 0], np.float32)
  plateau = np.array([0, 2, 2, 1, 2, 0], np.float32)
  return [
    ("connectivity_plus_one", lambda d: cc.restate_cc(diag, 1, defect=d)),
    ("connectivity_minus_one", lambda d: cc.restate_cc(diag, 2, defect=d)),
    ("numbered_backwards", lambda d: cc.restate_cc(line, 1, defect=d)),
    ("ge_in_marking", lambda d: cc.restate_em(plateau, 0.0, defect=d)),
    ("negative_zero_apart", lambda d: cc.restate_em(nz, 0.0, defect=d)),
    ("nan_as_plus_inf", lambda d: cc.restate_em(nan, 0.0, defect=d)),
  ]


@pytest.mark.parametrize("defect,run", _defect_volumes(), ids=[d[0] for d in _defect_volumes()])
def test_every_planted_defect_is_caught(defect, run):
  assert defect in cc.DEFECTS
  assert not np.array_equal(run(defect), run(None)), defect


@pytest.mark.parametrize("how", ["scipy", "bfs", "csgraph"])
def test_every_component_restatement_plants_the_graph_defects(how):
  rng = np.random.default_rng(3)
  lab = cc.random_labels(rng, (12, 14), nlabels=2, block=1, p=0.3)
  want = cc.restate_cc(lab, 1, how=how)
  for defect in ("connectivity_plus_one", "numbered_backwards"):
    assert not np.array_equal(cc.restate_cc(lab, 1, how=how, defect=defect), want), (how, defect)


def test_crossing_tiles_are_one_component_each():
  for name, lab, conn in cc.crossing_tiles():
    out = cc.restate_cc(lab, conn)
    assert out.max() == 1 and cc.restate_cc(lab, conn, how="bfs").max() == 1, name
