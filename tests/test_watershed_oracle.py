"""CPU tests of the watershed restatement (watershed_cases.py): it equals the brute-force definition, the
numpy-frontier flood and the model of the GPU's tile rounds on random tiny volumes for every connectivity;
worked examples (a constant image, strictly rising basins, two touching balls of -edt); and each planted
defect is caught."""
import numpy as np
import pytest

import watershed_cases as wc


def _same(a, b):
  return np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("shape", [(30,), (6, 7), (4, 5, 6)])
def test_the_restatement_equals_the_brute_force(shape, order):
  rng = np.random.default_rng(sum(shape) + (order == "F"))
  for conn in range(1, len(shape) + 1):
    for levels in (None, 3):
      img, mk, lab = wc.random_case(rng, shape, levels=levels, p=0.08)
      img.reshape(-1)[rng.integers(0, img.size, 3)] = [np.nan, np.inf, -np.inf]
      if order == "F":
        img, mk, lab = np.asfortranarray(img), np.asfortranarray(mk), np.asfortranarray(lab)
      for labels in (lab, None):
        want = wc.restate(img, mk, labels, conn, order)
        assert _same(want, wc.brute(img, mk, labels, conn, order)), (shape, conn, levels)
        assert _same(want, wc.flood(img, mk, labels, conn, order)), (shape, conn, levels)
        assert _same(want, wc.tiled(img, mk, labels, conn, order)), (shape, conn, levels)


def test_a_constant_image_gives_the_least_marker_of_each_component():
  lab = np.zeros((6, 9), np.uint8)
  lab[:, :4] = 1
  lab[:, 5:] = 1                   # the same label, cut in two
  lab[0, 4] = 2
  mk = np.zeros(lab.shape, np.int32)
  mk[1, 1], mk[4, 2], mk[2, 6], mk[5, 8] = 7, 3, 9, 4
  W, L = wc.restate(np.full(lab.shape, 2.5, np.float32), mk, lab)
  assert (W[:, :4][mk[:, :4] == 0] == 3).all() and W[1, 1] == 7
  assert (W[:, 5:][mk[:, 5:] == 0] == 4).all() and W[2, 6] == 9
  assert W[0, 4] == 0 and (W[lab == 0] == 0).all()
  assert (L[lab == 1] == 2.5).all() and L[0, 4] == np.inf and np.isinf(L[lab == 0]).all()


def test_strictly_rising_basins_give_the_basin_partition():
  """Altitude |x - c| around the nearest of three minima: every voxel goes to its own basin's marker, and
  the level is its own altitude."""
  x = np.arange(60)
  centres = np.array([8, 27, 50])
  basin = np.abs(x[:, None] - centres[None]).argmin(1)
  img = np.abs(x - centres[basin]).astype(np.float32) + 0.25 * basin
  img = np.tile(img, (5, 1))
  mk = np.zeros(img.shape, np.uint16)
  for k, c in enumerate(centres):
    mk[2, c] = 10 * (k + 1)
  for conn in (1, 2):
    W, L = wc.restate(img, mk, None, conn)
    ridge = np.isin(x, [17, 18, 38, 39])              # the voxels at the tops between two basins
    assert (W[:, ~ridge] == 10 * (basin[~ridge] + 1)).all()
    assert np.array_equal(L, img)


def test_two_touching_balls_of_minus_edt_split_at_the_neck():
  mask, mk = wc.balls((30, 30, 50), [(15, 15, 14), (15, 15, 30)], [10, 7])
  W, _ = wc.restate(wc.minus_edt(mask), mk, mask)
  row = W[15, 15]
  assert (row[4:24] == 1).all() and (row[26:38] == 2).all()
  assert set(np.unique(W[mask != 0])) == {1, 2} and (W[mask == 0] == 0).all()


def test_the_definition_examples_hold():
  img = np.array([0, 3, 1, 5, 2, 0], np.float32)
  mk = np.array([1, 0, 0, 0, 0, 2], np.uint8)
  W, L = wc.restate(img, mk)
  assert W.tolist() == [1, 1, 1, 1, 2, 2] and L.tolist() == [0, 3, 3, 5, 2, 0]


# ---- the planted defects ------------------------------------------------------------------------------

def test_seeds_overwritten_by_a_smaller_marker_is_caught():
  img = np.zeros((5, 6), np.float32)
  mk = np.zeros(img.shape, np.uint8)
  mk[2, 2], mk[2, 3] = 6, 1
  good = wc.restate(img, mk)
  bad = wc.restate(img, mk, defect="seeds_overwritten")
  assert good[0][2, 2] == 6 and bad[0][2, 2] == 1


def test_propagation_over_non_tight_edges_is_caught():
  img = np.array([[0, 1, 5, 1, 0, 9, 0]], np.float32)
  mk = np.array([[1, 0, 0, 0, 2, 0, 0]], np.uint8)
  good = wc.restate(img, mk)
  bad = wc.restate(img, mk, defect="non_tight")
  assert good[0].tolist() == [[1, 1, 1, 2, 2, 2, 2]] and not np.array_equal(good[0], bad[0])


@pytest.mark.parametrize("nd", [2, 3])
def test_connectivity_off_by_one_is_caught(nd):
  rng = np.random.default_rng(nd)
  caught = 0
  for _ in range(5):
    img, mk, lab = wc.random_case(rng, (7,) * nd, levels=4)
    good = wc.restate(img, mk, lab, 1)
    caught += not _same(good, wc.restate(img, mk, lab, 1, defect="connectivity_plus_one"))
  assert caught >= 3


def test_nan_not_read_as_plus_inf_is_caught():
  img = np.array([0, 2, np.nan, 2, 0], np.float32)
  mk = np.array([1, 0, 0, 0, 2], np.uint8)
  good = wc.restate(img, mk)
  bad = wc.restate(img, mk, defect="nan_as_minus_inf")
  assert good[1][2] == np.inf and bad[1][2] == 2 and not _same(good, bad)


@pytest.mark.parametrize("name,img,mk,lab,conn", [c for c in wc.seeded_at_tile_borders() if c[0].startswith("diag")],
                         ids=[c[0] for c in wc.seeded_at_tile_borders() if c[0].startswith("diag")])
def test_round_1_not_queuing_across_a_tile_corner_is_caught(name, img, mk, lab, conn):
  good = wc.restate(img, mk, lab, conn)
  assert _same(good, wc.tiled(img, mk, lab, conn))
  assert not _same(good, wc.tiled(img, mk, lab, conn, defect="round1_no_corner"))
