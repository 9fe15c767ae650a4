"""CPU tests of the two numpy restatements of nearest_labels (nearest_labels_cases.py): the per-pass rule and
the per-label one agree on the values always, and on the labels with integer weights (elsewhere only where
the k-th value is tied); the per-label values are the brute-force squared distances for integer weights; a
U-Net weight map from k = 2 equals one built from scipy's distance_transform_edt per label; and every
planted defect of the per-pass rule is caught by a case of the GPU suite's families."""
import numpy as np
import pytest

import nearest_labels_cases as nc

INTEGER_WEIGHTS = [(1.0, 1.0, 1.0), (2.0, 1.0, 3.0), (1.0, 4.0, 1.0)]
OTHER_WEIGHTS = [(0.7, 1.3, 2.9), (0.1, 0.3, 0.7), (1.1, 0.9, 1.7), (1e20, 1.0, 1.0), (1.0, 1e20, 0.5)]
DTYPES = [np.uint8, np.int16, np.uint32, np.int64, np.bool_]


def _cases(weights, seed):
  rng = np.random.default_rng(seed)
  for family in nc.FAMILIES:
    for k in (1, 2, 3, 4):
      for i, w in enumerate(weights):
        dtype = DTYPES[(k + i) % len(DTYPES)]
        yield family, k, w, nc.volume(family, (6, 9, 11), dtype, rng)


@pytest.mark.parametrize("d", [2.5, 4.5, 7.0])
def test_integer_weights_agree_exactly(d):
  for family, k, w, lab in _cases(INTEGER_WEIGHTS, int(d * 10)):
    a = nc.per_pass(lab, d, w, k)
    b = nc.per_label(lab, d, w, k)
    assert nc.same_bits(a[0], b[0]), (family, k, w)
    assert nc.same_bits(a[1], b[1]), (family, k, w)


@pytest.mark.parametrize("d", [2.5, 4.5, 7.0])
def test_other_weights_agree_on_values_and_on_labels_but_at_ties(d):
  for family, k, w, lab in _cases(OTHER_WEIGHTS, int(d * 10) + 1):
    a = nc.per_pass(lab, d, w, k)
    b = nc.per_label(lab, d, w, k)
    assert nc.same_bits(a[0], b[0]), (family, k, w)
    differ = a[1] != b[1]
    tied = a[0] == a[0][k - 1][None]
    assert not np.any(differ & ~tied), (family, k, w)


@pytest.mark.parametrize("w", INTEGER_WEIGHTS, ids=str)
def test_per_label_is_the_brute_force_squared_distance(w):
  rng = np.random.default_rng(int(sum(w)))
  for family in nc.FAMILIES:
    lab = nc.volume(family, (5, 7, 8), np.uint16, rng)
    ids, D = nc.per_label_values(lab, w)
    ids2, S = nc.brute_sqdist(lab, w)
    assert np.array_equal(ids, ids2)
    assert np.array_equal(D.astype(np.float64), np.where(np.isinf(D), np.inf, S)), family
    assert not np.any(np.isinf(D) & np.isfinite(S))


def test_unet_weight_map_matches_scipy():
  from scipy import ndimage
  rng = np.random.default_rng(8)
  w0, sigma = 10.0, 5.0
  for _ in range(6):
    cells = nc.volume("seeds", (40, 50), np.uint16, rng)
    d, _ = nc.per_pass(cells, 200.0, None, 2, squared=False)
    mine = np.where(cells == 0, w0 * np.exp(-(d[0].astype(np.float64) + d[1]) ** 2 / (2 * sigma ** 2)), 0)
    ids = np.unique(cells[cells != 0])
    per = np.sort(np.stack([ndimage.distance_transform_edt(cells != m) for m in ids]), axis=0)
    d1, d2 = per[0], per[1] if len(ids) > 1 else np.full(cells.shape, np.inf)
    want = np.where(cells == 0, w0 * np.exp(-(d1 + d2) ** 2 / (2 * sigma ** 2)), 0)
    np.testing.assert_allclose(mine, want, rtol=1e-5, atol=1e-30)


def _gpu_suite_family_cases():
  """The cases of test_nearest_labels_gpu.py::test_k_width_and_family."""
  dtypes = [np.uint8, np.uint16, np.uint32, np.uint64, np.bool_, np.int8, np.int16, np.int32, np.int64]
  for di, dtype in enumerate(dtypes):
    for k in (1, 2, 3, 4):
      for fi, family in enumerate(nc.FAMILIES):
        rng = np.random.default_rng(100 * di + 10 * k + fi)
        yield (family, k, np.dtype(dtype).name), nc.volume(family, (9, 13, 17), dtype, rng), k


@pytest.mark.parametrize("defect", nc.DEFECTS)
def test_each_defect_is_caught_by_the_gpu_families(defect):
  caught = []
  for name, lab, k in _gpu_suite_family_cases():
    a = nc.per_pass(lab, 4.5, (1.0, 2.0, 1.0), k)
    b = nc.per_pass(lab, 4.5, (1.0, 2.0, 1.0), k, defect=defect)
    if not (nc.same_bits(a[0], b[0]) and nc.same_bits(a[1], b[1])):
      caught.append(name)
    if len(caught) >= 3:
      break
  assert caught, defect
