"""CPU tests of the feature transform's site contract (tests/feature_cases.py): the brute-force
nearest site reaches exactly the oracle's distances, check_sites accepts it and rejects each kind of
wrong site, and the Python front door's argument handling that needs no device."""
import numpy as np
import pytest

import feature_cases as fc
from abi_checks import ABI_VERSION

ANISOTROPIES = ((1.0, 1.0, 1.0), (1.0, 2.0, 3.0), (0.7, 1.3, 2.9), (3.3, 3.3, 40.7))


def oracle_sq(oracle, lab, an, border, signed):
  if signed:
    return np.abs(oracle.sdfsq(lab, anisotropy=an, black_border=border))
  return oracle.edtsq(lab, anisotropy=an, black_border=border)


@pytest.mark.parametrize("an", ANISOTROPIES)
def test_bruteforce_minimum_is_the_oracle(oracle, an):
  rng = np.random.default_rng(int(sum(an) * 10))
  for k in range(15):
    shape = tuple(int(s) for s in rng.integers(1, 6, 3))
    lab = rng.integers(0, 3, shape).astype(np.uint8)
    for border in (False, True):
      for signed in (False, True):
        want = oracle_sq(oracle, lab, an, border, signed)
        dist, sites = fc.brute_sites(lab, an, border, signed)
        assert np.array_equal(dist, want), (k, shape, border, signed)
        fc.check_sites(lab, sites, want, an, border, signed)


@pytest.mark.parametrize("nd", [1, 2])
def test_bruteforce_lower_dimensions(oracle, nd):
  rng = np.random.default_rng(nd)
  for k in range(10):
    shape = tuple(int(s) for s in rng.integers(1, 7, nd))
    lab = rng.integers(0, 3, shape).astype(np.uint16)
    an = (1.3,) if nd == 1 else (0.7, 2.9)
    for border in (False, True):
      for signed in (False, True):
        want = oracle_sq(oracle, lab, an[0] if nd == 1 else an, border, signed)
        dist, sites = fc.brute_sites(lab, an, border, signed)
        assert np.array_equal(dist, want), (k, shape, border, signed)
        fc.check_sites(lab, sites, want, an, border, signed)


def test_fortran_order_axes():
  """In F order x is array axis 0: the same volume transposed gives transposed sites."""
  rng = np.random.default_rng(3)
  lab = rng.integers(0, 3, (4, 5, 3)).astype(np.uint8)
  an = (0.7, 1.3, 2.9)
  dist_c, sites_c = fc.brute_sites(lab, an, True, False, "C")
  lab_f = np.asfortranarray(lab.T)
  dist_f, sites_f = fc.brute_sites(lab_f, an[::-1], True, False, "F")
  assert np.array_equal(dist_f, dist_c.T)
  fc.check_sites(lab_f, sites_f, dist_f, an[::-1], True, False, "F")


def rejects(lab, sites, sq, an, border, signed, what):
  with pytest.raises(AssertionError, match=what):
    fc.check_sites(lab, sites, sq, an, border, signed)


def test_check_sites_rejects_planted_defects(oracle):
  an = (1.0, 1.0)
  # label 1 everywhere, label 2 in the last column: the site of (2, 2) is (2, 6)
  lab = np.ones((5, 7), np.uint8)
  lab[:, 6] = 2
  sq = oracle.edtsq(lab, anisotropy=an)
  _, sites = fc.brute_sites(lab, an, False, False)
  assert tuple(sites[:, 2, 2]) == (2, 6)
  fc.check_sites(lab, sites, sq, an, False, False)
  for planted, what in (((1, 6), "differs from the distance"),      # moved by one voxel
                        ((2, 3), "own label"),                        # a site of the same label
                        ((0, 6), "differs from the distance")):       # a farther site of the right label
    bad = sites.copy()
    bad[:, 2, 2] = planted
    rejects(lab, bad, sq, an, False, False, what)


def test_check_sites_rejects_direct_site_resolved_through_its_voxel(oracle):
  """(1, 3) lies under (0, 3), of label 2: that voxel is the site.  Following (0, 3)'s own
  first-axis site instead, (0, 5) of label 3, gives a site of another label but a larger value."""
  an = (1.0, 1.0)
  lab = np.ones((3, 7), np.uint8)
  lab[0, :] = 2
  lab[0, 5:] = 3
  sq = oracle.edtsq(lab, anisotropy=an)
  _, sites = fc.brute_sites(lab, an, False, False)
  assert tuple(sites[:, 1, 3]) == (0, 3)
  bad = sites.copy()
  bad[:, 1, 3] = (0, 5)
  rejects(lab, bad, sq, an, False, False, "differs from the distance")


def test_check_sites_rejects_face_site_without_border():
  an = (1.0, 1.0)
  lab = np.ones((3, 4), np.uint8)
  lab[:, 3] = 2
  dist, sites = fc.brute_sites(lab, an, True, False)
  assert tuple(sites[:, 1, 0]) == (1, -1)
  fc.check_sites(lab, sites, dist, an, True, False)
  # the same sites and their own values, claimed without black_border: only the face rule objects
  rejects(lab, sites, dist, an, False, False, "face site without black_border")


def test_check_sites_none_and_background():
  an = (1.0, 1.0)
  lab = np.ones((3, 3), np.uint8)
  dist, sites = fc.brute_sites(lab, an, False, False)
  assert np.isinf(dist).all() and (sites == -1).all()
  fc.check_sites(lab, sites, dist, an, False, False)
  lab[1, 1] = 0
  dist, sites = fc.brute_sites(lab, an, False, False)
  bad = sites.copy()
  bad[:, 1, 1] = (0, 1)
  rejects(lab, bad, dist, an, False, False, "background not mapped to itself")
  rejects(lab, sites, np.where(lab == 0, np.inf, dist).astype(np.float32), an, False, False, "'none' sites")


def expand_restated(lab, distance, sites, sq, square=True, order="C"):
  """expand_labels from given sites and squared distances, as the library forms it: a gather by
  C-order linear index from the labels flattened in `order` (right only for "C").  square=False
  compares the squared distance with `distance` itself."""
  limit = float(distance) ** 2 if square else float(distance)
  has = (sites >= 0).all(0)
  lin = np.ravel_multi_index(tuple(np.where(has, sites, 0)), lab.shape)
  grow = (lab == 0) & has & (sq.astype(np.float64) <= limit)
  return np.where(grow, lab.reshape(-1, order=order)[lin], lab)


def test_check_expand_rejects_wrong_expansions():
  """check_expand accepts an expansion grown from true nearest sites and rejects one that grows
  nothing, one that compares with `distance` instead of `distance**2`, and one whose gather takes
  the labels in the wrong memory order."""
  pytest.importorskip("scipy.ndimage")
  rng = np.random.default_rng(13)
  lab = np.where(rng.random((12, 15)) < 0.08, rng.integers(1, 9, (12, 15)), 0).astype(np.uint16)
  spacing = (1.0, 2.0)
  sq, sites = fc.brute_sites(lab, spacing, False, True)
  for distance in (1.0, 2.5, 7.5):
    want, sidx = fc.skimage_expand(lab, distance, spacing)
    fc.check_expand(lab, expand_restated(lab, distance, sites, sq), sites, want, sidx, distance, spacing)
    mutants = {"grows nothing": lab.copy(),
               "distance not squared": expand_restated(lab, distance, sites, sq, square=False),
               "gather in F order": expand_restated(lab, distance, sites, sq, order="F")}
    for what, bad in mutants.items():
      if np.array_equal(bad, want):
        assert what == "distance not squared" and distance == 1.0      # 1 == 1**2: nothing to tell apart
        continue
      with pytest.raises(AssertionError):
        fc.check_expand(lab, bad, sites, want, sidx, distance, spacing)


# ---- host-side argument handling (raises before any device is touched) ----

def test_feature_transform_argument_errors(edt):
  with pytest.raises(TypeError):
    edt.feature_transform(np.zeros((2, 2, 2, 2), np.uint8))
  with pytest.raises(TypeError):
    edt.feature_transform(np.zeros((3, 3), np.complex64))
  with pytest.raises(ValueError):
    edt.feature_transform(np.zeros((3, 3), np.uint8), anisotropy=(1.0, 2.0, 3.0))
  with pytest.raises(TypeError):
    edt.expand_labels(np.zeros((3, 3), np.complex64))


@pytest.mark.parametrize("shape", [(0,), (0, 3), (2, 0, 4)])
def test_feature_transform_empty(edt, shape):
  idx = edt.feature_transform(np.zeros(shape, np.uint8))
  assert idx.shape == (len(shape),) + shape and idx.dtype == np.int32
  dist, idx = edt.feature_transform(np.zeros(shape, np.float32), return_distances=True)
  assert dist.shape == shape and dist.dtype == np.float32 and idx.shape == (len(shape),) + shape


def test_feature_abi_argument_checks(edt):
  """EDTB200_EINVAL / EDTB200_ELIMIT come before any device is touched."""
  import ctypes
  lib = edt._lib()
  planes = (ctypes.c_void_p * 3)(1, 1, 1)
  dummy = ctypes.c_void_p(1)
  assert lib.edtb200_feature_transform(dummy, 3, 1, 4, 1, 1, 1.0, 1.0, 1.0, 0, 0, None, planes, 0, None) == -1
  assert lib.edtb200_feature_transform(dummy, 1, 4, 4, 1, 1, 1.0, 1.0, 1.0, 0, 0, None, planes, 0, None) == -1
  assert lib.edtb200_feature_transform(dummy, 1, 1, (1 << 30) + 1, 1, 1, 1.0, 1.0, 1.0, 0, 0, None, planes, 0,
                                       None) == -4
  assert lib.edtb200_feature_transform(dummy, 1, 1, 4, 1, 1, 1.0, 1.0, 1.0, 0, 0, None, None, 0, None) == -1


def test_feature_abi_version(edt):
  assert edt._lib().edtb200_version() == ABI_VERSION
