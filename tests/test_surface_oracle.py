"""CPU tests: the numpy / scipy restatement of the surface distances (surface_cases.py) against an
O(N^2) brute force of the definitions on small 1-D, 2-D and 3-D volumes, empty surfaces included.
The GPU tests then compare the library with that restatement."""
import itertools

import numpy as np
import pytest

import surface_cases as sc


def brute_surface(vol, key):
  """Voxels of label `key` with a face neighbour of another label, or on a face of the volume."""
  vol = np.asarray(vol)
  out = np.zeros(vol.shape, bool)
  for p in itertools.product(*(range(s) for s in vol.shape)):
    if vol[p] != key:
      continue
    for ax in range(vol.ndim):
      for step in (-1, 1):
        q = list(p)
        q[ax] += step
        if not 0 <= q[ax] < vol.shape[ax] or vol[tuple(q)] != key:
          out[p] = True
  return out


def brute_distances(from_surf, to_surf, anisotropy):
  """float64 distance from every voxel of from_surf to the nearest voxel of to_surf (inf: none)."""
  w = np.asarray(anisotropy, np.float64)
  src = np.argwhere(from_surf).astype(np.float64)
  dst = np.argwhere(to_surf).astype(np.float64)
  if dst.size == 0:
    return np.full(len(src), np.inf)
  d = ((src[:, None, :] - dst[None, :, :]) * w) ** 2
  return np.sqrt(d.sum(-1).min(1))


def brute_percentile(x, p):
  x = np.sort(x)
  pos = (len(x) - 1) * p / 100.0
  lo = int(np.floor(pos))
  hi = min(lo + 1, len(x) - 1)
  return x[lo] + (x[hi] - x[lo]) * (pos - lo)


def brute_metrics(a, b, key, anisotropy, tau, p):
  sa, sb = brute_surface(a, key), brute_surface(b, key)
  if not sa.any() and not sb.any():
    return dict(hd=np.nan, hd95=np.nan, asd=np.nan, assd=np.nan, dice=np.nan)
  if not sa.any() or not sb.any():
    return dict(hd=np.inf, hd95=np.inf, asd=np.inf, assd=np.inf, dice=0.0)
  ab = brute_distances(sa, sb, anisotropy).astype(np.float32).astype(np.float64)
  ba = brute_distances(sb, sa, anisotropy).astype(np.float32).astype(np.float64)
  return dict(hd=max(ab.max(), ba.max()), hd95=max(brute_percentile(ab, p), brute_percentile(ba, p)),
              asd=ab.sum() / len(ab), assd=(ab.sum() + ba.sum()) / (len(ab) + len(ba)),
              dice=((ab <= tau).sum() + (ba <= tau).sum()) / (len(ab) + len(ba)))


CASES = [
  ("1d", (23,), (1.0,)),
  ("1d_scaled", (19,), (2.5,)),
  ("2d", (9, 11), (1.0, 1.0)),
  ("2d_aniso", (8, 10), (2.0, 0.7)),
  ("3d", (6, 7, 5), (1.0, 2.0, 3.0)),
  ("3d_frac", (5, 6, 7), (0.9, 1.3, 2.1)),
]


@pytest.mark.parametrize("name,shape,anisotropy", CASES, ids=[c[0] for c in CASES])
def test_restatement_matches_brute_force(name, shape, anisotropy):
  rng = np.random.default_rng(len(shape) * 100 + shape[0])
  a, b = sc.random_pair(rng, shape, nlabels=3, flips=0.15)
  keys = list(sc.default_keys(a, b)) + [7]                # 7: in neither volume
  for k in keys:
    assert np.array_equal(sc.surface(a, k), brute_surface(a, k)), k
  segs = sc.segments(a, b, keys, anisotropy)
  for k, (ab, ba) in zip(keys, segs):
    sa, sb = brute_surface(a, k), brute_surface(b, k)
    if sa.any() and sb.any():
      np.testing.assert_allclose(ab, np.sort(brute_distances(sa, sb, anisotropy)).astype(np.float32), rtol=1e-6)
      np.testing.assert_allclose(ba, np.sort(brute_distances(sb, sa, anisotropy)).astype(np.float32), rtol=1e-6)
    want = brute_metrics(a, b, k, anisotropy, tau=1.5, p=95)
    got = dict(hd=sc.hausdorff(ab, ba), hd95=sc.hausdorff(ab, ba, 95), asd=sc.average(ab, ba),
               assd=sc.average(ab, ba, symmetric=True), dice=sc.dice(ab, ba, 1.5))
    for m in want:
      np.testing.assert_allclose(got[m], want[m], rtol=1e-12, err_msg="%s key %s" % (m, k))


def test_integer_anisotropy_distances_are_exact():
  """With integer weights scipy's float64 distance is sqrt of an exact integer, as is the brute force."""
  rng = np.random.default_rng(5)
  a, b = sc.random_pair(rng, (6, 8, 7), nlabels=3, flips=0.2)
  for k in sc.default_keys(a, b):
    sa, sb = brute_surface(a, k), brute_surface(b, k)
    if sa.any() and sb.any():
      ab, _ = sc.segments(a, b, [k], (1.0, 2.0, 3.0))[0]
      assert np.array_equal(ab, np.sort(brute_distances(sa, sb, (1.0, 2.0, 3.0)).astype(np.float32)))


def test_empty_surface_rules():
  a = np.zeros((5, 5), np.uint8)
  b = np.zeros((5, 5), np.uint8)
  a[1:3, 1:3] = 1
  ab, ba = sc.segments(a, b, [1], (1.0, 1.0))[0]
  assert ab.size == 4 and ba.size == 0
  assert sc.hausdorff(ab, ba) == np.inf and sc.hausdorff(ab, ba, 95, directed=True) == np.inf
  assert sc.average(ab, ba) == np.inf and sc.average(ab, ba, symmetric=True) == np.inf
  assert sc.dice(ab, ba, 10.0) == 0.0
  ab, ba = sc.segments(a, b, [2], (1.0, 1.0))[0]
  assert ab.size == 0 and ba.size == 0
  for v in (sc.hausdorff(ab, ba), sc.average(ab, ba), sc.dice(ab, ba, 1.0)):
    assert np.isnan(v)


def test_faces_count_as_surface():
  """A volume of one label is surface on its faces only; at size 2 along an axis every voxel is."""
  v = np.ones((4, 5, 6), np.uint8)
  s = sc.surface(v, 1)
  assert s.sum() == v.size - 2 * 3 * 4 and np.array_equal(s, brute_surface(v, 1))
  assert sc.surface(np.ones((2, 7), np.uint8), 1).all()
  assert np.array_equal(sc.surface(np.ones(3, np.uint8), 1), [True, False, True])
