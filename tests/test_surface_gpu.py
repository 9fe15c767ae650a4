"""GPU tests: surface_distances and the metrics formed from it against the numpy / scipy restatement
of tests/surface_cases.py.

With integer anisotropy every sorted segment equals scipy's float64 distances cast to float32 bit for
bit (sqrt rounded from 53 to 24 bits, which double rounding cannot change); with other anisotropy
every segment equals the library's own edt of the surface mask at those voxels, bit for bit.  Metrics
match the restatement within rtol 1e-12.
"""
import numpy as np
import pytest

import surface_cases as sc

pytestmark = pytest.mark.gpu


def _segments(sd, count=1):
  """[volume][key] -> (A->B, B->A) from a SurfaceDistances of numpy arrays."""
  nkeys = len(sd.labels)
  off, val = np.asarray(sd.offsets), np.asarray(sd.values)
  return [[(val[off[(v * nkeys + k) * 2]:off[(v * nkeys + k) * 2 + 1]],
            val[off[(v * nkeys + k) * 2 + 1]:off[(v * nkeys + k) * 2 + 2]]) for k in range(nkeys)]
          for v in range(count)]


def _assert_segments_equal(got, want):
  for k, ((gab, gba), (wab, wba)) in enumerate(zip(got, want)):
    assert gab.dtype == np.float32 and np.array_equal(gab, wab), ("A->B", k, gab[:8], wab[:8])
    assert np.array_equal(gba, wba), ("B->A", k, gba[:8], wba[:8])


def _check_metrics(edt, a, b, keys, anisotropy, stacked=False, segs=None):
  """The metrics against the restatement's, formed from `segs` ([volume][key] -> (A->B, B->A)): by
  default scipy's distances, which equal the library's with integer anisotropy only."""
  vols = list(zip(a, b)) if stacked else [(a, b)]
  if segs is None:
    segs = [sc.segments(x, y, keys, anisotropy) for x, y in vols]
  kw = dict(labels=keys, stacked=stacked)

  def per(fn, **m):
    return [np.array([fn(ab, ba, **m) for ab, ba in vol], np.float64) for vol in segs]
  want = {
    "hd": per(sc.hausdorff),
    "hd95": per(sc.hausdorff, percentile=95),
    "hd95d": per(sc.hausdorff, percentile=95, directed=True),
    "hd37": per(sc.hausdorff, percentile=37.5),
    "asd": per(sc.average),
    "assd": per(sc.average, symmetric=True),
    "dice": per(sc.dice, tolerance=1.5),
  }
  got = {
    "hd": edt.hausdorff_distance(a, b, anisotropy, **kw),
    "hd95": edt.hausdorff_distance(a, b, anisotropy, percentile=95, **kw),
    "hd95d": edt.hausdorff_distance(a, b, anisotropy, percentile=95, directed=True, **kw),
    "hd37": edt.hausdorff_distance(a, b, anisotropy, percentile=37.5, **kw),
    "asd": edt.average_surface_distance(a, b, anisotropy, **kw),
    "assd": edt.average_surface_distance(a, b, anisotropy, symmetric=True, **kw),
    "dice": edt.surface_dice(a, b, 1.5, anisotropy, **kw),
  }
  for m, w in want.items():
    w = np.stack(w) if stacked else w[0]
    g = got[m]
    assert isinstance(g, np.ndarray) and g.dtype == np.float64 and g.shape == w.shape, (m, g.shape, w.shape)
    np.testing.assert_allclose(g, w, rtol=1e-12, err_msg=m)


DTYPES = [np.uint8, np.uint16, np.int16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]
SHAPES = [(40,), (17, 23), (12, 9, 14), (1, 7, 5), (6, 1, 9)]


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("dtype", DTYPES, ids=[np.dtype(d).name for d in DTYPES])
@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
def test_integer_anisotropy_equals_scipy(edt, shape, dtype, order):
  rng = np.random.default_rng(sum(shape) * 7 + np.dtype(dtype).itemsize)
  a, b = sc.random_pair(rng, shape, nlabels=4, dtype=np.int64, flips=0.1)
  if np.dtype(dtype).kind == "i":
    a, b = np.where(a == 3, -3, a), np.where(b == 3, -3, b)       # a negative label
  a, b = a.astype(dtype), b.astype(dtype)
  b[b == 4] = 0                                                    # key 4 only in a
  if np.dtype(dtype).kind == "f":
    a[a == 2] = 2.5
    b[b == 2] = 2.5
  a, b = np.asarray(a, order=order), np.asarray(b, order=order)
  anisotropy = tuple([1.0, 2.0, 3.0][:len(shape)])
  sd = edt.surface_distances(a, b, anisotropy)
  keys = sc.default_keys(a, b)
  assert sd.labels.dtype == a.dtype and np.array_equal(sd.labels, keys)
  assert sd.offsets.dtype == np.int64 and sd.offsets.shape == (2 * len(keys) + 1,)
  _assert_segments_equal(_segments(sd)[0], sc.segments(a, b, keys, anisotropy))
  _check_metrics(edt, a, b, keys, anisotropy)


@pytest.mark.parametrize("shape,anisotropy", [((50,), (0.7,)), ((19, 21), (1.3, 0.45)),
                                              ((11, 13, 10), (0.7, 1.3, 2.9))])
def test_non_integer_anisotropy_equals_own_edt(edt, shape, anisotropy):
  rng = np.random.default_rng(11 + len(shape))
  a, b = sc.random_pair(rng, shape, nlabels=3, dtype=np.uint32, flips=0.1)
  keys = sc.default_keys(a, b)
  sd = edt.surface_distances(a, b, anisotropy)
  want = []
  for k in keys:
    sa, sb = sc.surface(a, k), sc.surface(b, k)
    da = edt.edt((~sa).astype(np.uint8), anisotropy) if sa.any() else np.full(shape, np.inf, np.float32)
    db = edt.edt((~sb).astype(np.uint8), anisotropy) if sb.any() else np.full(shape, np.inf, np.float32)
    want.append((np.sort(db[sa]), np.sort(da[sb])))
  _assert_segments_equal(_segments(sd)[0], want)
  _check_metrics(edt, a, b, keys, anisotropy, segs=[want])


def test_keys_given_in_caller_order_with_absent_keys(edt):
  rng = np.random.default_rng(3)
  a, b = sc.random_pair(rng, (14, 15, 9), nlabels=5, dtype=np.int32, flips=0.1)
  a[a == 5] = 0                        # 5 only in b
  keys = np.array([5, 2, 9, -7, 1], np.int32)    # 9 and -7 in neither volume
  sd = edt.surface_distances(a, b, labels=keys)
  assert np.array_equal(sd.labels, keys)
  _assert_segments_equal(_segments(sd)[0], sc.segments(a, b, keys, (1.0, 1.0, 1.0)))
  hd = edt.hausdorff_distance(a, b, labels=keys)
  assert hd[1] < np.inf and np.isnan(hd[2]) and np.isnan(hd[3]) and hd[0] == np.inf
  dice = edt.surface_dice(a, b, 2.0, labels=keys)
  assert dice[0] == 0.0 and np.isnan(dice[2])
  _check_metrics(edt, a, b, keys, (1.0, 1.0, 1.0))


def test_bool_labels_and_identical_volumes(edt):
  rng = np.random.default_rng(4)
  a = rng.random((20, 18)) < 0.5
  sd = edt.surface_distances(a, a)
  assert sd.labels.tolist() == [True]
  assert np.all(sd.values == 0) and sd.values.size == 2 * sc.surface(a, True).sum()
  assert edt.hausdorff_distance(a, a).tolist() == [0.0] and edt.surface_dice(a, a, 0.0).tolist() == [1.0]


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("vshape,anisotropy", [((30,), (2.0,)), ((13, 11), (1.0, 3.0)), ((7, 9, 8), (1.0, 2.0, 1.0)),
                                               ((9, 8, 7), (0.6, 1.1, 1.7))])
def test_stacked_equals_per_volume_calls(edt, vshape, anisotropy, order):
  rng = np.random.default_rng(len(vshape) + 20)
  pairs = [sc.random_pair(rng, vshape, nlabels=4, dtype=np.uint16, flips=0.1) for _ in range(5)]
  a, b = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
  b[3][b[3] == 2] = 0
  keys = sc.default_keys(a, b)
  if order == "F":      # the volume index is then the last axis
    af, bf = np.asfortranarray(np.moveaxis(a, 0, -1)), np.asfortranarray(np.moveaxis(b, 0, -1))
    sd = edt.surface_distances(af, bf, anisotropy, stacked=True)
    assert np.array_equal(edt.hausdorff_distance(af, bf, anisotropy, stacked=True),
                          edt.hausdorff_distance(a, b, anisotropy, stacked=True), equal_nan=True)
  else:
    sd = edt.surface_distances(a, b, anisotropy, stacked=True)
  assert np.array_equal(sd.labels, keys) and sd.offsets.shape == (len(pairs) * len(keys) * 2 + 1,)
  got = _segments(sd, len(pairs))
  for v, x in enumerate(a):
    one = edt.surface_distances(x, b[v], anisotropy, labels=keys)
    _assert_segments_equal(got[v], _segments(one)[0])
  if anisotropy == tuple(int(w) for w in anisotropy):
    for v, x in enumerate(a):
      _assert_segments_equal(got[v], sc.segments(x, b[v], keys, anisotropy))
  for m in ("hausdorff_distance", "average_surface_distance"):
    st = getattr(edt, m)(a, b, anisotropy, stacked=True)
    per = np.stack([getattr(edt, m)(x, y, anisotropy, labels=keys) for x, y in zip(a, b)])
    assert st.shape == (len(pairs), len(keys)) and np.array_equal(st, per, equal_nan=True), m
  _check_metrics(edt, a, b, keys, anisotropy, stacked=True, segs=got)


def test_small_budget_runs_many_groups_with_the_same_output(edt):
  import ctypes
  import torch
  rng = np.random.default_rng(9)
  a, b = sc.random_pair(rng, (3, 16, 12, 10), nlabels=6, dtype=np.uint32, flips=0.1)
  one = edt.surface_distances(a, b, (1.0, 2.0, 1.0), stacked=True)
  vol = 16 * 12 * 10
  for budget in (vol * 5, vol * 5 * 3 + 7, vol * 5 * 8):
    many = edt.surface_distances(a, b, (1.0, 2.0, 1.0), stacked=True, max_device_bytes=budget)
    assert np.array_equal(many.offsets, one.offsets) and np.array_equal(many.values, one.values), budget
  # the group count, and ENOMEM naming the least budget, through the C ABI
  ta, tb = torch.from_numpy(a.view(np.int32)).cuda(), torch.from_numpy(b.view(np.int32)).cuda()
  keys = np.arange(1, 7, dtype=np.uint32)
  nseg = 3 * 6 * 2
  counts = torch.zeros(nseg, dtype=torch.int64, device="cuda")
  lib = edt._lib()
  assert lib.edtb200_surface_count(ta.data_ptr(), tb.data_ptr(), 4, 3, 10, 12, 16, 3, keys.ctypes.data, 6, 12,
                                   counts.data_ptr(), 0, None) == 0
  offsets = torch.zeros(nseg + 1, dtype=torch.int64, device="cuda")
  offsets[1:] = torch.cumsum(counts, 0)
  values = torch.empty(int(offsets[-1]), dtype=torch.float32, device="cuda")
  groups = (ctypes.c_int64 * 1)()
  for budget, want in ((vol * 5, nseg), (vol * 5 * 8, 5), (vol * 5 * nseg, 1)):
    assert lib.edtb200_surface_distances(ta.data_ptr(), tb.data_ptr(), 4, 3, 10, 12, 16, 3, 1.0, 2.0, 1.0,
                                         keys.ctypes.data, 6, 12, offsets.data_ptr(), values.data_ptr(), 0, budget,
                                         groups, None) == 0
    assert groups[0] == want, (budget, groups[0])
  rc = lib.edtb200_surface_distances(ta.data_ptr(), tb.data_ptr(), 4, 3, 10, 12, 16, 3, 1.0, 2.0, 1.0,
                                     keys.ctypes.data, 6, 12, offsets.data_ptr(), values.data_ptr(), 0, vol * 5 - 1,
                                     groups, None)
  assert rc == -3 and groups[0] == 0 and (b"at least %d bytes" % (vol * 5)) in lib.edtb200_last_error()
  torch.cuda.synchronize()


def test_torch_input_returns_torch_tensors(edt):
  import torch
  rng = np.random.default_rng(12)
  a, b = sc.random_pair(rng, (10, 12, 14), nlabels=4, dtype=np.int32, flips=0.1)
  keys = sc.default_keys(a, b)
  ta, tb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
  sd = edt.surface_distances(ta, tb, (1.0, 2.0, 3.0))
  for x in sd:
    assert isinstance(x, torch.Tensor) and x.is_cuda
  assert sd.values.dtype == torch.float32 and sd.offsets.dtype == torch.int64
  host = edt.surface_distances(a, b, (1.0, 2.0, 3.0))
  assert np.array_equal(sd.labels.cpu().numpy(), host.labels)
  assert np.array_equal(sd.offsets.cpu().numpy(), host.offsets)
  assert np.array_equal(sd.values.cpu().numpy(), host.values)
  hd = edt.hausdorff_distance(ta, tb, (1.0, 2.0, 3.0), percentile=95)
  assert isinstance(hd, torch.Tensor) and hd.is_cuda and hd.dtype == torch.float64
  np.testing.assert_allclose(hd.cpu().numpy(), sc.metric(a, b, keys, (1.0, 2.0, 3.0), sc.hausdorff, percentile=95),
                             rtol=1e-12)
  dice = edt.surface_dice(ta, b, 1.0, (1.0, 2.0, 3.0), labels=keys)          # b goes up to a's device
  assert isinstance(dice, torch.Tensor) and dice.is_cuda
  np.testing.assert_allclose(dice.cpu().numpy(), sc.metric(a, b, keys, (1.0, 2.0, 3.0), sc.dice, tolerance=1.0),
                             rtol=1e-12)
  tf = ta.permute(2, 1, 0)           # an F-ordered view
  asd = edt.average_surface_distance(tf, tb.permute(2, 1, 0), (3.0, 2.0, 1.0))
  np.testing.assert_allclose(asd.cpu().numpy(), sc.metric(a, b, keys, (1.0, 2.0, 3.0), sc.average), rtol=1e-12)
