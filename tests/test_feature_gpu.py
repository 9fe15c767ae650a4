"""GPU tests (-m gpu) of feature_transform and expand_labels: the distances equal edt / sdf bit for
bit, the sites satisfy the site contract of tests/feature_cases.py against the oracle, on large
workload volumes against the library's own edtsq, against scipy's return_indices, and expand_labels
against a scipy restatement of skimage's algorithm."""
import os
import zlib

import numpy as np
import pytest

import feature_cases as fc

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
EDGES = os.path.join(HERE, "golden", "rounding_edges.npz")
ANISO = {"int": (1.0, 2.0, 3.0), "real": (0.7, 1.3, 2.9), "dyadic": (0.5, 0.25, 2.0)}
DTYPES = (np.uint8, np.uint16, np.uint32, np.uint64, np.int64, np.bool_, np.float32, np.float64)


def volume(rng, shape, dtype, kind):
  """Labels 0..2 in runs along the first axis ("blocks"), or iid ("noise")."""
  if kind == "noise":
    lab = rng.integers(0, 3, shape)
  else:
    lab = rng.integers(0, 3, tuple(max(1, s // 3) for s in shape))
    for ax, s in enumerate(shape):
      lab = np.repeat(lab, -(-s // lab.shape[ax]), axis=ax)
    lab = lab[tuple(slice(0, s) for s in shape)]
  lab = lab.astype(np.uint8)
  if dtype == np.bool_:
    return lab > 0
  if np.dtype(dtype).kind == "f":
    out = lab.astype(dtype)
    out[lab == 0] = -0.0                      # -0.0 is background too
    return out
  return (lab.astype(np.uint64) * np.uint64(0x1000001)).astype(dtype) if np.dtype(dtype).itemsize > 1 else lab


def oracle_sq(oracle, lab, an, border, signed):
  if signed:
    return np.abs(oracle.sdfsq(lab, anisotropy=an, black_border=border))
  return oracle.edtsq(lab, anisotropy=an, black_border=border)


def run_case(edt, oracle, lab, an, border, signed):
  dist, idx = edt.feature_transform(lab, an, border, signed=signed, return_distances=True)
  want = (edt.sdf if signed else edt.edt)(lab, an, border)
  assert dist.dtype == np.float32 and idx.dtype == np.int32 and idx.shape == (lab.ndim,) + lab.shape
  assert np.array_equal(dist.view(np.uint32), want.view(np.uint32)), "distances differ from %s" % (
    "sdf" if signed else "edt")
  fortran = lab.flags.f_contiguous and not lab.flags.c_contiguous
  for k in range(lab.ndim):      # each plane in the input's memory order
    assert (idx[k].flags.f_contiguous if fortran else idx[k].flags.c_contiguous), k
  only = edt.feature_transform(lab, an, border, signed=signed)
  assert np.array_equal(only, idx), "indices depend on return_distances"
  fc.check_sites(lab, idx, oracle_sq(oracle, lab, an, border, signed), an, border, signed)
  return idx


def cases():
  """(name, shape, dtype, kind, anisotropy class, order)"""
  out = []
  for i, dtype in enumerate(DTYPES):
    for nd, shape in ((1, (61,)), (2, (23, 37)), (3, (17, 13, 21))):
      out.append(("%s-%dd" % (np.dtype(dtype).name, nd), shape, dtype, ("blocks", "noise")[i % 2],
                  ("int", "real", "dyadic")[(i + nd) % 3], ("C", "F")[(i + nd) % 2]))
  out.append(("long-x", (3, 4500), np.uint32, "blocks", "real", "C"))
  out.append(("long-y", (4200, 3), np.uint16, "blocks", "int", "C"))
  out.append(("long-z", (4100, 2, 3), np.uint8, "blocks", "dyadic", "C"))
  out.append(("long-1d", (9000,), np.uint8, "blocks", "real", "C"))
  return out


@pytest.mark.parametrize("case", cases(), ids=lambda c: c[0])
def test_distances_and_sites(edt, oracle, case):
  name, shape, dtype, kind, acls, order = case
  rng = np.random.default_rng(zlib.crc32(name.encode()))
  lab = volume(rng, shape, dtype, kind)
  lab = np.asfortranarray(lab) if order == "F" else np.ascontiguousarray(lab)
  an = ANISO[acls][:len(shape)]
  for border in (False, True):
    for signed in (False, True):
      run_case(edt, oracle, lab, an, border, signed)


def test_double_rounding_tie(edt, oracle):
  """tie2d takes the all-double branch of the later pass."""
  z = np.load(EDGES)
  lab = z["tie2d_labels"]
  an = tuple(float(a) for a in z["tie2d_aniso"])
  bb = bool(z["tie2d_border"])
  for signed in (False, True):
    run_case(edt, oracle, lab, an, bb, signed)
    run_case(edt, oracle, lab, an, not bb, signed)


def test_exact_distance_to_site_is_bruteforce(edt, oracle):
  """Integer anisotropy: the exact squared distance to each site is the brute-force edtsq."""
  rng = np.random.default_rng(5)
  for k in range(6):
    shape = tuple(int(s) for s in rng.integers(2, 7, 3))
    lab = rng.integers(0, 3, shape).astype(np.uint32)
    an = (1.0, 2.0, 3.0)
    for border in (False, True):
      idx = edt.feature_transform(lab, an, border).astype(np.float64)
      p = np.indices(shape)
      exact = sum((an[k] * (idx[k] - p[k])) ** 2 for k in range(3))
      want = oracle.bruteforce_edtsq(lab, anisotropy=an, black_border=border)
      live = np.isfinite(want)
      assert np.array_equal(exact[live], want[live].astype(np.float64)), (k, border)


def check_sites_torch(torch, lab, idx, sq, an, border, signed):
  """check_sites on the device, for C-ordered (z, y, x) tensors, with the site values in float64."""
  nd = lab.dim()
  shape = tuple(lab.shape)
  none = (idx == -1).all(0) & (not border)
  assert torch.equal(none, torch.isinf(sq))
  p = torch.stack(torch.meshgrid(*[torch.arange(s, device=lab.device) for s in shape], indexing="ij"))
  bg = lab == 0
  if not signed:
    assert bool(((idx == p).all(0) | ~bg).all())
  live = ~none & (bg.logical_not() if not signed else torch.ones_like(bg))
  dims = torch.tensor(shape, device=lab.device).view((nd,) + (1,) * nd)
  out = (idx < 0) | (idx >= dims)
  nout = out.sum(0)
  face = live & (nout > 0)
  if bool(face.any()):
    assert border and bool((nout[face] == 1).all())
    assert bool(((idx == -1) | (idx == dims) | ~out).all())
  inside = live & (nout == 0)
  q = torch.where(inside, idx.long(), p)
  assert bool((lab[tuple(q)][inside] != lab[inside]).all())
  qv = torch.where(none, p, idx.long())
  v = fc.values(p, qv, shape, an, "C", xp=torch)
  bad = live & (v.view(torch.int32) != sq.view(torch.int32))
  assert not bool(bad.any()), int(bad.sum())


@pytest.mark.parametrize("name", ["cfg2", "cfg2b", "balls", "voronoi", "ones_nobb"])
def test_large_workloads(edt, name):
  import torch
  from edt_b200 import workloads
  lab, an, bb = workloads.generate(name, 256, "cuda")
  for signed in ((False, True) if name == "cfg2b" else (False,)):
    dist, idx = edt.feature_transform(lab, an, bb, signed=signed, return_distances=True)
    want = edt.sdf(lab, an, bb) if signed else edt.edt(lab, an, bb)
    assert torch.equal(dist.view(torch.int32), want.view(torch.int32))
    sq = edt.sdfsq(lab, an, bb).abs() if signed else edt.edtsq(lab, an, bb)
    check_sites_torch(torch, lab, idx, sq, an, bb, signed)
    del dist, idx, want, sq
  torch.cuda.empty_cache()


@pytest.mark.parametrize("sampling", [(1.0, 1.0, 1.0), (1.0, 2.0, 3.0), (2.0, 1.0)])
def test_scipy_return_indices(edt, sampling):
  ndi = pytest.importorskip("scipy.ndimage")
  rng = np.random.default_rng(11)
  shape = (40, 33, 29)[:len(sampling)]
  lab = (rng.random(shape) < 0.97).astype(np.uint8)
  lab[(0,) * len(shape)] = 0
  dist, idx = edt.feature_transform(lab, sampling, return_distances=True)
  sd, si = ndi.distance_transform_edt(lab, sampling=sampling, return_indices=True)
  np.testing.assert_allclose(dist, sd, rtol=1e-6)
  p = np.indices(shape)
  w = np.array(sampling).reshape((len(shape),) + (1,) * len(shape))
  ours = ((w * (idx - p)) ** 2).sum(0)
  theirs = ((w * (si - p)) ** 2).sum(0)
  diff = (idx != si).any(0)
  assert np.array_equal(ours[diff], theirs[diff])


@pytest.mark.parametrize("order", ["C", "F"])
def test_expand_labels(edt, order):
  pytest.importorskip("scipy.ndimage")
  import torch
  rng = np.random.default_rng(13)
  for shape, spacing, dtype in (((50, 40), (1.0, 2.0), np.uint16), ((30, 31, 32), (1.0, 1.0, 3.0), np.int32),
                                ((64,), (1.0,), np.uint64)):
    lab = np.where(rng.random(shape) < 0.02, rng.integers(1, 9, shape), 0).astype(dtype)
    lab[(0,) * len(shape)] = 3
    lab = np.asfortranarray(lab) if order == "F" else np.ascontiguousarray(lab)
    for distance in (0.0, 1.0, 2.5, 7.5):
      got = edt.expand_labels(lab, distance, spacing)
      assert got.dtype == lab.dtype and got.shape == lab.shape
      assert got.flags.f_contiguous == lab.flags.f_contiguous
      want, sidx = fc.skimage_expand(lab, distance, spacing)
      ours = edt.feature_transform(lab, spacing, signed=True)
      fc.check_expand(lab, got, ours, want, sidx, distance, spacing)
      t = torch.from_numpy(lab.view(np.dtype("i%d" % lab.dtype.itemsize))).cuda()
      dev = edt.expand_labels(t, distance, spacing)
      assert dev.is_cuda and dev.stride() == t.stride()
      assert np.array_equal(dev.cpu().numpy().view(lab.dtype), got)


def test_device_input_on_side_stream(edt):
  import torch
  rng = np.random.default_rng(17)
  for order in ("C", "F"):
    lab = rng.integers(0, 4, (40, 30, 20)).astype(np.int32)
    lab = np.asfortranarray(lab) if order == "F" else lab
    an = (1.0, 2.0, 3.0)
    hd, hi = edt.feature_transform(lab, an, True, signed=True, return_distances=True)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
      t = torch.from_numpy(lab).cuda()
      dd, di = edt.feature_transform(t, an, True, signed=True, return_distances=True)
    side.synchronize()
    assert dd.is_cuda and di.is_cuda and di.dtype == torch.int32
    assert np.array_equal(dd.cpu().numpy(), hd) and np.array_equal(di.cpu().numpy(), hi)
    assert di[0].stride() == t.stride()


def test_errors(edt):
  with pytest.raises(TypeError):
    edt.feature_transform(np.zeros((2, 2, 2, 2), np.uint8))
  with pytest.raises(ValueError):
    edt.feature_transform(np.zeros((3, 3), np.uint8), anisotropy=(1.0,))
  with pytest.raises(edt.EDTError, match="error -1"):          # EDTB200_EINVAL: no such device
    edt.feature_transform(np.ones((3, 3), np.uint8), device=4096)
  # EDTB200_ELIMIT: an X line longer than the first-axis kernel's shared-memory line buffer
  with pytest.raises(edt.EDTError, match="error -4"):
    edt.feature_transform(np.ones(1 << 19, np.uint8))
