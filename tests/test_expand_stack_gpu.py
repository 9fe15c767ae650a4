"""GPU tests (-m gpu) of expand_labels on stacks and of its gather kernel (edtb200_expand_gather).

A stacked result must equal np.stack of the per-volume expand_labels calls bit for bit, for every
label width, bool and float32 labels (with -0.0 and NaN labels), 1-D to 3-D volumes, both memory
orders, integer and fractional anisotropy and distances 0, 1, 2.5, 7.5, inf, -1 and NaN.  Boundary
traps fail if a gather leaves its volume.  The gather kernel is also checked on its own against a numpy
restatement, and the single-volume device path against the chunked host path, whose gather is
independent numpy code.
"""
import ctypes

import numpy as np
import pytest

import feature_cases as fc

pytestmark = pytest.mark.gpu

LABELS_ON_DEVICE, OUT_ON_DEVICE, LABELS_FLOAT = 4, 8, 16
BOTH = LABELS_ON_DEVICE | OUT_ON_DEVICE
DISTANCES = (0.0, 1.0, 2.5, 7.5, float("inf"), -1.0, float("nan"))
NAN_BITS = 0x7fc00123                                   # a quiet NaN with a payload
VSHAPES = {1: (29,), 2: (13, 17), 3: (6, 7, 9)}
ANISOTROPY = {1: ((1.0,), (1.5,)), 2: ((1.0, 2.0), (0.7, 1.3)), 3: ((1.0, 1.0, 3.0), (1.5, 0.75, 2.25))}
DTYPES = (np.uint8, np.uint16, np.int32, np.uint64, np.bool_, np.float32)


def bits(a):
  a = np.asarray(a)
  return a.view(np.uint8) if a.dtype == np.bool_ else a.view(np.dtype("u%d" % a.itemsize))


def same_bits(a, b):
  a, b = np.asarray(a), np.asarray(b)
  return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(bits(a), bits(b))


def random_labels(rng, shape, dtype, density=0.05, low=1, high=7):
  """Sparse labels; float32 ones also carry negative labels, -0.0 background and NaN labels."""
  if dtype == np.bool_:
    return rng.random(shape) < density
  lab = np.where(rng.random(shape) < density, rng.integers(low, high, shape), 0).astype(dtype)
  if dtype == np.float32:
    labelled = lab != 0
    lab[labelled & (rng.random(shape) < 0.3)] *= -1
    lab[~labelled & (rng.random(shape) < 0.5)] = np.float32(-0.0)
    lab.view(np.uint32)[labelled & (rng.random(shape) < 0.2)] = NAN_BITS
  return lab


def volumes(lab, order):
  return [lab[b] for b in range(lab.shape[0])] if order == "C" else [lab[..., b] for b in range(lab.shape[-1])]


def stack(vols, order):
  return np.ascontiguousarray(np.stack(vols, 0)) if order == "C" else np.asfortranarray(np.stack(vols, -1))


def per_volume(edt, lab, order, distance, anisotropy):
  return stack([edt.expand_labels(v, distance, anisotropy) for v in volumes(lab, order)], order)


def check_stacked(edt, lab, order, distance, anisotropy):
  got = edt.expand_labels(lab, distance, anisotropy, stacked=True)
  assert got.dtype == lab.dtype and got.shape == lab.shape
  assert got.flags.c_contiguous if order == "C" else got.flags.f_contiguous
  want = per_volume(edt, lab, order, distance, anisotropy)
  assert same_bits(got, want), (lab.shape, lab.dtype, order, distance, anisotropy)
  return got


@pytest.mark.parametrize("dtype", DTYPES, ids=[np.dtype(d).name for d in DTYPES])
@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("vnd", [1, 2, 3])
def test_stacked_equals_per_volume(edt, vnd, order, dtype):
  rng = np.random.default_rng(100 * vnd + DTYPES.index(dtype) + (50 if order == "F" else 0))
  count = 5
  shape = (count,) + VSHAPES[vnd] if order == "C" else VSHAPES[vnd] + (count,)
  lab = stack(volumes(random_labels(rng, shape, dtype), order), order)
  for anisotropy in ANISOTROPY[vnd]:
    for distance in DISTANCES:
      got = check_stacked(edt, lab, order, distance, anisotropy)
      if distance != distance or distance == 0.0:
        assert same_bits(got, lab)                       # NaN and 0 grow nothing


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("vnd", [1, 2, 3])
def test_stacked_boundary_traps(edt, vnd, order):
  """A volume with no labels, an all-labelled volume, disjoint label sets, and background at the first
  voxel of a volume next to a label at the last voxel of the one before it in memory."""
  rng = np.random.default_rng(7 + vnd)
  vshape = {1: (9,), 2: (6, 7), 3: (4, 5, 6)}[vnd]
  dt = np.uint16
  first, last = (0,) * vnd, (-1,) * vnd          # first / last voxel of a volume in its memory order
  v0 = random_labels(rng, vshape, dt, 0.1, 1, 5)
  v1 = np.zeros(vshape, dt)                                          # no labels: nothing may grow
  v2 = rng.integers(21, 25, vshape).astype(dt)                       # all labelled: unchanged
  v3 = random_labels(rng, vshape, dt, 0.1, 31, 35)
  v3[last] = 35
  v4 = np.zeros(vshape, dt)
  v4[last] = 41                                                      # the only label, far from `first`
  sets = [set(range(1, 5)), set(), set(range(21, 25)), set(range(31, 36)), {41}]
  lab = stack([v0, v1, v2, v3, v4], order)
  for anisotropy in ANISOTROPY[vnd]:
    for distance in (1.0, 2.5, float("inf")):
      got = volumes(check_stacked(edt, lab, order, distance, anisotropy), order)
      assert not got[1].any()
      assert np.array_equal(got[2], v2)
      for g, allowed in zip(got, sets):
        assert set(np.unique(g).tolist()) <= allowed | {0}, "a label from another volume"
      assert got[4][first] == (41 if distance == float("inf") else 0)


def test_stacked_matches_skimage(edt):
  pytest.importorskip("scipy.ndimage")
  rng = np.random.default_rng(23)
  for vshape, spacing, dtype in (((30, 41), (1.0, 2.0), np.uint16), ((12, 13, 14), (1.0, 1.0, 3.0), np.int32)):
    lab = np.where(rng.random((4,) + vshape) < 0.03, rng.integers(1, 9, (4,) + vshape), 0).astype(dtype)
    for distance in (1.0, 2.5, 7.5):
      got = edt.expand_labels(lab, distance, spacing, stacked=True)
      for b in range(lab.shape[0]):
        want, sidx = fc.skimage_expand(lab[b], distance, spacing)
        sites = edt.feature_transform(lab[b], spacing, signed=True)
        fc.check_expand(lab[b], got[b], sites, want, sidx, distance, spacing)


@pytest.mark.parametrize("order", ["C", "F"])
def test_stacked_device_input(edt, order):
  """C- and F-strided CUDA tensors, on a side stream: equal to the host result, strides kept."""
  import torch
  rng = np.random.default_rng(31)
  for vnd, dtype in ((2, np.int32), (3, np.float32), (1, np.uint8)):
    shape = (6,) + VSHAPES[vnd] if order == "C" else VSHAPES[vnd] + (6,)
    lab = stack(volumes(random_labels(rng, shape, dtype, 0.08), order), order)
    anisotropy = ANISOTROPY[vnd][1]
    want = edt.expand_labels(lab, 2.5, anisotropy, stacked=True)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
      t = torch.from_numpy(lab).cuda()
      got = edt.expand_labels(t, 2.5, anisotropy, stacked=True)
    side.synchronize()
    assert got.is_cuda and got.dtype == t.dtype and got.stride() == t.stride()
    assert same_bits(got.cpu().numpy(), want)


def test_single_volume_device_equals_chunked_host(edt):
  """The single-volume device path (the gather kernel) against the chunked host path (a numpy gather)."""
  import torch
  rng = np.random.default_rng(37)
  for shape, spacing, dtype in (((40, 33), (1.0, 2.0), np.uint16), ((20, 21, 22), (1.5, 1.0, 0.75), np.float32),
                                ((17, 18, 19), (1.0, 1.0, 1.0), np.uint8), ((25, 26), (0.7, 1.0), np.float32),
                                ((11, 12, 13), (2.0, 1.0, 1.0), np.int32), ((30, 9), (1.0, 1.0), np.bool_)):
    for order in ("C", "F"):
      lab = random_labels(rng, shape, dtype, 0.04)
      lab = np.asfortranarray(lab) if order == "F" else np.ascontiguousarray(lab)
      t = torch.from_numpy(lab).cuda()
      for distance in DISTANCES:
        want = edt.expand_labels(lab, distance, spacing, max_device_bytes=0)
        got = edt.expand_labels(t, distance, spacing)
        assert got.stride() == t.stride()
        assert same_bits(got.cpu().numpy(), want), (shape, dtype, order, distance)
        assert same_bits(edt.expand_labels(lab, distance, spacing), want)


# ---- edtb200_expand_gather on its own ---------------------------------------------------------------

def restated_gather(raw, as_float, sq, planes, limit_sq, dims, count):
  """edtb200_expand_gather in numpy: raw label bits, x-fastest flat arrays, planes[k] int32 (ndim of them)."""
  sx, sy, sz = dims
  vol = sx * sy * sz
  bg = raw.view(np.dtype("f%d" % raw.itemsize)) == 0 if as_float else raw == 0
  q = [p.astype(np.int64) for p in planes] + [np.zeros(raw.size, np.int64)] * (3 - len(planes))
  inside = (q[0] < sx) & (q[1] >= 0) & (q[1] < sy) & (q[2] >= 0) & (q[2] < sz)
  with np.errstate(invalid="ignore"):
    near = np.abs(sq).astype(np.float64) <= limit_sq
  grow = bg & (q[0] >= 0) & near & inside
  site = np.arange(raw.size) // vol * vol + (q[2] * sy + q[1]) * sx + q[0]
  out = raw.copy()
  out[grow] = raw[site[grow]]
  return out


def gather_case(rng, label_bytes, as_float, ndim, dims, count, limit_sq):
  """Labels (raw bits), distances and planes made by hand: every site a labelled voxel of the voxel's own
  volume, or -1 (none), or outside the volume; distances of both signs, some exactly at the limit and
  some one float32 ulp above it."""
  sx, sy, sz = dims
  vol = sx * sy * sz
  total = vol * count
  u = np.dtype("u%d" % label_bytes)
  if as_float:
    f = np.dtype("f%d" % label_bytes)
    vals = np.where(rng.random(total) < 0.3, rng.integers(1, 6, total) * rng.choice([-1, 1], total), 0).astype(f)
    vals[(vals == 0) & (rng.random(total) < 0.5)] = -0.0
    raw = vals.view(u).copy()
    raw[(vals != 0) & (rng.random(total) < 0.2)] = (NAN_BITS if label_bytes == 4 else 0x7ff8000000000123)
  else:
    raw = np.where(rng.random(total) < 0.3, rng.integers(1, 200, total), 0).astype(u)
  if as_float:
    labelled = raw.view(np.dtype("f%d" % label_bytes)) != 0
  else:
    labelled = raw != 0
  planes = [np.zeros(total, np.int32) for _ in range(ndim)]
  for b in range(count):
    sites = np.flatnonzero(labelled[b * vol:(b + 1) * vol])
    assert sites.size
    pick = sites[rng.integers(0, sites.size, vol)]
    coords = (pick % sx, pick // sx % sy, pick // (sx * sy))
    for k in range(ndim):
      planes[k][b * vol:(b + 1) * vol] = coords[k]
  none = rng.random(total) < 0.15
  planes[0][none] = -1
  if ndim >= 2:
    planes[1][none] = rng.integers(-5, 5, int(none.sum()))         # never read where idx[0] is -1
    outside = ~none & (rng.random(total) < 0.05)
    planes[1][outside] = np.where(rng.random(int(outside.sum())) < 0.5, -1, sy)
  outside_x = ~none & (rng.random(total) < 0.03)
  planes[0][outside_x] = sx
  sq = (rng.random(total) * 2.5 * limit_sq).astype(np.float32) * rng.choice([-1, 1], total).astype(np.float32)
  at = np.float32(limit_sq)
  above = np.nextafter(at, np.float32(np.inf))
  pick = rng.random(total)
  sq[pick < 0.1] = at
  sq[(pick >= 0.1) & (pick < 0.2)] = -at
  sq[(pick >= 0.2) & (pick < 0.3)] = above
  sq[(pick >= 0.3) & (pick < 0.35)] = -above
  sq[(pick >= 0.35) & (pick < 0.38)] = np.inf
  return raw, sq, planes


@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_expand_gather_against_numpy(edt, ndim):
  import torch
  lib = edt._lib()
  rng = np.random.default_rng(41 + ndim)
  dims = {1: (37, 1, 1), 2: (9, 11, 1), 3: (7, 5, 6)}[ndim]
  count = 4
  for label_bytes, as_float in ((1, False), (2, False), (4, False), (8, False), (4, True), (8, True)):
    raw, sq, planes = gather_case(rng, label_bytes, as_float, ndim, dims, count, 6.25)
    assert (np.abs(sq) == np.float32(6.25)).any() and (np.abs(sq) == np.nextafter(np.float32(6.25), np.inf)).any()
    signed = np.dtype("i%d" % label_bytes)
    lab_t = torch.from_numpy(raw.view(signed)).cuda()
    sq_t = torch.from_numpy(sq).cuda()
    plane_t = [torch.from_numpy(p).cuda() for p in planes]
    idx = (ctypes.c_void_p * 3)(*([p.data_ptr() for p in plane_t] + [None] * (3 - ndim)))
    flags = BOTH | (LABELS_FLOAT if as_float else 0)
    for limit_sq in (6.25, 0.0, float("inf"), float("nan")):
      want = restated_gather(raw, as_float, sq, planes, limit_sq, dims, count)
      out_t = torch.full_like(lab_t, 7)
      rc = lib.edtb200_expand_gather(lab_t.data_ptr(), label_bytes, ndim, *dims, count, sq_t.data_ptr(), idx,
                                     limit_sq, flags, out_t.data_ptr(), lab_t.device.index, None)
      assert rc == 0, lib.edtb200_last_error()
      got = out_t.cpu().numpy().view(raw.dtype)
      assert np.array_equal(got, want), (label_bytes, as_float, limit_sq, int((got != want).sum()))
      inplace = lab_t.clone()
      rc = lib.edtb200_expand_gather(inplace.data_ptr(), label_bytes, ndim, *dims, count, sq_t.data_ptr(), idx,
                                     limit_sq, flags, inplace.data_ptr(), lab_t.device.index, None)
      assert rc == 0, lib.edtb200_last_error()
      assert np.array_equal(inplace.cpu().numpy().view(raw.dtype), want)
      if limit_sq == 6.25:
        grown = got != raw
        assert grown.any()
        assert not (grown & (np.abs(sq) == np.nextafter(np.float32(6.25), np.inf))).any()
      if limit_sq != limit_sq:
        assert np.array_equal(got, raw)
    if as_float:                                  # without the flag -0.0 is a label: it never grows
      rc = lib.edtb200_expand_gather(lab_t.data_ptr(), label_bytes, ndim, *dims, count, sq_t.data_ptr(), idx,
                                     6.25, BOTH, out_t.data_ptr(), lab_t.device.index, None)
      assert rc == 0, lib.edtb200_last_error()
      got = out_t.cpu().numpy().view(raw.dtype)
      assert np.array_equal(got, restated_gather(raw, False, sq, planes, 6.25, dims, count))
      neg_zero = raw == (np.uint64(1) << np.uint64(8 * label_bytes - 1)).astype(raw.dtype)
      assert neg_zero.any() and np.array_equal(got[neg_zero], raw[neg_zero])
