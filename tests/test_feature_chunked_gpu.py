"""GPU tests: edtb200_feature_transform_chunked equals edtb200_feature_transform bit for bit.

Every case runs the one-shot host feature transform and the chunked one on the same labels and
compares the distances (as bits) and every index plane.  Budgets are forced small so that the phases
run in many chunks: one slice per chunk, uneven chunks, and the budget 0 (what the device has free);
the reported chunk counts must equal the plan documented in include/edt_b200.h, restated by `plan`.
"""
import ctypes
import os
import threading
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
EDGES = os.path.join(HERE, "golden", "rounding_edges.npz")
SQRT, SIGNED = 1, 2
ENOMEM = -3
ANISO = {"int": (1.0, 2.0, 3.0), "real": (0.7, 1.3, 2.9), "dyadic": (0.5, 0.25, 2.0)}
WIDTHS = (np.uint8, np.uint16, np.uint32, np.uint64)


# ---- the documented plan ------------------------------------------------------------------------

def per_voxel(ndim, L):
  """Device bytes per voxel of (phase 1, phase 2): slot buffers plus the hull of a later pass."""
  return (L + 20, L + 28) if ndim == 3 else (L + 8, L + 20)


def phase_chunks(extent, slice_bytes, budget):
  if extent * slice_bytes <= budget:
    return 1
  c = budget // (2 * slice_bytes)
  assert c > 0
  return -(-extent // c)


def slices(ndim, dims, L):
  sx, sy, sz = dims
  b1, b2 = per_voxel(ndim, L)
  return (sx * sy * b1, sx * sz * b2) if ndim == 3 else (sx * b1, sy * b2)


def extents(ndim, dims):
  sx, sy, sz = dims
  return (sz, sy) if ndim == 3 else (sy, sx)


def plan(ndim, dims, L, budget):
  (e1, e2), (s1, s2) = extents(ndim, dims), slices(ndim, dims, L)
  return [phase_chunks(e1, s1, budget), phase_chunks(e2, s2, budget)]


def least_budget(ndim, dims, L):
  (e1, e2), (s1, s2) = extents(ndim, dims), slices(ndim, dims, L)
  return max(min(e1, 2) * s1, min(e2, 2) * s2)


# ---- calls ------------------------------------------------------------------------------------------

class Volume:
  """A host array as the C ABI sees it: raw label bits, x-fastest dims and weights."""

  def __init__(self, edt, data, anisotropy):
    self.order = "F" if data.flags.f_contiguous and not data.flags.c_contiguous else "C"
    data = np.asfortranarray(data) if self.order == "F" else np.ascontiguousarray(data)
    self.labels = edt._label_view(data)
    self.ndim = data.ndim
    an = (anisotropy,) * data.ndim if np.ndim(anisotropy) == 0 else tuple(anisotropy)
    self.dims, self.w = edt._x_fastest(data.shape, an, self.order == "F")
    self.L = self.labels.dtype.itemsize
    self.size = data.size


def host_buffer(edt, nbytes, pinned):
  """(numpy uint8 array, keep-alive): page-locked memory from the library, or plain numpy memory."""
  if not pinned:
    return np.zeros(nbytes, np.uint8), None
  ptr = edt._lib().edtb200_host_alloc(ctypes.c_size_t(nbytes))
  assert ptr
  return np.frombuffer((ctypes.c_char * nbytes).from_address(ptr), dtype=np.uint8, count=nbytes), ptr


def call(edt, v, flags, border, with_dist, budget=None, pinned_labels=False, pinned_out=False):
  """-> (distances or None, index planes (ndim, size), chunks, rc); budget None: the one-shot call."""
  lib = edt._lib()
  keep = []
  try:
    lab, p = host_buffer(edt, v.labels.nbytes, pinned_labels)
    keep.append(p)
    lab[:] = np.ravel(v.labels, order="K").view(np.uint8)
    out, p = host_buffer(edt, (v.ndim + 1) * v.size * 4, pinned_out)
    keep.append(p)
    planes = out.view(np.int32).reshape(v.ndim + 1, v.size)
    planes[:] = -7
    dist = planes[v.ndim].view(np.float32) if with_dist else None
    ptrs = (ctypes.c_void_p * v.ndim)(*[planes[k].ctypes.data for k in range(v.ndim)])
    args = (lab.ctypes.data, v.L, v.ndim, *v.dims, *v.w, int(border), flags,
            dist.ctypes.data if with_dist else None, ptrs, 0)
    chunks = (ctypes.c_int64 * 2)()
    if budget is None:
      rc = lib.edtb200_feature_transform(*args, None)
    else:
      rc = lib.edtb200_feature_transform_chunked(*args, ctypes.c_size_t(budget), chunks)
    return (dist.copy() if with_dist else None), planes[:v.ndim].copy(), list(chunks), rc
  finally:
    for p in keep:
      if p:
        lib.edtb200_host_free(ctypes.c_void_p(p))


def oneshot(edt, v, flags, border):
  dist, idx, _, rc = call(edt, v, flags, border, True)
  assert rc == 0, edt._lib().edtb200_last_error()
  return dist, idx


def assert_same(got, want, what=""):
  gd, gi = got
  wd, wi = want
  if gd is not None:
    bad = gd.view(np.uint32) != wd.view(np.uint32)
    assert not bad.any(), "%s: %d distances differ, first at %d: %r vs %r" % (
      what, int(bad.sum()), int(np.argmax(bad)), gd[np.argmax(bad)], wd[np.argmax(bad)])
  for k in range(len(wi)):
    bad = gi[k] != wi[k]
    assert not bad.any(), "%s: plane %d: %d voxels differ, first at %d: %d vs %d" % (
      what, k, int(bad.sum()), int(np.argmax(bad)), gi[k][np.argmax(bad)], wi[k][np.argmax(bad)])


def check(edt, v, flags, border, budget, with_dist=True, want=None, exact_plan=True, **pinned):
  want = want or oneshot(edt, v, flags, border)
  dist, idx, chunks, rc = call(edt, v, flags, border, with_dist, budget, **pinned)
  assert rc == 0, edt._lib().edtb200_last_error()
  assert_same((dist, idx), want, (v.dims, flags, border, budget, with_dist))
  if exact_plan:
    assert chunks == plan(v.ndim, v.dims, v.L, budget or (1 << 50)), (v.dims, budget, chunks)
  return chunks


def labels_of(rng, shape, dtype, kind):
  """Labels 0..2 in blocks, or iid ("noise"), as `dtype`."""
  if kind == "noise":
    lab = rng.integers(0, 3, shape)
  else:
    lab = rng.integers(0, 3, tuple(max(1, s // 3) for s in shape))
    for ax, s in enumerate(shape):
      lab = np.repeat(lab, -(-s // lab.shape[ax]), axis=ax)
    lab = lab[tuple(slice(0, s) for s in shape)]
  return (lab.astype(np.uint64) * np.uint64(0x1000001)).astype(dtype)


# ---- random cases: every label width, both orders, odd sizes, singleton axes, every weight class --

SHAPES = [(17, 13, 21), (23, 37), (1, 9, 5), (7, 1, 1), (5, 1), (1, 1, 13), (30, 1, 11), (2, 3)]


def cases():
  out = []
  for i, shape in enumerate(SHAPES):
    for j, dtype in enumerate(WIDTHS):
      out.append(("%s-%s" % ("x".join(map(str, shape)), np.dtype(dtype).name), shape, dtype,
                  ("blocks", "noise")[(i + j) % 2], ("int", "real", "dyadic")[(i + j) % 3], ("C", "F")[j % 2]))
  return out


@pytest.mark.parametrize("case", cases(), ids=lambda c: c[0])
def test_random_cases_bit_equal(edt, case):
  name, shape, dtype, kind, acls, order = case
  rng = np.random.default_rng(zlib.crc32(name.encode()))
  lab = labels_of(rng, shape, dtype, kind)
  lab = np.asfortranarray(lab) if order == "F" else np.ascontiguousarray(lab)
  v = Volume(edt, lab, ANISO[acls][:len(shape)])
  tight = least_budget(v.ndim, v.dims, v.L)
  n = 0
  for border in (False, True):
    for flags in (0, SQRT, SIGNED, SQRT | SIGNED):
      want = oneshot(edt, v, flags, border)
      for budget in (tight, 3 * tight - 1, 0):
        n += 1
        check(edt, v, flags, border, budget, with_dist=n % 2 == 0, want=want)


def test_python_orders_and_dtypes(edt):
  """feature_transform(max_device_bytes=...) equals the one-shot call in both memory orders."""
  rng = np.random.default_rng(3)
  for dtype in (np.uint8, np.int16, np.int32, np.uint64, np.float32, np.bool_):
    for order in ("C", "F"):
      lab = labels_of(rng, (19, 14, 11), np.uint8, "blocks")
      lab = lab.astype(dtype) if dtype != np.bool_ else lab > 0
      lab = np.asfortranarray(lab) if order == "F" else np.ascontiguousarray(lab)
      for signed in (False, True):
        wd, wi = edt.feature_transform(lab, (1.0, 2.0, 0.5), True, signed=signed, return_distances=True)
        for budget in (20000, 0):
          gd, gi = edt.feature_transform(lab, (1.0, 2.0, 0.5), True, signed=signed, return_distances=True,
                                         max_device_bytes=budget)
          assert gi.shape == wi.shape and np.array_equal(gi, wi), (dtype, order, signed, budget)
          assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32))
          assert gd.flags.f_contiguous == wd.flags.f_contiguous
          only = edt.feature_transform(lab, (1.0, 2.0, 0.5), True, signed=signed, max_device_bytes=budget)
          assert np.array_equal(only, wi)


def test_double_rounding_tie(edt):
  z = np.load(EDGES)
  lab = z["tie2d_labels"]
  an = tuple(float(a) for a in z["tie2d_aniso"])
  bb = bool(z["tie2d_border"])
  v = Volume(edt, lab, an)
  for border in (bb, not bb):
    for flags in (0, SQRT | SIGNED, SIGNED):
      for budget in (least_budget(2, v.dims, v.L), 0):
        check(edt, v, flags, border, budget)
        check(edt, v, flags, border, budget, with_dist=False)


# ---- no site, face sites ---------------------------------------------------------------------------

def test_no_site_crosses_the_phases(edt):
  """Slices of one label have no site within the slice (kSiteNone from phase 1); their voxels reach
  a site through the Z pass, or have none at all."""
  lab = np.ones((20, 24, 28), np.uint16)                  # C order: z = 20 slices
  lab[15, 3, 5] = 2
  lab[15, 20:, :] = 0
  lab[18, :, 27] = 3
  for order in ("C", "F"):
    arr = np.asfortranarray(lab) if order == "F" else lab
    v = Volume(edt, arr, (1.0, 1.0, 1.0))
    for flags in (0, SIGNED | SQRT):
      want = oneshot(edt, v, flags, False)
      for budget in (least_budget(3, v.dims, v.L), 0):
        check(edt, v, flags, False, budget, want=want)
        check(edt, v, flags, False, budget, with_dist=False, want=want)
  for shape in ((9, 10, 11), (13, 7)):                   # no site anywhere
    v = Volume(edt, np.full(shape, 5, np.uint8), (1.0,) * len(shape))
    want = oneshot(edt, v, SQRT, False)
    assert (want[1] == -1).all() and np.isinf(want[0]).all()
    check(edt, v, SQRT, False, least_budget(v.ndim, v.dims, v.L), want=want)


def test_face_sites(edt):
  """With black_border a uniform volume's sites are all faces: -1 and n, never "no site"."""
  for shape in ((9, 10, 11), (13, 7), (1, 6, 5)):
    v = Volume(edt, np.full(shape, 5, np.uint32), (1.0, 3.0, 2.0)[:len(shape)])
    for flags in (0, SQRT | SIGNED):
      want = oneshot(edt, v, flags, True)
      outside = (want[1] < 0) | (want[1] >= np.array(v.dims[:v.ndim]).reshape(-1, 1))
      assert (outside.sum(0) == 1).all()                # one face coordinate per site
      for budget in (least_budget(v.ndim, v.dims, v.L), 0):
        check(edt, v, flags, True, budget, want=want)


# ---- budgets: one slice per chunk, uneven chunks; the origin of later chunks ----------------------

def test_budget_formula_one_slice_and_uneven(edt):
  rng = np.random.default_rng(3)
  for shape in [(13, 17, 19), (40, 31, 9), (20, 20, 15), (23, 29), (50, 3)]:
    lab = rng.integers(0, 5, shape).astype(np.uint8)
    lab[lab == 4] = 0                                   # unsigned background in every chunk
    v = Volume(edt, lab, (1.0,) * len(shape))
    s1, s2 = slices(v.ndim, v.dims, v.L)
    least = least_budget(v.ndim, v.dims, v.L)
    for flags, border in ((SQRT, True), (0, False)):
      want = oneshot(edt, v, flags, border)
      for budget in (least, 2 * s1, 2 * s2, 2 * max(s1, s2), 3 * 2 * max(s1, s2) + 1, 7 * 2 * max(s1, s2) - 1,
                     10 ** 12, 0):
        if budget and budget < least:
          continue
        check(edt, v, flags, border, budget, want=want)
    # two slices of the dearer phase: one slice per chunk there
    k = 1 if s2 >= s1 else 0
    chunks = check(edt, v, SQRT, True, 2 * max(s1, s2))
    assert chunks[k] == extents(v.ndim, v.dims)[k] > 2


def test_long_z_lines(edt):
  """z lines of 5000 voxels (more than 4096) in every chunk."""
  rng = np.random.default_rng(8)
  labels = np.asfortranarray(rng.integers(0, 2, (8, 6, 5000)).astype(np.uint32))
  labels[:, :, 1000:4500] = 1
  v = Volume(edt, labels, (1.0, 2.0, 1.0))
  assert v.dims == [8, 6, 5000]
  for flags in (0, SQRT | SIGNED):
    for border in (False, True):
      want = oneshot(edt, v, flags, border)
      tight = least_budget(3, v.dims, v.L)
      for budget in (tight, 3 * tight + 5, 0):
        check(edt, v, flags, border, budget, want=want)


# ---- host buffers ---------------------------------------------------------------------------------

@pytest.mark.parametrize("pinned_labels,pinned_out", [(False, False), (True, False), (False, True), (True, True)])
def test_pinned_and_pageable(edt, pinned_labels, pinned_out):
  rng = np.random.default_rng(12)
  small = rng.integers(0, 9, (12, 30, 40)).astype(np.uint32)
  labels = np.repeat(np.repeat(np.repeat(small, 8, 0), 8, 1), 8, 2)[:90, :231, :317]    # 6.6 M voxels
  v = Volume(edt, labels, (1.0, 1.0, 2.0))
  want = oneshot(edt, v, SQRT | SIGNED, True)
  s1 = slices(3, v.dims, v.L)[0]
  for budget in (least_budget(3, v.dims, v.L), 13 * s1, 60 * s1, 0):
    check(edt, v, SQRT | SIGNED, True, budget, want=want, pinned_labels=pinned_labels, pinned_out=pinned_out)


@pytest.mark.parametrize("pinned", [False, True])
def test_pitched_rows_longer_than_a_staging_buffer(edt, pinned):
  """(4, 1500, 17000) uint8 in three phase-2 chunks of 500 y rows: each pitched row of a distance or
  index plane is 34 MB, more than one 32 MiB staging buffer."""
  rng = np.random.default_rng(13)
  labels = np.repeat(rng.integers(0, 3, (4, 1500, 17000 // 8)).astype(np.uint8), 8, axis=2)
  v = Volume(edt, labels, (1.0, 1.0, 1.0))
  assert v.dims == [17000, 1500, 4]
  budget = 2 * 500 * slices(3, v.dims, v.L)[1]
  assert 500 * 17000 * 4 > 32 << 20
  chunks = check(edt, v, 0, False, budget, pinned_labels=pinned, pinned_out=pinned)
  assert chunks[1] == 3


# ---- errors ---------------------------------------------------------------------------------------

def test_budget_below_one_chunk_is_enomem(edt):
  rng = np.random.default_rng(14)
  for shape in [(10, 20, 30), (30, 20, 10), (17, 40)]:
    v = Volume(edt, rng.integers(0, 3, shape).astype(np.uint16), (1.0,) * len(shape))
    need = least_budget(v.ndim, v.dims, v.L)
    _, _, chunks, rc = call(edt, v, 0, False, True, need - 1)
    assert rc == ENOMEM and chunks == [0, 0]
    msg = edt._lib().edtb200_last_error().decode()
    assert "needs at least %d bytes" % need in msg, msg
    check(edt, v, 0, False, need)


# ---- concurrency ----------------------------------------------------------------------------------

def test_two_threads_chunked_and_oneshot(edt):
  rng = np.random.default_rng(15)
  vols = [Volume(edt, rng.integers(0, 4, (60, 70, 80)).astype(np.uint32), (1.0, 2.0, 3.0)),
          Volume(edt, np.asfortranarray(rng.integers(0, 2, (50, 90, 40)).astype(np.uint8)), (2.0, 1.0, 1.0))]
  want = [oneshot(edt, v, SQRT | SIGNED, True) for v in vols]
  results = {}

  def work(name, fn):
    try:
      results[name] = [fn() for _ in range(4)]
    except Exception as e:                  # reported below
      results[name] = e

  budget = 3 * least_budget(3, vols[0].dims, vols[0].L) + 1
  jobs = [("chunked0", lambda: call(edt, vols[0], SQRT | SIGNED, True, True, budget)),
          ("oneshot1", lambda: call(edt, vols[1], SQRT | SIGNED, True, True))]
  threads = [threading.Thread(target=work, args=job) for job in jobs]
  for t in threads:
    t.start()
  for t in threads:
    t.join()
  for name, idx in (("chunked0", 0), ("oneshot1", 1)):
    runs = results[name]
    assert not isinstance(runs, Exception), runs
    for dist, planes, _, rc in runs:
      assert rc == 0
      assert_same((dist, planes), want[idx], name)


# ---- Python ---------------------------------------------------------------------------------------

def test_python_max_device_bytes(edt):
  rng = np.random.default_rng(17)
  x = np.asfortranarray(rng.integers(0, 5, (40, 33, 21)).astype(np.uint16))
  budget = 3 * least_budget(3, [40, 33, 21], 2)
  for signed in (False, True):
    wd, wi = edt.feature_transform(x, (1.0, 2.0, 3.0), True, signed=signed, return_distances=True)
    gd, gi = edt.feature_transform(x, (1.0, 2.0, 3.0), True, signed=signed, return_distances=True,
                                   max_device_bytes=budget)
    assert np.array_equal(gi, wi) and np.array_equal(gd.view(np.uint32), wd.view(np.uint32))
  y = np.ascontiguousarray(x[:, :, 0])
  assert np.array_equal(edt.feature_transform(y, max_device_bytes=0), edt.feature_transform(y))
  with pytest.raises(edt.EDTError) as info:
    edt.feature_transform(x, max_device_bytes=1000)
  assert info.value.code == ENOMEM
  import torch
  with pytest.raises(ValueError, match="device-resident"):
    edt.feature_transform(torch.ones((4, 4, 4), dtype=torch.uint8, device="cuda"), max_device_bytes=1 << 20)
  with pytest.raises(ValueError, match="device-resident"):
    edt.expand_labels(torch.ones((4, 4, 4), dtype=torch.uint8, device="cuda"), max_device_bytes=1 << 20)


@pytest.mark.parametrize("order", ["C", "F"])
def test_expand_labels_max_device_bytes(edt, order):
  rng = np.random.default_rng(13)
  for shape, spacing, dtype in (((50, 40), (1.0, 2.0), np.uint16), ((30, 31, 32), (1.0, 1.0, 3.0), np.int32),
                                ((20, 21, 22), (1.0, 1.0, 1.0), np.float32), ((9, 8, 7), (2.0, 1.0, 1.0), np.uint8)):
    lab = np.where(rng.random(shape) < 0.02, rng.integers(1, 9, shape), 0).astype(dtype)
    lab[(0,) * len(shape)] = 3
    lab = np.asfortranarray(lab) if order == "F" else np.ascontiguousarray(lab)
    for distance in (0.0, 1.0, 2.5, 7.5):
      want = edt.expand_labels(lab, distance, spacing)
      for budget in (3 * least_budget(len(shape), Volume(edt, lab, spacing).dims, lab.dtype.itemsize), 0):
        got = edt.expand_labels(lab, distance, spacing, max_device_bytes=budget)
        assert got.dtype == lab.dtype and got.shape == lab.shape
        assert got.flags.f_contiguous == lab.flags.f_contiguous
        assert np.array_equal(got, want), (shape, dtype, distance, budget)


def test_python_falls_back_on_enomem(edt, monkeypatch):
  rng = np.random.default_rng(16)
  x = rng.integers(0, 5, (33, 45, 27)).astype(np.int32)
  x[x == 4] = 0
  x2 = np.asfortranarray(x[0])
  want3 = edt.feature_transform(x, (1.0, 2.0, 3.0), signed=True, return_distances=True)
  want2 = edt.feature_transform(x2, black_border=True, return_distances=True)
  want_e = edt.expand_labels(x, 2.5, (1.0, 2.0, 3.0))
  calls = []
  lib = edt._lib()

  def out_of_memory(*args):
    calls.append(args)
    return ENOMEM

  monkeypatch.setattr(lib, "edtb200_feature_transform", out_of_memory)
  got3 = edt.feature_transform(x, (1.0, 2.0, 3.0), signed=True, return_distances=True)
  got2 = edt.feature_transform(x2, black_border=True, return_distances=True)
  got_e = edt.expand_labels(x, 2.5, (1.0, 2.0, 3.0))
  assert len(calls) == 3
  for (gd, gi), (wd, wi) in ((got3, want3), (got2, want2)):
    assert np.array_equal(gi, wi) and np.array_equal(gd.view(np.uint32), wd.view(np.uint32))
  assert np.array_equal(got_e, want_e)
  with pytest.raises(edt.EDTError) as info:                  # 1-D has no chunked path
    edt.feature_transform(x[0, 0])
  assert info.value.code == ENOMEM


# ---- the run statistic ----------------------------------------------------------------------------

def tile_ctas(edt):
  """CTAs per SM of the next tile pass (2: label noise predicted, 3: not), read off a pass_later."""
  import torch
  lt = torch.ones((200, 4, 8), dtype=torch.int32, device="cuda")
  ft = torch.arange(200 * 4 * 8, dtype=torch.float32, device="cuda").reshape(200, 4, 8) % 7
  lib = edt._lib()
  rc = lib.edtb200_pass_later(lt.data_ptr(), 4, 2, 8, 4, 200, 1.0, 1, 0, 0, ft.data_ptr(), 0, ctypes.c_void_p(None))
  assert rc == 0, lib.edtb200_last_error()
  torch.cuda.synchronize()
  v = edt.last_later_launch()
  assert v["kernel"] == "tile" and v["tma"] == 1, v
  return v["ctas"]


def test_chunked_feature_leaves_the_run_statistic(edt):
  """A chunked feature transform publishes no run statistic: the next tile pass still follows the
  last edtsq, whatever the feature transform's volume looked like."""
  rng = np.random.default_rng(0)
  noise = rng.integers(0, 256, (64, 64, 16), dtype=np.uint32)
  quiet = np.ones((64, 64, 16), np.uint32)
  for before, during, ctas in ((noise, quiet, 2), (quiet, noise, 3)):
    edt.edtsq(before)
    assert tile_ctas(edt) == ctas
    edt.edtsq(before)
    edt.feature_transform(during, max_device_bytes=least_budget(3, [16, 64, 64], 4))
    assert tile_ctas(edt) == ctas
