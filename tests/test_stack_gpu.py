"""GPU tests (-m gpu) of stacked=True and the C ABI's edtb200_transform_stack /
edtb200_feature_transform_stack: a stack of same-shaped volumes along the slowest axis in memory is
transformed with one launch per pass, and the result must equal np.stack of the per-volume calls bit
for bit (a subset is also checked against the oracle).

Beyond label widths, memory orders, volume dimensions, the four functions, borders and weights, the
boundary traps below each fail if a line or a run leaks from one volume into the next: a volume with
no site between volumes with sites, an all-ones stack under a black border, label noise whose next
volume starts with a copy of the previous volume's last slice (on the run-start plane plan), volumes
whose voxel count is not a multiple of 4 (the Z pass without TMA) and weights whose sums are not exact
(the Z pass on the long-line kernel over several volumes).
"""
import ctypes

import numpy as np
import pytest

import slab_cases

pytestmark = pytest.mark.gpu

ENOMEM = -3
SHAPES = {1: (37,), 2: (23, 36), 3: (9, 13, 20)}          # one volume, C order (x last)
WEIGHTS = {"int": (3.0, 2.0, 1.0), "frac": (2.9, 1.3, 0.7)}
DTYPES = (np.uint8, np.uint16, np.uint32, np.uint64, np.bool_, np.float32)
FUNCTIONS = ("edtsq", "edt", "sdfsq", "sdf")


def bits(a):
  a = np.ascontiguousarray(a)
  return a.view(np.uint32) if a.dtype == np.float32 else a.view(np.int32)


def same(got, want):
  return got.shape == want.shape and np.array_equal(bits(got), bits(want))


def blocks(rng, shape, dtype, cell=3, labels=4):
  """Runs of 1..cell equal labels along every axis, with background."""
  small = rng.integers(0, labels, shape)                    # every element repeated at least once
  out = small
  for ax in range(len(shape)):
    out = np.repeat(out, rng.integers(1, cell + 1, out.shape[ax]), axis=ax)
  out = out[tuple(slice(0, s) for s in shape)]
  if dtype == np.bool_:
    return out > 0
  if dtype == np.float32:
    return (out.astype(np.float32) - 1.0) * 0.5
  return out.astype(dtype)


def stack_of(volumes, order):
  """Volumes along axis 0 (C order) or along the last axis (F order)."""
  if order == "C":
    return np.ascontiguousarray(np.stack(volumes, axis=0))
  return np.asfortranarray(np.stack([np.asfortranarray(v) for v in volumes], axis=-1))


def volumes_of(stack, order):
  n = stack.shape[0] if order == "C" else stack.shape[-1]
  return [stack[b] if order == "C" else stack[..., b] for b in range(n)]


def per_volume(fn, stack, order, **kw):
  outs = [fn(v, **kw) for v in volumes_of(stack, order)]
  return np.stack(outs, axis=0 if order == "C" else -1)


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("vnd", [1, 2, 3])
@pytest.mark.parametrize("dtype", DTYPES, ids=[np.dtype(d).name for d in DTYPES])
def test_stack_equals_per_volume(edt, dtype, vnd, order):
  rng = np.random.default_rng(vnd * 10 + DTYPES.index(dtype))
  shape = SHAPES[vnd] if order == "C" else SHAPES[vnd][::-1]
  stack = stack_of([blocks(rng, shape, dtype) for _ in range(7)], order)
  for kind in WEIGHTS:
    w = WEIGHTS[kind][3 - vnd:]                             # one weight per volume axis, in array order
    for name in FUNCTIONS:
      for border in (False, True):
        fn = getattr(edt, name)
        got = fn(stack, anisotropy=w, black_border=border, stacked=True)
        want = per_volume(fn, stack, order, anisotropy=w, black_border=border)
        assert same(got, want), (name, kind, border)
        assert got.flags.c_contiguous if order == "C" else got.flags.f_contiguous


@pytest.mark.parametrize("vnd", [1, 2, 3])
def test_stack_equals_oracle(edt, oracle, vnd):
  rng = np.random.default_rng(40 + vnd)
  stack = stack_of([blocks(rng, SHAPES[vnd], np.uint32) for _ in range(5)], "C")
  w = WEIGHTS["frac"][3 - vnd:]
  for name in FUNCTIONS:
    for border in (False, True):
      got = getattr(edt, name)(stack, anisotropy=w, black_border=border, stacked=True)
      want = np.stack([getattr(oracle, name)(v, anisotropy=w, black_border=border) for v in stack])
      assert same(got, want), (name, border)


@pytest.mark.parametrize("count", [1, 2, 7, 300])
def test_counts(edt, count):
  rng = np.random.default_rng(count)
  for shape in ((3, 5, 8), (6, 12), (11,)):
    stack = stack_of([blocks(rng, shape, np.uint16, cell=2) for _ in range(count)], "C")
    for name in ("edtsq", "sdf"):
      fn = getattr(edt, name)
      assert same(fn(stack, black_border=True, stacked=True), per_volume(fn, stack, "C", black_border=True))


# ---- boundary traps ------------------------------------------------------------------------

@pytest.mark.parametrize("shape", [(8, 12, 16), (12, 16), (40,)])
def test_volume_without_a_site_stays_infinite(edt, shape):
  rng = np.random.default_rng(7)
  vols = [blocks(rng, shape, np.uint32), np.ones(shape, np.uint32), blocks(rng, shape, np.uint32)]
  stack = stack_of(vols, "C")
  for name in ("edtsq", "edt"):
    fn = getattr(edt, name)
    got = fn(stack, stacked=True)
    assert np.all(np.isposinf(got[1]))
    assert same(got, per_volume(fn, stack, "C"))


@pytest.mark.parametrize("shape", [(8, 12, 16), (9, 10, 11), (12, 16), (40,)])
def test_all_ones_with_black_border(edt, shape):
  stack = np.ones((6,) + shape, np.uint8)
  got = edt.edtsq(stack, black_border=True, stacked=True)
  alone = edt.edtsq(np.ones(shape, np.uint8), black_border=True)
  for b in range(6):
    assert got[b].max() == alone.max()
    assert same(got[b], alone)


def noise(rng, shape, dtype):
  lab = rng.integers(1, 1 << 20, shape).astype(dtype)
  lab[rng.random(shape) < 0.02] = 0
  return lab


@pytest.mark.parametrize("dtype", [np.uint32, np.uint64], ids=["uint32", "uint64"])
@pytest.mark.parametrize("shape", [(9, 40, 64), (5, 33, 128), (40, 64)])
def test_noise_whose_next_volume_repeats_the_last_slice(edt, oracle, dtype, shape):
  """On the plane plan (label noise, taken from the second call on) the first slice (2-D: first row)
  of every volume must start a run even where it equals the previous volume's last."""
  rng = np.random.default_rng(sum(shape))
  stack = noise(rng, (4,) + shape, dtype)
  for b in range(3):
    stack[b + 1, 0] = stack[b, -1]
  for name in ("edtsq", "edt"):
    for border in (False, True):
      fn = getattr(edt, name)
      fn(stack, black_border=border, stacked=True)          # leaves the run statistic of label noise behind
      got = fn(stack, black_border=border, stacked=True)
      info = edt.last_later_launch()
      assert info["kernel"] == "tile" and info["ctas"] == 2 and info["tma"] == 1, info
      want = np.stack([getattr(oracle, name)(v, black_border=border) for v in stack])
      assert same(got, want), (name, border)
  t = __import__("torch").from_numpy(stack.view(np.int32 if dtype == np.uint32 else np.int64)).cuda()
  edt.edt_cuda(t, stacked=True)
  got = edt.edt_cuda(t, stacked=True).cpu().numpy()
  assert edt.last_later_launch()["ctas"] == 2
  assert same(got, np.stack([oracle.edtsq(v) for v in stack]))


def test_volumes_not_a_multiple_of_four_voxels(edt):
  rng = np.random.default_rng(11)
  stack = stack_of([blocks(rng, (5, 7, 9), np.uint32) for _ in range(5)], "C")
  for name in FUNCTIONS:
    fn = getattr(edt, name)
    got = fn(stack, anisotropy=(1.0, 2.0, 1.0), stacked=True)
    assert edt.last_later_launch()["tma"] == 0
    assert same(got, per_volume(fn, stack, "C", anisotropy=(1.0, 2.0, 1.0)))


def test_readout_weights_take_the_long_line_kernel(edt, oracle):
  """slab_cases.readout_volume under its weights: every volume of the stack equals its own transform,
  and the first volume differs from the reference at READOUT_VOXELS only, where the GPU returns the
  least candidate (test_slab_gpu.py's test_reference_readout_keeps_earlier_vertex)."""
  vol = slab_cases.readout_volume()
  vols = [vol, vol[::-1].copy(), np.roll(vol, 5, axis=0), vol]
  stack = np.ascontiguousarray(np.stack(vols).astype(np.int32))
  w = slab_cases.TIE_W
  for name in ("sdfsq", "edtsq", "sdf"):
    for border in (False, True):
      fn = getattr(edt, name)
      got = fn(stack, anisotropy=w, black_border=border, stacked=True)
      assert edt.last_later_launch()["kernel"] == "long"
      assert same(got, per_volume(fn, stack, "C", anisotropy=w, black_border=border)), (name, border)
  got = edt.sdfsq(stack, anisotropy=w, stacked=True)
  bad = {tuple(int(i) for i in p) for p in np.argwhere(got[0] != oracle.sdfsq(vol, anisotropy=w))}
  assert bad == set(slab_cases.READOUT_VOXELS), bad


# ---- device tensors ----------------------------------------------------------------------

def test_device_stack_on_a_side_stream(edt):
  import torch
  rng = np.random.default_rng(21)
  stack = stack_of([blocks(rng, (10, 12, 16), np.uint32) for _ in range(6)], "C")
  t = torch.from_numpy(stack.view(np.int32)).cuda()
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    got = edt.edt(t, anisotropy=(2.0, 1.0, 1.5), black_border=True, stacked=True)
    got_sq = edt.edt_cuda(t, (2.0, 1.0, 1.5), True, stacked=True)
  side.synchronize()
  assert isinstance(got, torch.Tensor) and got.shape == t.shape
  assert same(got.cpu().numpy(), per_volume(edt.edt, stack, "C", anisotropy=(2.0, 1.0, 1.5), black_border=True))
  assert same(got_sq.cpu().numpy(), per_volume(edt.edtsq, stack, "C", anisotropy=(2.0, 1.0, 1.5), black_border=True))


def test_device_fortran_view_and_out(edt):
  import torch
  rng = np.random.default_rng(22)
  host_f = stack_of([blocks(rng, (16, 12, 10), np.uint16) for _ in range(5)], "F")      # volumes along the last axis
  t = torch.from_numpy(np.ascontiguousarray(host_f.T).view(np.int16)).cuda().permute(3, 2, 1, 0)
  assert not t.is_contiguous() and tuple(t.shape) == host_f.shape
  w = (1.0, 2.5, 3.0)
  got = edt.sdf(t, anisotropy=w, stacked=True)
  assert got.shape == t.shape and got.stride() == t.stride()
  assert same(got.cpu().numpy(), edt.sdf(host_f, anisotropy=w, stacked=True))
  assert same(got.cpu().numpy(), per_volume(edt.sdf, host_f, "F", anisotropy=w))
  c = torch.from_numpy(np.ascontiguousarray(host_f.T).view(np.int16)).cuda()           # (B, ...) C order
  buf = torch.full(c.shape, 7.0, dtype=torch.float32, device=c.device)
  ret = edt.edt_cuda(c, tuple(reversed(w)), sqrt=True, signed=True, out=buf, stacked=True)
  assert ret.data_ptr() == buf.data_ptr()
  assert same(buf.cpu().numpy(), np.ascontiguousarray(got.cpu().numpy().T))


# ---- host groups -------------------------------------------------------------------------

def _stack_call(edt, stack, device_bytes):
  lib = edt._lib()
  out = np.empty(stack.shape, np.float32)
  groups = (ctypes.c_int64 * 1)(-1)
  sz, sy, sx = stack.shape[1:]
  rc = lib.edtb200_transform_stack(stack.ctypes.data, stack.dtype.itemsize, 3, sx, sy, sz, stack.shape[0],
                                   1.0, 1.5, 2.0, 1, 1, out.ctypes.data, 0, device_bytes, groups, None)
  return rc, out, groups[0], lib.edtb200_last_error()


def test_host_groups(edt):
  rng = np.random.default_rng(31)
  stack = stack_of([blocks(rng, (24, 20, 16), np.uint16) for _ in range(50)], "C")
  per_vol = 24 * 20 * 16 * (2 + 4)
  rc, one, groups, err = _stack_call(edt, stack, 0)
  assert rc == 0 and groups == 1, err
  rc, several, groups, err = _stack_call(edt, stack, 20 * per_vol)
  assert rc == 0 and groups == 5, (err, groups)
  assert same(several, one)
  rc, odd, groups, err = _stack_call(edt, stack, 2 * per_vol + 7)
  assert rc == 0 and groups == 50, (err, groups)
  assert same(odd, one)
  want = per_volume(edt.edt, stack, "C", anisotropy=(2.0, 1.5, 1.0), black_border=True)
  assert same(one, want)
  got = edt.edt(stack, anisotropy=(2.0, 1.5, 1.0), black_border=True, max_device_bytes=6 * per_vol, stacked=True)
  assert same(got, want)
  # a budget below two volumes (a pipeline needs two slots) cannot hold a group
  rc, _, groups, err = _stack_call(edt, stack, 2 * per_vol - 1)
  assert rc == ENOMEM and groups == 0
  assert b"at least %d bytes" % (2 * per_vol) in err, err
  with pytest.raises(edt.EDTError) as info:
    edt.edtsq(stack, max_device_bytes=per_vol, stacked=True)
  assert info.value.code == ENOMEM


def test_host_groups_pinned_and_pageable(edt):
  import torch
  rng = np.random.default_rng(32)
  stack = stack_of([blocks(rng, (64, 256), np.uint32) for _ in range(300)], "C")          # 2-D slices, 78 MB out
  pinned = torch.empty(stack.shape, dtype=torch.int32, pin_memory=True).numpy()
  pinned[...] = stack.view(np.int32)
  want = per_volume(edt.edtsq, stack, "C")
  for src in (stack, pinned.view(np.uint32)):
    for budget in (None, 40 * 64 * 256 * 8 * 2):
      assert same(edt.edtsq(src, stacked=True, max_device_bytes=budget), want)


# ---- feature transform ---------------------------------------------------------------------

@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("vnd", [1, 2, 3])
def test_feature_stack_equals_per_volume(edt, vnd, order):
  import torch
  rng = np.random.default_rng(50 + vnd)
  shape = SHAPES[vnd] if order == "C" else SHAPES[vnd][::-1]
  vols = [blocks(rng, shape, np.uint32) for _ in range(5)]
  vols[2] = np.ones(shape, np.uint32)                       # no site without a border
  stack = stack_of(vols, order)
  w = WEIGHTS["frac"][3 - vnd:]
  for signed in (False, True):
    for border in (False, True):
      kw = dict(anisotropy=w, black_border=border, signed=signed, return_distances=True)
      dist, idx = edt.feature_transform(stack, stacked=True, **kw)
      parts = [edt.feature_transform(v, **kw) for v in volumes_of(stack, order)]
      want_d = np.stack([p[0] for p in parts], axis=0 if order == "C" else -1)
      want_i = np.stack([p[1] for p in parts], axis=1 if order == "C" else -1)
      assert idx.shape == (vnd,) + stack.shape
      assert same(dist, want_d) and np.array_equal(idx, want_i), (signed, border)
      if not border:
        assert np.all(np.isposinf(np.abs(dist[2] if order == "C" else dist[..., 2])))
      t = torch.from_numpy(stack.view(np.int32)).cuda()
      if order == "F":
        t = torch.from_numpy(np.ascontiguousarray(stack.T).view(np.int32)).cuda().permute(*reversed(range(stack.ndim)))
      d_dev, i_dev = edt.feature_transform(t, stacked=True, **kw)
      assert same(d_dev.cpu().numpy(), want_d) and np.array_equal(i_dev.cpu().numpy(), want_i), (signed, border)
