"""GPU tests of spherical_erode, spherical_open, spherical_dilate and spherical_close: bit for bit against
the threshold restatement on the CPU oracle (morphology_cases.threshold) for every label width, float
labels with -0.0 and NaN payloads, bool, C and F order, 1-D to 3-D, both black_border values, integer
and non-integer anisotropy, and radii from 0 to far beyond the window limit -- with the path the last
pass took asserted through last_later_launch; stacks against the per-volume calls; host input and
device input on a non-default stream; and the lattice properties of opening and closing."""
import ctypes

import numpy as np
import pytest

import morphology_cases as mc

pytestmark = pytest.mark.gpu

FNS = {"erode": "spherical_erode", "open": "spherical_open", "dilate": "spherical_dilate", "close": "spherical_close"}


def run(edt, op, arr, r, w=None, bb=False, **kw):
  fn = getattr(edt, FNS[op])
  if op == "dilate":
    return fn(arr, r, w, **kw)
  return fn(arr, r, w, bb, **kw)


def want(op, arr, r, w=None, bb=False):
  return mc.threshold(op, arr, r, w, bb and op != "dilate")


def same(got, exp):
  return got.dtype == exp.dtype and got.shape == exp.shape and np.array_equal(mc._raw(got), mc._raw(exp))


def last_pass_windowed(edt, arr, r, w):
  """Whether the transform's last pass takes the window kernel (edtb200_bounded_plan, bit 0)."""
  nd = arr.ndim
  w = (1.0,) * nd if w is None else tuple(w)
  dims, weights = list(arr.shape), list(w)
  if not (arr.flags.f_contiguous and not arr.flags.c_contiguous):
    dims, weights = dims[::-1], weights[::-1]
  dims += [1] * (3 - nd)
  weights += [1.0] * (3 - nd)
  radius, windowed = (ctypes.c_int64 * 3)(), (ctypes.c_int * 3)()
  assert edt._lib().edtb200_bounded_plan(nd, *dims, *weights, r, radius, windowed) == 0
  return bool(windowed[nd - 1] & 1)


def check_path(edt, arr, r, w):
  if arr.ndim >= 2:
    kernel = edt.last_later_launch()["kernel"]
    assert (kernel == "window") == last_pass_windowed(edt, arr, r, w), (kernel, r, w)


def float_labels(rng, shape, dtype):
  """Blocks of float labels, background as -0.0 in places, and one region of a NaN with a payload."""
  base = mc.touching(rng, shape, np.int32).astype(dtype)
  bits = np.uint32(0x7FC01234) if dtype == np.float32 else np.uint64(0x7FF8000000ABCDEF)
  nan = np.array([bits]).view(dtype)[0]
  base[base == 2] = nan
  base[base == 3] = -1.5
  zero = base == 0
  base[zero & (rng.random(shape) < 0.5)] = -0.0
  return base


DTYPES = [np.uint8, np.int16, np.uint32, np.int64, np.float32, np.float64, np.bool_]
# r: 0; within the window limit (R = 1, 2); just above it (R = 3); far above (R = 12)
RADII = [0.0, 1.5, 2.0, 3.0, 12.5]


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("op", mc.OPS)
def test_dtypes_orders_radii(edt, op, dtype, order):
  rng = np.random.default_rng(mc.OPS.index(op) * 10 + DTYPES.index(dtype))
  shape = (30, 27, 22)
  if dtype == np.bool_:
    arr = mc.balls(rng, shape, 6, 8.0, np.uint8) != 0
  elif np.dtype(dtype).kind == "f":
    arr = float_labels(rng, shape, dtype)
  else:
    arr = mc.seeded(rng, ("voronoi", "balls", "touching")[DTYPES.index(dtype) % 3], shape, dtype)
  arr = np.asfortranarray(arr) if order == "F" else np.ascontiguousarray(arr)
  for r in RADII:
    for bb in (False, True):
      got = run(edt, op, arr, r, None, bb)
      check_path(edt, arr, r, None)
      assert same(got, want(op, arr, r, None, bb)), (r, bb)
      assert got.flags.f_contiguous == (order == "F")
      if op in ("erode", "open") and r == 0.0 and dtype != np.bool_:
        assert same(got, mc._keep(arr, arr != 0))          # identity, background as all-zero bits


@pytest.mark.parametrize("w", [(1.0, 2.0, 1.0), (0.7, 1.3, 2.9), (3.0, 1.0, 0.5)])
@pytest.mark.parametrize("op", mc.OPS)
def test_anisotropy(edt, op, w):
  rng = np.random.default_rng(7)
  arr = np.asfortranarray(mc.voronoi(rng, (26, 21, 24), 7, np.uint16))
  for r in (0.9, 2.0, 2.6, 4.2, 11.0):
    for bb in (False, True):
      got = run(edt, op, arr, r, w, bb)
      check_path(edt, arr, r, w)
      assert same(got, want(op, arr, r, w, bb)), (r, bb)


@pytest.mark.parametrize("op", mc.OPS)
@pytest.mark.parametrize("shape", [(300,), (70, 45), (9, 300)], ids=["1d", "2d", "2d_tall"])
def test_one_and_two_dimensions(edt, op, shape):
  rng = np.random.default_rng(len(shape) * 3 + shape[0])
  for kind in mc.KINDS:
    arr = mc.seeded(rng, kind, shape, np.uint32)
    for r in (0.0, 1.0, 2.0, 2.5, 3.0, 17.0):
      for bb in (False, True):
        w = (1.5,) if len(shape) == 1 else (1.0, 2.0)
        got = run(edt, op, arr, r, w, bb)
        check_path(edt, arr, r, w)
        assert same(got, want(op, arr, r, w, bb)), (kind, r, bb)


def test_bridges_and_specks(edt):
  arr = mc.bridges((30, 16, 14))
  opened = edt.spherical_open(arr, 1.0)
  assert not (opened == 3).any()                          # the speck of 3 is gone
  assert same(opened, want("open", arr, 1.0))
  assert same(edt.spherical_erode(arr, 1.0), want("erode", arr, 1.0))


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("nd", [2, 3, 4])
@pytest.mark.parametrize("op", mc.OPS)
def test_stacks_equal_the_per_volume_calls(edt, op, nd, order):
  rng = np.random.default_rng(nd * 7 + (order == "F"))
  vshape = {2: (200,), 3: (40, 33), 4: (19, 17, 23)}[nd]
  count = 3
  vols = [mc.seeded(rng, mc.KINDS[b % 4], vshape, np.int32) for b in range(count)]
  w = (1.0, 2.0, 0.7)[:nd - 1]
  if order == "C":
    stack = np.ascontiguousarray(np.stack(vols))
  else:
    stack = np.asfortranarray(np.stack(vols, axis=-1))
  for r in (1.0, 2.0, 3.5):
    for bb in (False, True):
      got = run(edt, op, stack, r, w, bb, stacked=True)
      per = [run(edt, op, v, r, w, bb) for v in vols]
      exp = np.stack(per) if order == "C" else np.stack(per, axis=-1)
      assert same(got, exp), (r, bb)
      assert same(per[0], want(op, vols[0], r, w, bb))
      assert got.flags.f_contiguous == (order == "F")


def test_every_pass_windowed_on_a_stack(edt):
  """r = 2 with unit weights: both later passes take the window kernel, the first writing distances
  through the scratch volume, the last writing the labels."""
  rng = np.random.default_rng(3)
  vols = [mc.voronoi(rng, (36, 34, 40), 9, np.uint64) for _ in range(2)]
  stack = np.stack(vols)
  for op in mc.OPS:
    got = run(edt, op, stack, 2.0, None, True, stacked=True)
    assert edt.last_later_launch()["kernel"] == "window"
    assert same(got, np.stack([want(op, v, 2.0, None, True) for v in vols])), op


@pytest.mark.parametrize("op", mc.OPS)
def test_device_input_on_a_non_default_stream(edt, op):
  import torch
  rng = np.random.default_rng(21)
  arr = mc.voronoi(rng, (28, 31, 25), 6, np.int32)
  stack = np.stack([arr, mc.balls(rng, arr.shape, 5, 7.0, np.int32)])
  dev = torch.from_numpy(arr).cuda()
  devf =torch.from_numpy(np.ascontiguousarray(arr.T)).cuda().permute(2, 1, 0)        # F-ordered view
  devs = torch.from_numpy(stack).cuda()
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    outs = [run(edt, op, x, 2.5, (1.0, 1.0, 2.0), True) for x in (dev, devf)]
    outs.append(run(edt, op, devs, 2.5, (1.0, 1.0, 2.0), True, stacked=True))
  side.synchronize()
  exp = want(op, arr, 2.5, (1.0, 1.0, 2.0), True)
  for o in outs:
    assert isinstance(o, torch.Tensor) and o.is_cuda
  assert same(outs[0].cpu().numpy(), exp)
  assert not outs[1].is_contiguous() and outs[1].permute(2, 1, 0).is_contiguous()
  assert same(outs[1].cpu().numpy(), exp)
  assert same(outs[2].cpu().numpy(), np.stack([exp, want(op, stack[1], 2.5, (1.0, 1.0, 2.0), True)]))


def test_device_float_labels(edt):
  import torch
  rng = np.random.default_rng(4)
  arr = float_labels(rng, (20, 24, 18), np.float64)
  for op in mc.OPS:
    got = run(edt, op, torch.from_numpy(arr).cuda(), 2.0, None, True).cpu().numpy()
    assert same(got, want(op, arr, 2.0, None, True)), op


def test_lattice_properties(edt):
  rng = np.random.default_rng(9)
  for arr in (mc.voronoi(rng, (30, 28, 26), 8, np.uint16), mc.balls(rng, (30, 28, 26), 8, 9.0, np.uint16),
              mc.bridges((30, 28, 26))):
    for r in (1.0, 2.0, 3.0, 6.5):
      for w in (None, (1.0, 0.7, 2.2)):
        for bb in (False, True):
          opened = edt.spherical_open(arr, r, w, bb)
          assert np.array_equal(opened[opened != 0], arr[opened != 0])      # open(x) within x, labels kept
          assert np.array_equal(edt.spherical_open(opened, r, w, bb), opened)
        closed = edt.spherical_close(arr, r, w)
        assert closed[arr != 0].all()                                     # x within close(x)
        assert np.array_equal(edt.spherical_dilate(arr, r, w), want("dilate", arr, r, w))
