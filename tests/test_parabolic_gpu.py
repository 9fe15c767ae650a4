"""GPU tests: parabolic_erode / parabolic_dilate equal the restatement in parabolic_cases.py bit for bit,
on every kernel (tile X and Y / Z passes, the long-line hull past 1024 samples, the brute-force minimum
past 23170, the copy of an overflowing w^2), every value family, both memory orders, stacks, host and
device residency, in place and on a side stream; and the identities: a 0 / +inf mask gives edtsq, C order
equals F order."""
import ctypes

import numpy as np
import pytest

import parabolic_cases as pc

pytestmark = pytest.mark.gpu
OPS = ["erode", "dilate"]
WEIGHTS3 = [(1.0, 1.0, 1.0), (6.0, 6.0, 30.0), (0.7, 1.3, 2.9), (2.0 ** -26,) * 3, (1e20, 1.0, 1e20)]


def _call(edt, op, f, w=None, **kw):
  return getattr(edt, "parabolic_" + op)(f, w, **kw)


def _check(edt, op, f, w=None, order="C", stacked=False):
  got = _call(edt, op, f, w, stacked=stacked)
  want = pc.restate(op, f, w, order=order, stacked=stacked)
  assert isinstance(got, np.ndarray) and got.dtype == np.float32 and got.shape == np.shape(f)
  want = want.astype(np.float32)
  bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))         # element by element, any layout
  assert len(bad) == 0, (op, np.shape(f), w, order, len(bad), [(tuple(b), got[tuple(b)], want[tuple(b)]) for b in bad[:4]])


SIZES = [1, 2, 31, 32, 33, 1023, 1024, 1025]


@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("n", SIZES)
def test_every_axis_at_every_size(edt, axis, n):
  rng = np.random.default_rng(10 * n + axis)
  shape = [3, 4, 5]
  shape[axis] = n
  for k, op in enumerate(OPS):
    fam = pc.FAMILIES[(SIZES.index(n) + axis + k) % len(pc.FAMILIES)]
    f = pc.values(fam, tuple(shape), rng)
    _check(edt, op, f, WEIGHTS3[(axis + k) % 3])


@pytest.mark.parametrize("family", pc.FAMILIES)
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("w", WEIGHTS3, ids=["1", "6-6-30", "frac", "tiny", "overflow"])
def test_every_value_family(edt, family, op, w):
  rng = np.random.default_rng(pc.FAMILIES.index(family))
  f = pc.values(family, (19, 34, 37), rng)
  _check(edt, op, f, w)


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("shape", [(3, 700), (700, 3), (700, 2, 3), (2, 2100)], ids=str)
def test_near_ties(edt, op, shape):
  rng = np.random.default_rng(len(shape))
  # lines along every axis carry the construction: transpose it onto the axis of length >= 700
  axis = int(np.argmax(shape))
  moved = list(shape)
  moved[axis], moved[-1] = moved[-1], moved[axis]
  f = np.swapaxes(pc.values("near_tie", tuple(moved), rng), axis, -1).copy()
  if op == "dilate":
    f = -f
  w = [1.0] * len(shape)
  w[axis] = pc.NEAR_TIE_W
  _check(edt, op, f, tuple(w))


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("family", ["wide", "special", "integers"])
def test_long_lines(edt, op, family):
  rng = np.random.default_rng(3)
  _check(edt, op, pc.values(family, (2, 3000), rng), (0.7, 1.3))        # X: the long-line hull
  _check(edt, op, pc.values(family, (3000, 3), rng), (2.9, 1.0))        # Y: the long-line hull
  _check(edt, op, pc.values(family, (23170,), rng), 1.3)                 # the last length the hull takes


@pytest.mark.parametrize("op", OPS)
def test_lines_past_the_exact_hull(edt, op):
  rng = np.random.default_rng(4)
  _check(edt, op, pc.values("wide", (23200,), rng), 0.7)                 # the brute-force minimum
  f = pc.values("uniform", (23171, 1), rng)
  _check(edt, op, f, (1.0, 3.0))                                         # Y pass, and in place


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("shape", [(40,), (33, 47), (17, 33, 29)], ids=lambda s: "%dd" % len(s))
def test_orders_and_the_c_f_identity(edt, op, order, shape):
  rng = np.random.default_rng(5)
  f = pc.values("wide", shape, rng)
  w = (0.7, 1.3, 2.9)[:len(shape)]
  arr = np.asfortranarray(f) if order == "F" else f
  _check(edt, op, arr, w, order=order)
  fo = np.asfortranarray(f.T)                                            # the same bytes, F order
  got_c = _call(edt, op, f, w)
  got_f = _call(edt, op, fo, tuple(reversed(w)))
  assert got_f.flags.f_contiguous or len(shape) == 1
  assert pc.same_bits(got_c.T, got_f)


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("count,shape", [(1, (9, 10, 11)), (3, (9, 10, 11)), (3, (40, 33)), (4000, (4, 5)),
                                         (5000, (7,))], ids=str)
def test_stacks(edt, op, count, shape):
  rng = np.random.default_rng(count)
  f = pc.values("uniform" if count < 100 else "special", (count,) + shape, rng)
  w = (1.3, 0.7, 2.9)[:len(shape)]
  got = _call(edt, op, f, w, stacked=True)
  assert pc.same_bits(got, np.stack([pc.restate(op, v, w) for v in f]))
  got_f = _call(edt, op, np.asfortranarray(f.T), tuple(reversed(w)), stacked=True)
  assert pc.same_bits(got_f.T, got)


@pytest.mark.parametrize("dtype", [np.float64, np.float16, np.int32, np.uint8, np.bool_])
def test_dtypes_convert_to_float32_first(edt, dtype):
  rng = np.random.default_rng(6)
  f = (rng.uniform(-100, 100, (9, 14, 12)) if dtype != np.bool_ else rng.random((9, 14, 12)) < 0.5).astype(dtype)
  if np.dtype(dtype).kind in "iu":
    f = np.abs(f)
  _check(edt, "erode", f, (0.7, 1.3, 2.9))
  _check(edt, "dilate", f.tolist() if dtype == np.int32 else f, (0.7, 1.3, 2.9))


@pytest.mark.parametrize("w", [(1.0, 1.0, 1.0), (6.0, 6.0, 30.0), (2.0, 3.0, 5.0)])
def test_a_mask_gives_edtsq(edt, w):
  rng = np.random.default_rng(7)
  mask = rng.random((33, 40, 37)) < 0.9
  got = edt.parabolic_erode(np.where(mask, np.inf, 0), w)
  assert pc.same_bits(got, edt.edtsq(mask.astype(np.uint8), w))
  stack = rng.random((3, 20, 33)) < 0.9
  got = edt.parabolic_erode(np.where(stack, np.inf, 0), w[:2], stacked=True)
  assert pc.same_bits(got, edt.edtsq(stack.astype(np.uint8), w[:2], stacked=True))


def test_device_residency_in_place_and_side_stream(edt):
  import torch
  rng = np.random.default_rng(8)
  f = pc.values("wide", (21, 34, 40), rng)
  w = (0.7, 1.3, 2.9)
  want = pc.erode(f, w)
  t = torch.from_numpy(f).cuda()
  got = edt.parabolic_erode(t, w)
  assert got.is_cuda and got.dtype == torch.float32 and pc.same_bits(got.cpu().numpy(), want)
  tf = torch.from_numpy(np.asfortranarray(f)).cuda().permute(2, 1, 0).contiguous().permute(2, 1, 0)
  got = edt.parabolic_dilate(tf, w)                                      # an F-ordered device view
  assert got.stride() == tf.stride() and pc.same_bits(got.cpu().numpy(), pc.dilate(np.asfortranarray(f), w, "F"))
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    t2 = torch.from_numpy(f).cuda()
    got = edt.parabolic_erode(t2, w)
  side.synchronize()
  assert pc.same_bits(got.cpu().numpy(), want)
  # in place through the C ABI: out == f
  t3 = torch.from_numpy(f).cuda()
  lib = edt._lib()
  stream = torch.cuda.current_stream().cuda_stream
  rc = lib.edtb200_parabolic(t3.data_ptr(), 3, 40, 34, 21, 1, 2.9, 1.3, 0.7, 0, 12, t3.data_ptr(), 0,
                             ctypes.c_void_p(stream))
  assert rc == 0
  assert pc.same_bits(t3.cpu().numpy(), want)
  # in place past both the tile and the exact-hull limits
  g = pc.values("uniform", (23171,), rng)
  t4 = torch.from_numpy(g).cuda()
  assert lib.edtb200_parabolic(t4.data_ptr(), 1, 23171, 1, 1, 1, 0.7, 1.0, 1.0, 1, 12, t4.data_ptr(), 0,
                               ctypes.c_void_p(stream)) == 0
  assert pc.same_bits(t4.cpu().numpy(), pc.dilate(g, 0.7))
  g = pc.values("wide", (2, 1500), rng)
  t5 = torch.from_numpy(g).cuda()
  assert lib.edtb200_parabolic(t5.data_ptr(), 2, 1500, 2, 1, 1, 0.7, 1.3, 1.0, 0, 12, t5.data_ptr(), 0,
                               ctypes.c_void_p(stream)) == 0
  assert pc.same_bits(t5.cpu().numpy(), pc.erode(g, (1.3, 0.7)))


def test_empty_device_input(edt):
  import torch
  got = edt.parabolic_erode(torch.zeros((0, 3), device="cuda"))
  assert got.is_cuda and got.shape == (0, 3)


# Lines where the hull predicates' double evaluation has the wrong sign (parabolic_cases.CANCEL_CASES):
# only the exact fallback gives these results.  On the tile kernels (the pattern inside one segment and
# across the boundary of the segments of a 4-warp tile: n = 40 has segments of 10) and on the long-line
# hull, along every axis, eroded and dilated.
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("case", [0, 1], ids=["read_out", "hull"])
@pytest.mark.parametrize("n,at", [(2, 0), (3, 0), (40, 3), (40, 9), (1024, 500), (1500, 700)], ids=str)
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_only_the_exact_fallback_decides(edt, op, case, n, at, axis):
  src, want = pc.CANCEL_CASES[case]
  if at + len(src) > n:
    pytest.skip("the pattern does not fit")
  line = pc.cancel_line(n, case, at)
  shape = [2, 3, 2]
  shape[axis] = n
  f = np.moveaxis(np.broadcast_to(line, tuple(shape[:axis] + shape[axis + 1:]) + (n,)), -1, axis).copy()
  w = [1.0, 1.0, 1.0]
  w[axis] = pc.CANCEL_W
  sign = 1.0 if op == "erode" else -1.0
  got = _call(edt, op, sign * f, tuple(w))
  idx = [slice(None)] * 3
  idx[axis] = slice(at, at + len(src))
  expect = np.moveaxis(np.broadcast_to(np.float32(want), tuple(shape[:axis] + shape[axis + 1:]) + (len(src),)), -1, axis)
  assert pc.same_bits(got[tuple(idx)], np.where(expect == 0, np.float32(0), sign * expect))
  _check(edt, op, sign * f, tuple(w))
