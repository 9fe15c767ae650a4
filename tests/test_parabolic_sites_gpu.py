"""GPU tests: parabolic_erode / parabolic_dilate with return_indices=True.  The values are bit for bit those
of the call without indices, and the indices equal the restatement in parabolic_sites_cases.py exactly, on
every kernel (tile X and Y / Z passes with 1, 2 or 4 segments, the long-line hull, the brute-force minimum
past 23170 samples, the copy of an overflowing w^2), every value family and weight set, near ties and the
lines only the exact predicates decide, both memory orders, dtypes, stacks, device input, in place, a side
stream and empty input; and at scale, a power diagram by the chain identity and by brute force."""
import ctypes

import numpy as np
import pytest

import parabolic_cases as pc
import parabolic_sites_cases as sc

pytestmark = pytest.mark.gpu
OPS = ["erode", "dilate"]
WEIGHTS3 = [(1.0, 1.0, 1.0), (6.0, 6.0, 30.0), (0.7, 1.3, 2.9), (2.0 ** -26,) * 3, (1e20, 1.0, 1e20)]
SIZES = [1, 2, 31, 32, 33, 1023, 1024, 1025]


def _call(edt, op, f, w=None, **kw):
  return getattr(edt, "parabolic_" + op)(f, w, **kw)


def _check(edt, op, f, w=None, order="C", stacked=False):
  vals, idx = _call(edt, op, f, w, stacked=stacked, return_indices=True)
  plain = _call(edt, op, f, w, stacked=stacked)
  want_v, want_i = sc.restate(op, f, w, order=order, stacked=stacked)
  assert isinstance(idx, np.ndarray) and idx.dtype == np.int32 and idx.shape == want_i.shape
  assert pc.same_bits(vals, plain), "the values differ from the call without indices"
  assert pc.same_bits(vals, want_v)
  bad = np.argwhere(np.any(idx != want_i, axis=0))
  assert len(bad) == 0, (op, np.shape(f), w, order, len(bad),
                         [(tuple(b), idx[(slice(None),) + tuple(b)], want_i[(slice(None),) + tuple(b)]) for b in bad[:4]])
  return vals, idx


@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("n", SIZES)
def test_every_axis_at_every_size(edt, axis, n):
  rng = np.random.default_rng(10 * n + axis)
  shape = [3, 4, 5]
  shape[axis] = n
  for k, op in enumerate(OPS):
    fam = pc.FAMILIES[(SIZES.index(n) + axis + k) % len(pc.FAMILIES)]
    _check(edt, op, pc.values(fam, tuple(shape), rng), WEIGHTS3[(axis + k) % 3])
    _check(edt, op, pc.values("integers", tuple(shape), rng), (1.0, 1.0, 1.0))      # many exact ties


@pytest.mark.parametrize("family", pc.FAMILIES)
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("w", WEIGHTS3, ids=["1", "6-6-30", "frac", "tiny", "overflow"])
def test_every_value_family(edt, family, op, w):
  rng = np.random.default_rng(pc.FAMILIES.index(family))
  _check(edt, op, pc.values(family, (9, 34, 37), rng), w)


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("shape", [(3, 700), (700, 3), (700, 2, 3), (2, 2100)], ids=str)
def test_near_ties(edt, op, shape):
  rng = np.random.default_rng(len(shape))
  axis = int(np.argmax(shape))
  moved = list(shape)
  moved[axis], moved[-1] = moved[-1], moved[axis]
  f = np.swapaxes(pc.values("near_tie", tuple(moved), rng), axis, -1).copy()
  if op == "dilate":
    f = -f
  w = [1.0] * len(shape)
  w[axis] = pc.NEAR_TIE_W
  _check(edt, op, f, tuple(w))
  # the same line on every row: the next pass compares equal values above 2^24
  line = np.take(f, [0], axis=0 if axis else 1)
  _check(edt, op, np.repeat(line, 3, axis=0 if axis else 1).copy(), tuple(w))


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("family", ["wide", "special", "integers"])
def test_long_lines(edt, op, family):
  rng = np.random.default_rng(3)
  _check(edt, op, pc.values(family, (2, 1500), rng), (0.7, 1.3))        # X: the long-line hull
  _check(edt, op, pc.values(family, (1500, 3), rng), (2.9, 1.0))        # Y: the long-line hull
  _check(edt, op, pc.values(family, (23170,), rng), 1.3)                 # the last length the hull takes


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("family", ["wide", "integers", "special"])
def test_lines_past_the_exact_hull(edt, op, family):
  rng = np.random.default_rng(4)
  _check(edt, op, pc.values(family, (23171,), rng), 0.7)                 # the brute-force minimum
  _check(edt, op, pc.values(family, (23172, 1), rng), (1.0, 3.0))        # its Y pass


# The lines of test_parabolic_gpu.test_only_the_exact_fallback_decides, and their negations (+inf padding
# kept), on which two candidates one row apart round alike: only an exact comparison names the site, in
# one segment or across the boundary of two (n = 40 has segments of 10 on a 4-warp tile).
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("case", [0, 1], ids=["read_out", "hull"])
@pytest.mark.parametrize("n,at", [(2, 0), (3, 0), (40, 3), (40, 9), (1024, 500), (1500, 700)], ids=str)
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_only_the_exact_predicates_decide(edt, op, case, n, at, axis):
  src = pc.CANCEL_CASES[case][0]
  if at + len(src) > n:
    pytest.skip("the pattern does not fit")
  line = pc.cancel_line(n, case, at)
  shape = [2, 3, 2]
  shape[axis] = n
  w = [1.0, 1.0, 1.0]
  w[axis] = pc.CANCEL_W
  sign = 1.0 if op == "erode" else -1.0
  for pattern in (line, np.where(np.isinf(line), line, -line)):
    f = np.moveaxis(np.broadcast_to(pattern, tuple(shape[:axis] + shape[axis + 1:]) + (n,)), -1, axis).copy()
    _check(edt, op, sign * f, tuple(w))


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("shape", [(40,), (33, 47), (17, 33, 29)], ids=lambda s: "%dd" % len(s))
def test_orders(edt, op, order, shape):
  rng = np.random.default_rng(5)
  f = pc.values("integers", shape, rng)
  w = (1.0, 2.0, 1.0)[:len(shape)]
  arr = np.asfortranarray(f) if order == "F" else f
  _check(edt, op, arr, w, order=order)
  # the bytes of f in F order: the same passes, so the same sites, the axes reversed
  _, idx_t = _call(edt, op, np.asfortranarray(f.T), tuple(reversed(w)), return_indices=True)
  assert np.array_equal(idx_t[::-1].transpose((0,) + tuple(range(len(shape), 0, -1))), sc.restate(op, f, w)[1])


@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("count,shape", [(1, (9, 10, 11)), (3, (9, 10, 11)), (3, (40, 33)), (4000, (4, 5)),
                                         (5000, (7,))], ids=str)
def test_stacks(edt, op, count, shape):
  rng = np.random.default_rng(count)
  f = pc.values("integers" if count < 100 else "special", (count,) + shape, rng)
  w = (1.0, 2.0, 1.0)[:len(shape)]
  _, idx = _check(edt, op, f, w, stacked=True)
  for b in range(min(count, 3)):
    assert np.array_equal(idx[:, b], sc.restate(op, f[b], w)[1])
  _, idx_f = _call(edt, op, np.asfortranarray(f.T), tuple(reversed(w)), stacked=True, return_indices=True)
  assert np.array_equal(idx_f[::-1].transpose((0,) + tuple(range(len(shape) + 1, 0, -1))), idx)


@pytest.mark.parametrize("dtype", [np.float64, np.float16, np.int32, np.uint8, np.bool_])
def test_dtypes_convert_to_float32_first(edt, dtype):
  rng = np.random.default_rng(6)
  f = (rng.uniform(-100, 100, (9, 14, 12)) if dtype != np.bool_ else rng.random((9, 14, 12)) < 0.5).astype(dtype)
  if np.dtype(dtype).kind in "iu":
    f = np.abs(f)
  _check(edt, "erode", f, (1.0, 1.0, 1.0))
  _check(edt, "dilate", f, (0.7, 1.3, 2.9))


def test_a_mask_gives_its_edtsq_at_the_index(edt):
  rng = np.random.default_rng(7)
  mask = rng.random((33, 40, 37)) < 0.9
  w = (2.0, 3.0, 5.0)
  vals, idx = edt.parabolic_erode(np.where(mask, np.inf, 0), w, return_indices=True)
  P = np.indices(mask.shape)
  d2 = sum((w[k] * (P[k] - idx[k]).astype(np.float64)) ** 2 for k in range(3))
  assert pc.same_bits(d2.astype(np.float32), edt.edtsq(mask.astype(np.uint8), w)) and pc.same_bits(vals, d2)
  assert not mask[tuple(idx)].any()


def test_device_input_in_place_side_stream_and_empty(edt):
  import torch
  rng = np.random.default_rng(8)
  f = pc.values("integers", (21, 34, 40), rng)
  w = (1.0, 2.0, 1.0)
  want_v, want_i = sc.restate("erode", f, w)
  vals, idx = edt.parabolic_erode(torch.from_numpy(f).cuda(), w, return_indices=True)
  assert vals.is_cuda and idx.is_cuda and idx.dtype == torch.int32 and tuple(idx.shape) == (3,) + f.shape
  assert pc.same_bits(vals.cpu().numpy(), want_v) and np.array_equal(idx.cpu().numpy(), want_i)
  tf = torch.from_numpy(np.asfortranarray(f)).cuda().permute(2, 1, 0).contiguous().permute(2, 1, 0)
  vals, idx = edt.parabolic_dilate(tf, w, return_indices=True)                 # an F-ordered device view
  dv, di = sc.restate("dilate", np.asfortranarray(f), w, order="F")
  assert vals.stride() == tf.stride() and pc.same_bits(vals.cpu().numpy(), dv)
  assert np.array_equal(idx.cpu().numpy(), di)
  st = torch.from_numpy(f[:4]).cuda()
  vals, idx = edt.parabolic_erode(st, w[1:], stacked=True, return_indices=True)
  assert np.array_equal(idx.cpu().numpy(), sc.restate("erode", f[:4], w[1:], stacked=True)[1])
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    vals, idx = edt.parabolic_erode(torch.from_numpy(f).cuda(), w, return_indices=True)
  side.synchronize()
  assert pc.same_bits(vals.cpu().numpy(), want_v) and np.array_equal(idx.cpu().numpy(), want_i)
  # in place through the C ABI (out == f), idx x first, on every kernel
  lib = edt._lib()
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  for arr, ww in ((f, w), (pc.values("wide", (2, 1500), rng), (1.3, 0.7)), (pc.values("uniform", (23171,), rng), (0.7,))):
    t = torch.from_numpy(arr).cuda()
    planes = torch.full((arr.ndim,) + arr.shape, 7, dtype=torch.int32, device="cuda")
    sizes = list(reversed(arr.shape)) + [1] * (3 - arr.ndim)
    wx = list(reversed(ww)) + [1.0] * (3 - arr.ndim)
    assert lib.edtb200_parabolic_sites(t.data_ptr(), arr.ndim, *sizes, 1, *wx, 0, 12, t.data_ptr(),
                                       planes.data_ptr(), 0, stream) == 0
    rv, ri = sc.restate("erode", arr, ww)
    assert pc.same_bits(t.cpu().numpy(), rv) and np.array_equal(planes.flip(0).cpu().numpy(), ri)
  vals, idx = edt.parabolic_erode(torch.zeros((0, 3), device="cuda"), return_indices=True)
  assert vals.is_cuda and idx.is_cuda and tuple(idx.shape) == (2, 0, 3)


def _power_seeds(rng, shape, count):
  flat = rng.choice(int(np.prod(shape)), count, replace=False)
  seeds = np.stack(np.unravel_index(flat, shape), axis=1)
  omega = rng.integers(0, 400, count).astype(np.float32)      # integer weights: every value exact
  return seeds, omega


def test_a_power_diagram_at_scale(edt):
  rng = np.random.default_rng(21)
  shape = (256, 256, 256)
  seeds, omega = _power_seeds(rng, shape, 3000)
  f = np.full(shape, np.inf, np.float32)
  f[tuple(seeds.T)] = -omega
  labels = np.zeros(shape, np.int32)
  labels[tuple(seeds.T)] = np.arange(1, len(seeds) + 1)
  vals, idx = edt.parabolic_erode(f, return_indices=True)
  assert pc.same_bits(vals, edt.parabolic_erode(f))
  assert pc.same_bits(vals, sc.chain("erode", f, idx))                         # every voxel
  cells = labels[tuple(idx)]
  assert cells.min() >= 1
  # brute force at 10^5 voxels: the seed named attains the least power distance |p - c|^2 - omega_c
  pick = rng.integers(0, 256, (100000, 3))
  got = cells[tuple(pick.T)] - 1
  for s in range(0, len(pick), 2000):
    p = pick[s:s + 2000]
    power = ((p[:, None, :] - seeds[None, :, :]) ** 2).sum(axis=2) - omega[None, :].astype(np.int64)
    low = power.min(axis=1)
    assert np.array_equal(power[np.arange(len(p)), got[s:s + 2000]], low)
    assert np.array_equal(vals[tuple(p.T)], low.astype(np.float32))
