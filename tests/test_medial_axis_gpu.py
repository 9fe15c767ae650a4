"""GPU tests: medial_axis equals the restatement in medial_axis_cases.py exactly -- every label dtype (-0.0
included), both memory orders, 1-D to 3-D, both borders, integer weights; for other weights it equals the
composition of the public calls (edtsq, then parabolic_dilate with return_indices) and rebuilds every label.
Also stacks against per-volume calls, host and device residency, a side stream, empty arrays, one-label
volumes, return_distance against edt() bit for bit, the long-line tiers of the parabolic passes, and at
256^3 Voronoi cells and balls against the composition and the reconstruction at every voxel."""
import ctypes

import numpy as np
import pytest

import medial_axis_cases as mac
import parabolic_cases as pc

pytestmark = pytest.mark.gpu

INT_WEIGHTS = {1: [(1.0,), (3.0,)], 2: [(1.0, 1.0), (2.0, 1.0)], 3: [(1.0, 1.0, 1.0), (1.0, 2.0, 3.0)]}
FRAC_WEIGHTS = {1: (0.7,), 2: (1.3, 0.45), 3: (0.9, 1.7, 2.3)}
SHAPES = {1: (61,), 2: (23, 37), 3: (9, 13, 17)}


def _composition(edt, labels, w, border, order="C", stacked=False):
  """What a user computes today from the public calls: (medial, D2, V)."""
  d2 = edt.edtsq(labels, w, border, stacked=stacked) if stacked else edt.edtsq(labels, w, border)
  v, idx = edt.parabolic_dilate(d2, w, stacked=stacked, return_indices=True)
  return mac.mark(labels, idx, order, stacked), d2, v


def _check(edt, labels, w, border, order="C", stacked=False, exact=True):
  medial, dist = edt.medial_axis(labels, w, border, return_distance=True, stacked=stacked)
  assert isinstance(medial, np.ndarray) and medial.dtype == np.bool_ and medial.shape == labels.shape
  assert medial.flags.f_contiguous if order == "F" and labels.ndim > 1 else medial.flags.c_contiguous
  assert np.array_equal(edt.medial_axis(labels, w, border, stacked=stacked), medial)
  comp, d2, v = _composition(edt, labels, w, border, order, stacked)
  assert np.array_equal(medial, comp), (labels.shape, w, border, order, int((medial != comp).sum()))
  if stacked:
    want_dist = edt.edt(labels, w, border, stacked=True)
  else:
    want_dist = edt.edt(labels, w, border)
  assert pc.same_bits(dist, want_dist)
  if exact:
    want = mac.restate(labels, w, border, order, stacked)[0]
    assert np.array_equal(medial, want), (labels.shape, w, border, order, int((medial != want).sum()))
  fg = labels != 0
  rec = mac.reconstruct(medial, d2, w, order, stacked)
  assert np.array_equal(rec[fg], v[fg]) and np.all(rec[fg] > 0)
  if exact:
    assert np.array_equal(rec > 0, fg)
  return medial


@pytest.mark.parametrize("dtype", [np.bool_, np.uint8, np.uint16, np.uint32, np.uint64, np.int32, np.float32,
                                   np.float64])
def test_every_label_dtype(edt, dtype):
  rng = np.random.default_rng(np.dtype(dtype).num)
  for kind in mac.KINDS:
    base = mac.seeded(rng, kind, (11, 14, 16), np.uint16)
    if dtype == np.bool_:
      labels = base != 0
    elif np.dtype(dtype).kind == "f":
      labels = np.where(base == 0, np.where(rng.random(base.shape) < 0.5, -0.0, 0.0), base * 1.5 - 2.0).astype(dtype)
      assert not (labels == 0).any() or np.signbit(labels[labels == 0]).any()
    elif dtype == np.int32:
      labels = (base.astype(np.int32) - 2) * (base != 0)               # negative labels too
    else:
      labels = (base.astype(np.uint64) * (np.iinfo(dtype).max // 7)).astype(dtype)
    for border in (False, True):
      _check(edt, labels, (1.0, 2.0, 1.0), border)


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("nd", [1, 2, 3])
@pytest.mark.parametrize("border", [False, True])
def test_orders_dims_borders_and_weights(edt, order, nd, border):
  rng = np.random.default_rng(nd + 7 * border)
  for kind in mac.KINDS + ("noise",):
    labels = (rng.integers(0, 3, SHAPES[nd]).astype(np.uint32) if kind == "noise"
              else mac.seeded(rng, kind, SHAPES[nd], np.uint32))
    labels = np.asfortranarray(labels) if order == "F" else np.ascontiguousarray(labels)
    for w in INT_WEIGHTS[nd]:
      _check(edt, labels, w, border, order)
    _check(edt, labels, FRAC_WEIGHTS[nd], border, order, exact=False)


@pytest.mark.parametrize("order", ["C", "F"])
def test_stacks_are_the_per_volume_calls(edt, order):
  rng = np.random.default_rng(4)
  for shape, w in (((5, 40), (1.0,)), ((4, 13, 9), (2.0, 1.0)), ((3, 7, 6, 5), (1.0, 1.0, 2.0)),
                   ((6, 8, 8), (0.8, 1.3))):
    vols = [mac.seeded(rng, mac.KINDS[i % 4], shape[1:], np.uint8) for i in range(shape[0])]
    vols[1][...] = 0
    vols[-1][...] = 3                                                      # a one-label volume: one mark
    labels = np.stack(vols) if order == "C" else np.asfortranarray(np.stack([v.T for v in vols]).T)
    axis = 0 if order == "C" else labels.ndim - 1
    # a volume keeps the stack's memory order: x is its fastest axis, which decides the passes and ties
    vol = (lambda i: np.asfortranarray(np.take(labels, i, axis))) if order == "F" else (lambda i: labels[i])
    for border in (False, True):
      got = _check(edt, labels, w, border, order, stacked=True, exact=w[0] == int(w[0]))
      each = [edt.medial_axis(vol(i), w, border) for i in range(labels.shape[axis])]
      assert np.array_equal(got, np.stack(each, axis))
      if not border:                                                       # each volume marks its own first voxel
        last = np.take(got, labels.shape[axis] - 1, axis)
        assert last.sum() == 1 and last.reshape(-1, order=order)[0]
      assert not np.take(got, 1, axis).any()


def test_one_label_volumes_and_empty_arrays(edt):
  for shape in ((9,), (4, 6), (3, 5, 2)):
    for dtype in (np.uint8, np.float64):
      labels = np.full(shape, 5, dtype)
      medial, dist = edt.medial_axis(labels, return_distance=True)
      assert np.flatnonzero(medial).tolist() == [0] and np.all(np.isinf(dist))
      assert np.array_equal(edt.medial_axis(np.asfortranarray(labels)).reshape(-1, order="F"),
                            np.arange(labels.size) == 0)
      _check(edt, labels, None, True)
  for shape in ((0,), (3, 0), (0, 2, 2)):
    medial, dist = edt.medial_axis(np.zeros(shape, np.uint16), return_distance=True)
    assert medial.shape == shape and dist.shape == shape and medial.dtype == np.bool_


def test_the_worked_examples(edt):
  five = np.array([0, 1, 1, 1, 1, 1, 0], np.uint8)
  assert np.flatnonzero(edt.medial_axis(five)).tolist() == [3]
  four = np.array([0, 2, 2, 2, 2, 0], np.int64)
  assert np.flatnonzero(edt.medial_axis(four)).tolist() == [2, 3]


def test_device_residency_and_a_side_stream(edt):
  import torch
  rng = np.random.default_rng(9)
  labels = mac.seeded(rng, "voronoi", (12, 17, 19), np.int32)
  w = (1.0, 1.0, 2.0)
  want, want_dist = edt.medial_axis(labels, w, True, return_distance=True)
  assert np.array_equal(want, mac.restate(labels, w, True)[0])
  t = torch.from_numpy(labels).cuda()
  got, dist = edt.medial_axis(t, w, True, return_distance=True)
  assert got.is_cuda and got.dtype == torch.bool and dist.is_cuda and dist.dtype == torch.float32
  assert np.array_equal(got.cpu().numpy(), want) and pc.same_bits(dist.cpu().numpy(), want_dist)
  # an F-ordered device view: x is its first axis, which decides the passes and ties, as for a host F array
  tf = torch.from_numpy(np.asfortranarray(labels)).cuda().permute(2, 1, 0).contiguous().permute(2, 1, 0)
  got = edt.medial_axis(tf, w, True)
  want_f = mac.restate(np.asfortranarray(labels), w, True, order="F")[0]
  assert got.stride() == tf.stride() and np.array_equal(got.cpu().numpy(), want_f)
  assert np.array_equal(edt.medial_axis(np.asfortranarray(labels), w, True), want_f)
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    got, dist = edt.medial_axis(torch.from_numpy(labels).cuda(), w, True, return_distance=True)
  side.synchronize()
  assert np.array_equal(got.cpu().numpy(), want) and pc.same_bits(dist.cpu().numpy(), want_dist)
  floats = torch.from_numpy(np.where(labels == 1, -0.0, labels).astype(np.float32)).cuda()
  assert np.array_equal(edt.medial_axis(floats, w).cpu().numpy(),
                        mac.restate(np.where(labels == 1, 0, labels), w)[0])
  stack = torch.from_numpy(labels[:5]).cuda()
  got = edt.medial_axis(stack, w[1:], stacked=True)
  assert np.array_equal(got.cpu().numpy(), np.stack([edt.medial_axis(v, w[1:]) for v in labels[:5]]))
  empty = edt.medial_axis(torch.zeros((0, 3), dtype=torch.uint8, device="cuda"), return_distance=True)
  assert empty[0].is_cuda and tuple(empty[0].shape) == (0, 3) and tuple(empty[1].shape) == (0, 3)
  # the C ABI without distances on the caller's stream, a host mask from device labels
  lib = edt._lib()
  mask = np.full(labels.size, 9, np.uint8)
  assert lib.edtb200_medial_axis(t.data_ptr(), 4, 3, 19, 17, 12, 1, 2.0, 1.0, 1.0, 1, 4, mask.ctypes.data, None, 0,
                                 None) == 0
  assert np.array_equal(mask.reshape(labels.shape).astype(bool), want) and mask.max() == 1


def test_the_long_line_tiers(edt):
  rng = np.random.default_rng(11)
  line = (rng.random(23200) < 0.97).astype(np.uint8)                  # past 23170: the brute-force tier
  line[5000:9000] = 2
  for border in (False, True):
    _check(edt, line, (1.0,), border)
  for shape in ((3, 1500), (1100, 4)):                                  # rows of 1025 to 23170: the long-line hull
    labels = mac.balls(rng, shape, 12, 200.0, np.uint16)
    for border in (False, True):
      _check(edt, labels, (1.0, 2.0), border)
    _check(edt, labels, (0.6, 1.1), True, exact=False)


@pytest.mark.parametrize("kind", ["voronoi", "balls"])
def test_at_256_cubed(edt, kind):
  rng = np.random.default_rng(256)
  shape = (256, 256, 256)
  if kind == "voronoi":
    labels = mac.voronoi(rng, shape, 200, np.uint32)
  else:
    labels = mac.balls(rng, shape, 64, 40.0, np.uint8)
  import torch
  t = torch.from_numpy(labels).cuda()
  medial, dist = edt.medial_axis(t, return_distance=True)
  d2 = edt.edtsq(t)
  v, idx = edt.parabolic_dilate(d2, return_indices=True)
  comp = torch.zeros(shape, dtype=torch.bool, device="cuda")
  fg = t != 0
  comp[tuple(i[fg].long() for i in idx)] = True
  assert torch.equal(medial, comp)
  assert torch.equal(dist.view(torch.int32), edt.edt(t).view(torch.int32))
  rec = edt.parabolic_dilate(torch.where(medial, d2, torch.tensor(-float("inf"), device="cuda")))
  assert torch.equal(rec > 0, fg)
  assert torch.equal(rec[fg], v[fg])
  assert 0 < int(medial.sum()) < int(fg.sum())
