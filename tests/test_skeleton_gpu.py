"""GPU tests: skeletonize equals the restatement in skeleton_cases.py byte for byte -- every label width and
bool, both memory orders, 2-D and 3-D, both borders, anisotropic weights, empty and one-label volumes,
stacks against per-volume calls, device input on a side stream, return_distance against edt() bit for bit.
At 256^3 (Voronoi cells and balls) every label keeps its topology invariants and the result is thin, and
past 2^32 voxels small restated cases at even offsets of a uint8 volume come back unchanged."""
import numpy as np
import pytest

import parabolic_cases as pc
import skeleton_cases as skc

pytestmark = pytest.mark.gpu

SHAPES = {2: (29, 37), 3: (11, 14, 17)}
WEIGHTS = {2: [(1.0, 1.0), (2.0, 1.0), (1.3, 0.45)], 3: [(1.0, 1.0, 1.0), (1.0, 2.0, 3.0), (4.0, 4.0, 40.0),
                                                         (0.9, 1.7, 2.3)]}


def _check(edt, labels, w, border, order="C", stacked=False):
  skel, dist = edt.skeletonize(labels, w, border, return_distance=True, stacked=stacked)
  assert isinstance(skel, np.ndarray) and skel.dtype == np.bool_ and skel.shape == labels.shape
  assert skel.flags.f_contiguous if order == "F" else skel.flags.c_contiguous
  assert np.array_equal(edt.skeletonize(labels, w, border, stacked=stacked), skel)
  want_dist = edt.edt(labels, w, border, stacked=True) if stacked else edt.edt(labels, w, border)
  assert pc.same_bits(dist, want_dist)
  want = skc.restate(labels, w, border, order, stacked)
  assert np.array_equal(skel, want), (labels.shape, w, border, order, int((skel != want).sum()))
  return skel


@pytest.mark.parametrize("dtype", [np.bool_, np.uint8, np.int8, np.uint16, np.int16, np.uint32, np.int32,
                                   np.uint64, np.int64])
def test_every_label_width(edt, dtype):
  rng = np.random.default_rng(np.dtype(dtype).num)
  for kind in skc.KINDS:
    base = skc.seeded(rng, kind, (11, 14, 16), np.uint16)
    if dtype == np.bool_:
      labels = base != 0
    elif np.dtype(dtype).kind == "i":
      labels = ((base.astype(np.int64) - 2) * (base != 0)).astype(dtype)          # negative labels too
    else:
      labels = (base.astype(np.uint64) * (np.iinfo(dtype).max // 7)).astype(dtype)
    for border in (False, True):
      _check(edt, labels, (1.0, 2.0, 1.0), border)


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("nd", [2, 3])
@pytest.mark.parametrize("border", [False, True])
def test_orders_dims_borders_and_weights(edt, order, nd, border):
  rng = np.random.default_rng(nd + 7 * border)
  for kind in skc.KINDS + ("noise",):
    labels = (rng.integers(0, 3, SHAPES[nd]).astype(np.uint32) if kind == "noise"
              else skc.seeded(rng, kind, SHAPES[nd], np.uint32))
    labels = np.asfortranarray(labels) if order == "F" else np.ascontiguousarray(labels)
    for w in WEIGHTS[nd]:
      _check(edt, labels, w, border, order)


def test_empty_one_label_and_unlabelled_volumes(edt):
  for shape in ((0, 3), (3, 0, 2), (0, 4, 4)):
    skel, dist = edt.skeletonize(np.zeros(shape, np.uint16), return_distance=True)
    assert skel.shape == shape and dist.shape == shape and skel.dtype == np.bool_
  for shape in ((9, 7), (4, 6, 5), (1, 1), (1, 1, 1)):
    for border in (False, True):
      _check(edt, np.full(shape, 5, np.uint8), None, border)
      _check(edt, np.zeros(shape, np.int32), None, border)
  # without a border a one-label volume is all R = +inf: the final round alone thins it
  assert edt.skeletonize(np.full((5, 5, 5), 1, np.uint8)).sum() >= 1


@pytest.mark.parametrize("order", ["C", "F"])
def test_stacks_are_the_per_volume_calls(edt, order):
  rng = np.random.default_rng(4)
  for shape, w in (((4, 13, 9), (2.0, 1.0)), ((3, 7, 6, 5), (1.0, 1.0, 2.0)), ((6, 8, 8), (0.8, 1.3)),
                   ((2, 5, 9, 12), (4.0, 4.0, 40.0))):
    vols = [skc.seeded(rng, skc.KINDS[i % 4], shape[1:], np.uint8) for i in range(shape[0])]
    vols[1][...] = 0                                                       # no labels
    vols[-1][...] = 3 if shape[0] > 2 else vols[-1]                        # one label
    labels = np.stack(vols) if order == "C" else np.asfortranarray(np.stack([v.T for v in vols]).T)
    axis = 0 if order == "C" else labels.ndim - 1
    vol = (lambda i: np.asfortranarray(np.take(labels, i, axis))) if order == "F" else (lambda i: labels[i])
    for border in (False, True):
      got = _check(edt, labels, w, border, order, stacked=True)
      each = [edt.skeletonize(vol(i), w, border) for i in range(labels.shape[axis])]
      assert np.array_equal(got, np.stack(each, axis))
      assert not np.take(got, 1, axis).any()


def test_the_worked_examples(edt):
  cube = np.zeros((5, 5, 5), np.uint8)
  cube[1:4, 1:4, 1:4] = 1
  assert np.argwhere(edt.skeletonize(cube)).tolist() == [[2, 2, 2]]
  box = np.zeros((6, 8, 14), np.uint8)
  box[1:5, 1:7, 1:13] = 1
  assert np.argwhere(edt.skeletonize(box)).tolist() == [[3, 4, x] for x in range(4, 11)]
  line = np.zeros((5, 9), np.uint8)
  line[2, 1:8] = 1
  assert np.array_equal(edt.skeletonize(line), line != 0)
  yy, xx = np.indices((15, 15))
  assert np.argwhere(edt.skeletonize((yy - 7) ** 2 + (xx - 7) ** 2 <= 36)).tolist() == [[7, 7]]


def test_device_residency_and_a_side_stream(edt):
  import torch
  rng = np.random.default_rng(9)
  labels = skc.seeded(rng, "voronoi", (12, 17, 19), np.int32)
  w = (1.0, 1.0, 2.0)
  want, want_dist = edt.skeletonize(labels, w, True, return_distance=True)
  assert np.array_equal(want, skc.restate(labels, w, True))
  t = torch.from_numpy(labels).cuda()
  got, dist = edt.skeletonize(t, w, True, return_distance=True)
  assert got.is_cuda and got.dtype == torch.bool and dist.is_cuda and dist.dtype == torch.float32
  assert np.array_equal(got.cpu().numpy(), want) and pc.same_bits(dist.cpu().numpy(), want_dist)
  # an F-ordered device view: x is its first axis, as for a host F array
  tf = torch.from_numpy(np.asfortranarray(labels)).cuda().permute(2, 1, 0).contiguous().permute(2, 1, 0)
  got = edt.skeletonize(tf, w, True)
  want_f = skc.restate(np.asfortranarray(labels), w, True, order="F")
  assert got.stride() == tf.stride() and np.array_equal(got.cpu().numpy(), want_f)
  assert np.array_equal(edt.skeletonize(np.asfortranarray(labels), w, True), want_f)
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    src = torch.from_numpy(labels).cuda()
    got, dist = edt.skeletonize(src, w, True, return_distance=True)
  side.synchronize()
  assert np.array_equal(got.cpu().numpy(), want) and pc.same_bits(dist.cpu().numpy(), want_dist)
  stack = torch.from_numpy(labels[:5]).cuda()
  got = edt.skeletonize(stack, w[1:], stacked=True)
  assert np.array_equal(got.cpu().numpy(), np.stack([edt.skeletonize(v, w[1:]) for v in labels[:5]]))
  empty = edt.skeletonize(torch.zeros((0, 3), dtype=torch.uint8, device="cuda"), return_distance=True)
  assert empty[0].is_cuda and tuple(empty[0].shape) == (0, 3) and tuple(empty[1].shape) == (0, 3)
  # the C ABI without distances: a host skeleton from device labels
  lib = edt._lib()
  mask = np.full(labels.size, 9, np.uint8)
  assert lib.edtb200_skeletonize(t.data_ptr(), 4, 3, 19, 17, 12, 1, 2.0, 1.0, 1.0, 1, 4, mask.ctypes.data, None, 0,
                                 None) == 0
  assert np.array_equal(mask.reshape(labels.shape).astype(bool), want) and mask.max() == 1


@pytest.mark.parametrize("kind", ["voronoi", "balls"])
def test_at_256_cubed_every_label_keeps_its_topology_and_the_result_is_thin(edt, kind):
  rng = np.random.default_rng(256)
  shape = (256, 256, 256)
  labels = skc.voronoi(rng, shape, 200, np.uint32) if kind == "voronoi" else skc.balls(rng, shape, 64, 40.0, np.uint8)
  for w, border in (((1.0, 1.0, 1.0), False), ((4.0, 4.0, 40.0), True)):
    skel = edt.skeletonize(labels, w, border)
    assert not (skel & (labels == 0)).any()
    assert skc.topology_kept(labels, skel) == []
    assert skc.not_thin(labels, skel) == 0
    assert 0 < int(skel.sum()) < int((labels != 0).sum())


def test_past_2_to_the_32_voxels(edt):
  """Restated cases at even offsets of a uint8 volume of more than 2^32 voxels: each tile's skeleton is its
  own (a tile keeps a background margin, so its R and its neighbourhoods are those of the tile alone), and
  nothing else is marked."""
  import torch
  shape = (1044, 2048, 2048)
  need = 14 * int(np.prod(shape)) + (6 << 30)
  free = torch.cuda.mem_get_info()[0]
  if free < need:
    pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 1e9, free / 1e9))
  rng = np.random.default_rng(32)
  tiles = []
  for kind in ("voronoi", "balls", "touching"):
    t = np.zeros((18, 20, 22), np.uint8)
    t[1:-1, 1:-1, 1:-1] = skc.seeded(rng, kind, (16, 18, 20), np.uint8)
    tiles.append((t, skc.restate(t, (1.0, 2.0, 1.0))))
  at = [(0, 0, 0), (512, 1000, 1000), (1024, 2026, 2024), (1026, 0, 2024), (600, 2026, 0)]
  vol = torch.zeros(shape, dtype=torch.uint8, device="cuda")
  for n, (z, y, x) in enumerate(at):
    t = tiles[n % len(tiles)][0]
    vol[z:z + t.shape[0], y:y + t.shape[1], x:x + t.shape[2]] = torch.from_numpy(t).cuda()
  assert (at[2][0] * shape[1] + at[2][1]) * shape[2] > 1 << 32
  skel = edt.skeletonize(vol, (1.0, 2.0, 1.0))
  del vol
  total = 0
  for n, (z, y, x) in enumerate(at):
    t, want = tiles[n % len(tiles)]
    got = skel[z:z + t.shape[0], y:y + t.shape[1], x:x + t.shape[2]].cpu().numpy()
    assert np.array_equal(got, want), (n, int((got != want).sum()))
    total += int(want.sum())
  assert int(skel.sum()) == total
