"""GPU tests: geodesic_distance equals the restatement in geodesic_cases.py bit for bit -- the float32
distances and every index plane -- over 1-D to 3-D volumes, every label width and bool, bool and integer
seeds, both memory orders, non-integer and rounding-stressing weights, corridors that cross tiles only
through an edge or a corner, mazes that take many rounds, components without a seed, seeds on background and
sizes that are not multiples of the tile; stacks against per-volume calls; device input on a side stream;
and a uint8 volume past 2^31 voxels whose corridor's answer is known in closed form."""
import numpy as np
import pytest

import geodesic_cases as gc

pytestmark = pytest.mark.gpu

WEIGHTS = {1: [(1.0,), (0.7,)], 2: [(1.0, 1.0), (1.0, 1.33355), (40.0, 4.0)],
           3: [(1.0, 1.0, 1.0), (1.7, 1.0, 3.1), (4.0, 4.0, 40.0), (1.33355, 1.0, 2.0 ** -26)]}
SHAPES = {1: (300,), 2: (37, 45), 3: (19, 21, 26)}


def _same(got, want):
  return np.array_equal(np.asarray(got).view(np.uint32), np.asarray(want).view(np.uint32))


def _check(edt, labels, seeds, w, order="C"):
  dist, idx = edt.geodesic_distance(labels, seeds, w, return_indices=True)
  assert isinstance(dist, np.ndarray) and dist.dtype == np.float32 and dist.shape == labels.shape
  assert dist.flags.f_contiguous if order == "F" else dist.flags.c_contiguous
  assert idx.dtype == np.int32 and idx.shape == (labels.ndim,) + labels.shape
  want, S = gc.restate(labels, seeds, w, order)
  assert _same(dist, want), (labels.shape, w, order, int((dist != want).sum()))
  planes = gc.index_planes(S, labels.shape, order)
  assert np.array_equal(idx, planes), (labels.shape, w, order, int((idx != planes).sum()))
  assert _same(edt.geodesic_distance(labels, seeds, w), dist)
  return dist, idx


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("nd", [1, 2, 3])
def test_random_labels_orders_dims_and_weights(edt, order, nd):
  rng = np.random.default_rng(nd * 10 + (order == "F"))
  for w in WEIGHTS[nd]:
    labels = gc.random_labels(rng, SHAPES[nd], nlabels=3, block=2 if nd == 3 else 3)
    seeds = gc.random_seeds(rng, SHAPES[nd], 0.01)
    if order == "F":
      labels, seeds = np.asfortranarray(labels), np.asfortranarray(seeds)
    _check(edt, labels, seeds, w, order)


@pytest.mark.parametrize("dtype", [np.bool_, np.uint8, np.int8, np.uint16, np.int16, np.uint32, np.int32,
                                   np.uint64, np.int64])
def test_every_label_width(edt, dtype):
  rng = np.random.default_rng(np.dtype(dtype).num)
  base = gc.random_labels(rng, (13, 17, 18), nlabels=4)
  if dtype == np.bool_:
    labels = base != 0
  elif np.dtype(dtype).kind == "i":
    labels = ((base.astype(np.int64) - 2) * (base != 0)).astype(dtype)           # negative labels too
  else:
    labels = (base.astype(np.uint64) * (np.iinfo(dtype).max // 7)).astype(dtype)
  seeds = gc.random_seeds(rng, labels.shape, 0.02)
  _check(edt, labels, seeds, (1.0, 2.0, 1.33355))


@pytest.mark.parametrize("dtype", [np.bool_, np.uint8, np.int16, np.uint32, np.int64])
def test_seed_dtypes(edt, dtype):
  rng = np.random.default_rng(5)
  labels = gc.random_labels(rng, (12, 30, 31), nlabels=2)
  raw = rng.integers(0, 200, labels.shape) * (rng.random(labels.shape) < 0.01)
  seeds = (raw != 0) if dtype == np.bool_ else (raw * (np.iinfo(dtype).max // 300 + 1)).astype(dtype)
  _check(edt, labels, seeds, (1.0, 1.0, 1.7))


def test_components_without_seeds_and_seeds_on_background(edt):
  labels = np.zeros((20, 22, 24), np.uint16)
  labels[2:9, 2:20, 2:22] = 1
  labels[11:18, 2:20, 2:22] = 1          # the same label, cut off: no seed reaches it
  labels[:, :, 23] = 2                   # a label with no seed
  seeds = np.zeros(labels.shape, np.uint8)
  seeds[5, 10, 10] = 1
  seeds[10, 10, 10] = 3                  # on background: ignored
  seeds[0, 0, 0] = 1                     # on background
  dist, idx = _check(edt, labels, seeds, (1.0, 1.0, 1.0))
  assert np.isinf(dist[11:18]).all() and (idx[:, 11:18] == -1).all()
  assert np.isinf(dist[labels == 0]).all() and (idx[:, labels == 0] == -1).all()
  nothing = edt.geodesic_distance(labels, np.zeros(labels.shape, bool))
  assert np.isinf(nothing).all()


@pytest.mark.parametrize("nd,cross", [(1, "corner"), (2, "corner"), (3, "corner"), (3, "edge")])
def test_corridors_that_cross_tiles_through_an_edge_or_a_corner(edt, nd, cross):
  lab_x = gc.corridor_through_corner(nd, cross=cross)
  labels = np.ascontiguousarray(lab_x.T)
  pts = np.argwhere(labels)
  seeds = np.zeros(labels.shape, bool)
  seeds[tuple(pts[pts[:, -1].argmin()])] = True
  dist, _ = _check(edt, labels, seeds, (1.0,) * nd)
  assert np.isfinite(dist[labels != 0]).all()
  _check(edt, np.asfortranarray(lab_x), np.asfortranarray(seeds.T), (1.0,) * nd, "F")
  # offset by a voxel along every axis, so that the crossing falls elsewhere on the tiling
  pad = np.pad(labels, [(1, 0)] * nd)
  _check(edt, pad, np.pad(seeds, [(1, 0)] * nd), (1.3,) * nd)


def test_mazes_take_many_rounds(edt):
  lab = gc.spiral(61)
  seeds = np.zeros(lab.shape, bool)
  seeds[0, 0] = True
  dist, _ = _check(edt, lab, seeds, (1.0, 1.0))
  assert dist[np.isfinite(dist)].max() > 500
  maze = np.ascontiguousarray(gc.serpentine((40, 41, 9), period=4).T)     # (z, y, x)
  seeds = np.zeros(maze.shape, np.uint8)
  seeds[0, 0, 0] = 1
  seeds[4, 40, 39] = 1
  _check(edt, maze, seeds, (1.0, 1.0, 1.0))
  _check(edt, maze, seeds, (1.33355, 1.0, 2.0 ** -26))


@pytest.mark.parametrize("order", ["C", "F"])
def test_stacks_are_the_per_volume_calls(edt, order):
  rng = np.random.default_rng(4)
  for shape, w in (((4, 21, 19), (2.0, 1.0)), ((3, 7, 10, 9), (1.0, 1.0, 2.0)), ((5, 70), (0.7,)),
                   ((2, 9, 11, 12), (4.0, 4.0, 40.0))):
    vols = [gc.random_labels(rng, shape[1:], nlabels=2) for _ in range(shape[0])]
    seeds = [gc.random_seeds(rng, shape[1:], 0.03) for _ in range(shape[0])]
    seeds[1][...] = False                                                  # no seeds
    if order == "C":
      labels, sd = np.stack(vols), np.stack(seeds)
      axis = 0
    else:
      labels = np.asfortranarray(np.stack([v.T for v in vols]).T)
      sd = np.asfortranarray(np.stack([s.T for s in seeds]).T)
      axis = labels.ndim - 1
    dist, idx = edt.geodesic_distance(labels, sd, w, stacked=True, return_indices=True)
    assert idx.shape == (labels.ndim - 1,) + labels.shape
    vol = (lambda a, i: np.asfortranarray(np.take(a, i, axis))) if order == "F" else (lambda a, i: a[i])
    for i in range(labels.shape[axis]):
      d1, i1 = edt.geodesic_distance(vol(labels, i), vol(sd, i), w, return_indices=True)
      assert _same(np.take(dist, i, axis), d1)
      assert np.array_equal(np.take(idx, i, axis + 1), i1)
      want, S = gc.restate(vol(labels, i), vol(sd, i), w, order)
      assert _same(d1, want) and np.array_equal(i1, gc.index_planes(S, want.shape, order))
    assert np.isinf(np.take(dist, 1, axis)).all()


def test_device_residency_and_a_side_stream(edt):
  import torch
  rng = np.random.default_rng(9)
  labels = gc.random_labels(rng, (18, 23, 29), nlabels=3).astype(np.int32)
  seeds = gc.random_seeds(rng, labels.shape, 0.01)
  w = (1.0, 1.33355, 2.0)
  want, want_idx = edt.geodesic_distance(labels, seeds, w, return_indices=True)
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    t = torch.from_numpy(labels).cuda()
    s = torch.from_numpy(seeds).cuda()
    dist, idx = edt.geodesic_distance(t, s, w, return_indices=True)
  side.synchronize()
  assert dist.is_cuda and dist.dtype == torch.float32 and idx.is_cuda and idx.dtype == torch.int32
  assert _same(dist.cpu().numpy(), want) and np.array_equal(idx.cpu().numpy(), want_idx)
  # host seeds are moved to the labels' device
  got = edt.geodesic_distance(t, seeds.astype(np.uint8), w)
  assert _same(got.cpu().numpy(), want)
  # an F-ordered device view: x is its first axis, as for a host F array
  tf = torch.from_numpy(np.asfortranarray(labels)).cuda().permute(2, 1, 0).contiguous().permute(2, 1, 0)
  dist, idx = edt.geodesic_distance(tf, s, w, return_indices=True)
  want_f, want_fidx = edt.geodesic_distance(np.asfortranarray(labels), np.asfortranarray(seeds), w,
                                            return_indices=True)
  wf, S = gc.restate(np.asfortranarray(labels), seeds, w, "F")
  assert _same(want_f, wf) and np.array_equal(want_fidx, gc.index_planes(S, labels.shape, "F"))
  assert dist.stride() == tf.stride() and _same(dist.cpu().numpy(), want_f)
  assert np.array_equal(idx.cpu().numpy(), want_fidx)
  # a host F array with C-ordered seeds: the seeds are read in the labels' order
  assert _same(edt.geodesic_distance(np.asfortranarray(labels), seeds, w), want_f)
  stack = edt.geodesic_distance(t[:5], s[:5], w[1:], stacked=True)
  each = np.stack([edt.geodesic_distance(labels[i], seeds[i], w[1:]) for i in range(5)])
  assert _same(stack.cpu().numpy(), each)
  empty = edt.geodesic_distance(torch.zeros((0, 3), dtype=torch.uint8, device="cuda"),
                                torch.zeros((0, 3), dtype=torch.bool, device="cuda"), return_indices=True)
  assert empty[0].is_cuda and tuple(empty[0].shape) == (0, 3) and tuple(empty[1].shape) == (2, 0, 3)


@pytest.mark.parametrize("name,lab,seeds", gc.seeded_at_tile_borders(), ids=[c[0] for c in gc.seeded_at_tile_borders()])
def test_seeds_on_tile_borders_reach_both_sides(edt, name, lab, seeds):
  """A seed on a tile's face, edge or corner that is its structure's only contact with the tiles beyond it:
  the distances and indices reach across in both phases."""
  dist, idx = _check(edt, lab, seeds, (1.0,) * lab.ndim)
  assert np.isfinite(dist[lab != 0]).all() and (idx[:, lab != 0] >= 0).all()
  _check(edt, np.asfortranarray(lab), np.asfortranarray(seeds), (1.0,) * lab.ndim, "F")
  _check(edt, lab, seeds, (1.33355,) * lab.ndim)


def test_the_docstring_examples(edt):
  labels = np.zeros((3, 9), np.uint8)
  labels[1, 1:8] = 1
  seeds = np.zeros((3, 9), bool)
  seeds[1, 1] = True
  d = edt.geodesic_distance(labels, seeds, (1.0, 0.5))
  assert d[1, 1:8].tolist() == [0, 0.5, 1, 1.5, 2, 2.5, 3] and np.isinf(d[labels == 0]).all()
  labels = np.zeros((5, 5), np.uint8)
  labels[0, :] = 1
  labels[:, 4] = 1
  seeds = np.zeros((5, 5), bool)
  seeds[0, 0] = True
  assert edt.geodesic_distance(labels, seeds)[4, 4] == np.float32(6 + np.sqrt(2))
  # the seed-splitting recipe: two touching discs, one marker each
  yy, xx = np.indices((30, 50))
  mask = (((yy - 15) ** 2 + (xx - 15) ** 2 <= 144) | ((yy - 15) ** 2 + (xx - 34) ** 2 <= 144)).astype(np.uint8)
  markers = np.zeros(mask.shape, np.int32)
  markers[15, 15], markers[15, 34] = 1, 2
  dist, idx = edt.geodesic_distance(mask, markers != 0, return_indices=True)
  split = np.where(idx[0] >= 0, markers[tuple(idx)], 0)
  assert set(np.unique(split[mask != 0])) == {1, 2} and (split[mask == 0] == 0).all()
  assert (split[15, :20][mask[15, :20] != 0] == 1).all() and (split[15, 30:][mask[15, 30:] != 0] == 2).all()


def test_past_2_to_the_31_voxels(edt):
  """A uint8 volume of more than 2^31 voxels, background but for a walled corridor near its end: a straight
  run along x and a diagonal run in the (y, x) plane from one seed, whose distances are known in closed form
  (the float32 step length added in double, step by step), +inf everywhere else, and whose index planes
  hold the seed's coordinates on the corridor and -1 elsewhere."""
  import torch
  shape = (514, 2048, 2049)                                # (z, y, x): 2.16e9 voxels
  total = int(np.prod(shape))
  assert total > 1 << 31
  # labels, seeds, D and S of the call, its distances and three index planes
  need = 34 * total + (2 << 30)
  free = torch.cuda.mem_get_info()[0]
  if free < need:
    pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 1e9, free / 1e9))
  z, y0, x0 = 512, 1000, 3
  vol = torch.zeros(shape, dtype=torch.uint8, device="cuda")
  vol[z, y0, x0:x0 + 2000] = 7                             # along x
  for k in range(1, 40):
    vol[z, y0 + k, x0 + k] = 7                             # a diagonal from the run's first voxel
  seeds = torch.zeros(shape, dtype=torch.uint8, device="cuda")
  seeds[z, y0, x0] = 1
  w = (1.0, 1.5, 0.7)
  assert (z * shape[1] + y0) * shape[2] + x0 > 1 << 31
  dist, idx = edt.geodesic_distance(vol, seeds, w, return_indices=True)
  del vol, seeds
  row = dist[z, y0, x0:x0 + 2000].cpu().numpy()
  wx, wy = float(np.float32(0.7)), float(np.float32(1.5))      # the weights as float32, promoted to double
  acc, want = 0.0, []
  for _ in range(2000):
    want.append(acc)
    acc += wx
  assert _same(row, np.float32(want))
  diag = np.array([float(dist[z, y0 + k, x0 + k]) for k in range(1, 40)], np.float32)
  step = float(np.sqrt(wx * wx + wy * wy))
  acc, want = 0.0, []
  for _ in range(39):
    acc += step
    want.append(acc)
  assert _same(diag, np.float32(want))
  reached = torch.isfinite(dist)
  assert int(reached.sum()) == 2000 + 39
  del dist
  for k, c in enumerate((z, y0, x0)):
    plane = idx[k]
    assert bool((plane[reached] == c).all()), k
    assert int((plane >= 0).sum()) == 2000 + 39 and int((plane == -1).sum()) == total - 2000 - 39, k
