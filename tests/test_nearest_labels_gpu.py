"""GPU tests: nearest_labels equals the per-pass restatement in nearest_labels_cases.py bit for bit, values and
labels, for k = 1..4, every label width and the bool and signed dtypes (where the unsigned tie order shows),
1-D to 3-D volumes in C and F order, axis lengths at the edges of the tiles and windows, both later-pass
variants (staged and global), label-dense windows, equidistant labels, fewer labels than k, weights whose
rounding merges candidates or whose square overflows, stacks, device input and a side stream; and at scale
a 256^3 Voronoi volume of 200 cells against every cell's parabolic_erode on the GPU."""
import ctypes

import numpy as np
import pytest

import nearest_labels_cases as nc

pytestmark = pytest.mark.gpu
DTYPES = [np.uint8, np.uint16, np.uint32, np.uint64, np.bool_, np.int8, np.int16, np.int32, np.int64]
SIZES = [1, 31, 32, 33, 63, 64, 65, 1100]


def _check(edt, labels, d, w=None, k=2, order="C", stacked=False, squared=True):
  dist, near = edt.nearest_labels(labels, d, w, k=k, squared=squared, stacked=stacked)
  want_d, want_l = nc.per_pass(labels, d, w, k, order=order, stacked=stacked, squared=squared)
  assert isinstance(dist, np.ndarray) and dist.dtype == np.float32 and dist.shape == (k,) + labels.shape
  assert near.dtype == labels.dtype and near.shape == (k,) + labels.shape
  for q in range(k):
    assert dist[q].flags.f_contiguous if order == "F" and labels.ndim > 1 else dist[q].flags.c_contiguous
  bad_d = np.argwhere(np.any(np.ascontiguousarray(dist).view(np.uint32) != want_d.view(np.uint32), axis=0))
  bad_l = np.argwhere(np.any(np.ascontiguousarray(near) != want_l, axis=0))
  where = lambda b: [(tuple(x), dist[(slice(None),) + tuple(x)], near[(slice(None),) + tuple(x)],
                      want_d[(slice(None),) + tuple(x)], want_l[(slice(None),) + tuple(x)]) for x in b[:3]]
  assert len(bad_d) == 0, (labels.shape, d, w, k, len(bad_d), where(bad_d))
  assert len(bad_l) == 0, (labels.shape, d, w, k, len(bad_l), where(bad_l))
  return dist, near


def _plan(edt, shape_xyz, w_xyz, d, k, label_bytes):
  radius = (ctypes.c_int64 * 3)()
  variant = (ctypes.c_int * 3)()
  sx, sy, sz = (list(shape_xyz) + [1, 1])[:3]
  wx, wy, wz = (list(w_xyz) + [1.0, 1.0])[:3]
  rc = edt._lib().edtb200_nearest_labels_plan(len(shape_xyz), sx, sy, sz, wx, wy, wz, d, k, label_bytes, radius,
                                              variant)
  assert rc == 0
  return list(radius), list(variant)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda t: np.dtype(t).name)
@pytest.mark.parametrize("k", [1, 2, 3, 4])
@pytest.mark.parametrize("family", nc.FAMILIES)
def test_k_width_and_family(edt, dtype, k, family):
  rng = np.random.default_rng(100 * DTYPES.index(dtype) + 10 * k + nc.FAMILIES.index(family))
  _check(edt, nc.volume(family, (9, 13, 17), dtype, rng), 4.5, (1.0, 2.0, 1.0), k)


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("shape", [(200,), (37, 45), (11, 12, 13)], ids=str)
@pytest.mark.parametrize("squared", [True, False])
def test_dims_and_orders(edt, order, shape, squared):
  rng = np.random.default_rng(len(shape))
  for family in ("dense", "seeds", "lattice"):
    lab = np.asarray(nc.volume(family, shape, np.uint32, rng), order=order)
    _check(edt, lab, 5.0, None, 3, order=order, squared=squared)


@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("n", SIZES)
def test_axis_lengths(edt, axis, n):
  rng = np.random.default_rng(100 * n + axis)
  shape = [3, 4, 5]
  shape[axis] = n
  for family, k in (("seeds", 2), ("dense", 4)):
    _check(edt, nc.volume(family, tuple(shape), np.uint16, rng), 6.0, None, k)


@pytest.mark.parametrize("k,dtype,d,want", [(1, np.uint8, 7.0, 1), (2, np.uint32, 40.0, 1), (4, np.uint64, 20.0, 1),
                                            (4, np.uint64, 50.0, 2), (3, np.uint32, 130.0, 2),
                                            (2, np.uint16, 256.0, 1)])
def test_variants(edt, k, dtype, d, want):
  """Each later-pass variant, chosen by the plan, on the Y and Z passes."""
  shape = (24, 90, 40)                   # z, y, x
  radius, variant = _plan(edt, shape[::-1], (1.0, 1.0, 1.0), d, k, np.dtype(dtype).itemsize)
  assert variant == [0, want, want] and radius[1] == radius[2] == int(d)
  rng = np.random.default_rng(k)
  _check(edt, nc.volume("seeds", shape, dtype, rng), d, None, k)
  lab = np.zeros(shape, dtype)
  lab[rng.integers(0, 24, 6), rng.integers(0, 90, 6), rng.integers(0, 40, 6)] = nc._random_labels(6, dtype, rng)
  _check(edt, lab, d, None, k)


def test_global_equals_staged(edt):
  """The same pass on both variants: k = 4 uint64 stages radii up to 43 and reads 44 and beyond from global
  memory; a radius of 43.9 and of 44 agree wherever both windows hold every candidate."""
  assert _plan(edt, (30, 100, 30), (1.0,) * 3, 43.9, 4, 8)[1] == [0, 1, 1]
  assert _plan(edt, (30, 100, 30), (1.0,) * 3, 44.0, 4, 8)[1] == [0, 2, 2]
  rng = np.random.default_rng(5)
  lab = nc.volume("seeds", (30, 100, 30), np.uint64, rng)
  a = _check(edt, lab, 43.9, None, 4)
  b = _check(edt, lab, 44.0, None, 4)
  inside = a[0] <= np.float32(43.9 ** 2)
  assert np.array_equal(a[0][inside], b[0][inside]) and np.array_equal(a[1][inside], b[1][inside])


@pytest.mark.parametrize("w", [(1.0, 1.0, 1.0), (2.0, 1.0, 3.0), (0.7, 1.3, 2.9), (1.1, 0.9, 1.7), (1e20, 1.0, 1.0),
                               (1.0, 1e20, 0.5)], ids=["1", "2-1-3", "frac", "merge", "overflow-z", "overflow-y"])
@pytest.mark.parametrize("family", nc.FAMILIES)
def test_weights(edt, w, family):
  rng = np.random.default_rng(nc.FAMILIES.index(family))
  _check(edt, nc.volume(family, (10, 14, 18), np.int32, rng), 5.5, w, 3)


def test_rounding_merges_candidates(edt):
  """Weights whose squares are not integers: at these distances fl32 merges candidates that differ in
  the reals, so the label at the k-th slot is decided by the per-pass rule only."""
  rng = np.random.default_rng(9)
  w = (0.1, 0.3, 0.7)
  lab = nc.volume("lattice", (12, 16, 20), np.uint32, rng)
  dist, near = _check(edt, lab, 4.0, w, 2)
  ref_d, _ = nc.per_label(lab, 4.0, w, 2)
  assert nc.same_bits(np.ascontiguousarray(dist), ref_d)       # the values are exact all the same


def test_more_labels_than_k_and_ties(edt):
  """Every voxel of a 3x3x3 block has 27 distinct labels within reach; equidistant ones tie."""
  lab = np.arange(1, 28, dtype=np.uint16)[::-1].reshape(3, 3, 3).copy()
  lab = np.pad(lab, 2)
  for k in (1, 2, 3, 4):
    _check(edt, lab, 3.0, None, k)
    _check(edt, lab.astype(np.int16) * -1, 3.0, None, k)       # negative labels: unsigned tie order


def test_zero_distance_and_empty(edt):
  rng = np.random.default_rng(2)
  lab = nc.volume("dense", (5, 6, 7), np.uint8, rng)
  dist, near = _check(edt, lab, 0.0, None, 2)
  assert np.array_equal(near[0], lab) and np.all(np.isinf(dist[1]))
  dist, near = edt.nearest_labels(np.zeros((0, 4), np.uint32), 3.0, k=3)
  assert dist.shape == (3, 0, 4) and near.shape == (3, 0, 4)
  _check(edt, np.zeros((6, 7), np.uint32), 3.0, None, 2)      # no site at all


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("vshape", [(50,), (17, 19), (7, 8, 9)], ids=str)
def test_stacks(edt, order, vshape):
  rng = np.random.default_rng(len(vshape))
  vols = [nc.volume("seeds", vshape, np.uint32, rng) for _ in range(5)]
  stack = np.asarray(np.stack(vols) if order == "C" else np.stack(vols, axis=-1), order=order)
  dist, near = _check(edt, stack, 4.0, None, 2, order=order, stacked=True)
  for i, v in enumerate(vols):
    want_d, want_l = nc.per_pass(v, 4.0, None, 2, order=order)
    got_d = dist[:, i] if order == "C" else dist[..., i]
    assert nc.same_bits(np.ascontiguousarray(got_d), want_d)


def test_device_input_and_side_stream(edt):
  import torch
  rng = np.random.default_rng(11)
  lab = nc.volume("dense", (20, 30, 40), np.int32, rng)
  want_d, want_l = nc.per_pass(lab, 5.0, (1.0, 1.5, 2.0), 3, squared=False)
  t = torch.from_numpy(lab).cuda()
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    dist, near = edt.nearest_labels(t, 5.0, (1.0, 1.5, 2.0), k=3)
  side.synchronize()
  assert dist.is_cuda and near.dtype == torch.int32 and dist.shape == (3, 20, 30, 40)
  assert nc.same_bits(dist.cpu().numpy(), want_d) and np.array_equal(near.cpu().numpy(), want_l)
  # an F-ordered tensor: planes in its own memory order
  tf = torch.from_numpy(np.ascontiguousarray(lab.transpose(2, 1, 0))).cuda().permute(2, 1, 0)
  dist, near = edt.nearest_labels(tf, 5.0, (1.0, 1.5, 2.0), k=3)
  assert nc.same_bits(dist.contiguous().cpu().numpy(), want_d)
  assert dist[0].permute(2, 1, 0).is_contiguous()


def test_voronoi_256(edt):
  """256^3, 200 Voronoi cells, integer weights: every voxel's values and labels equal the k least
  (D_M, M) over every cell M, each D_M a parabolic_erode of the cell's indicator on the GPU."""
  import torch
  n, cells, k, d = 256, 200, 2, 6.0
  g = torch.Generator(device="cuda").manual_seed(7)
  seeds = torch.randint(0, n, (cells, 3), device="cuda", generator=g).float()
  ax = torch.arange(n, device="cuda", dtype=torch.float32)
  lab = torch.empty((n, n, n), dtype=torch.int32, device="cuda")
  for z in range(n):
    pts = torch.stack(torch.meshgrid(torch.full((1,), float(z), device="cuda"), ax, ax, indexing="ij"), -1).reshape(-1, 3)
    lab[z] = (torch.cdist(pts, seeds).argmin(1) + 1).reshape(n, n).int()
  dist, near = edt.nearest_labels(lab, d, k=k, squared=True)
  B = float(nc.bound_of(d))
  best_v = torch.full((k, n, n, n), float("inf"), device="cuda")
  best_l = torch.zeros((k, n, n, n), dtype=torch.int64, device="cuda")
  for m in range(1, cells + 1):
    f = torch.where(lab == m, 0.0, float("inf")).float()
    if not bool((lab == m).any()):
      continue
    dm = edt.parabolic_erode(f)
    dm = torch.where(dm <= B, dm, torch.full_like(dm, float("inf")))
    v = torch.cat([best_v, dm[None]])
    l = torch.cat([best_l, torch.where(torch.isinf(dm), 0, m)[None].long()])
    o = torch.sort(l, dim=0, stable=True).indices
    v, l = v.gather(0, o), l.gather(0, o)
    o = torch.sort(v, dim=0, stable=True).indices[:k]
    best_v, best_l = v.gather(0, o), l.gather(0, o)
  assert torch.equal(dist.view(torch.int32), best_v.view(torch.int32))
  assert torch.equal(near.long(), best_l)
  assert torch.equal(near[0], lab) and bool((dist[0] == 0).all())
