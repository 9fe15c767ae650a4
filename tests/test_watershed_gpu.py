"""GPU tests: watershed equals the restatement in watershed_cases.py -- W byte for byte and the level bit for
bit -- over 1-D to 3-D volumes, every connectivity, every label width and no labels, every marker width and
bool, both memory orders, NaN, +-inf and -0.0 altitudes and plateaus, seeds on tile faces, edges and corners,
markers on label 0, repeated marker values, a seed beside a smaller-valued flood, mazes that take hundreds of
rounds and a 256^3 volume; stacks against per-volume calls; device input on a side stream; and a uint8
volume past 2^32 voxels of walled slabs whose answer is known."""
import numpy as np
import pytest

import watershed_cases as wc

pytestmark = pytest.mark.gpu

SHAPES = {1: (300,), 2: (37, 45), 3: (19, 21, 26)}


def _same_level(got, want):
  return np.array_equal(np.asarray(got).view(np.uint32), np.asarray(want).view(np.uint32))


def _check(edt, image, markers, labels=None, connectivity=1, order="C", want=None):
  W, L = edt.watershed(image, markers, labels, connectivity=connectivity, return_level=True)
  m = np.asarray(markers)
  assert isinstance(W, np.ndarray) and W.dtype == wc.out_dtype(m) and W.shape == m.shape
  assert L.dtype == np.float32 and L.shape == m.shape
  assert W.flags.f_contiguous if order == "F" else W.flags.c_contiguous
  want_w, want_l = want if want is not None else wc.restate(image, markers, labels, connectivity, order)
  assert np.array_equal(W, want_w), (m.shape, connectivity, order, int((W != want_w).sum()))
  assert _same_level(L, want_l), (m.shape, connectivity, order, int((L.view(np.uint32) != want_l.view(np.uint32)).sum()))
  assert np.array_equal(edt.watershed(image, markers, labels, connectivity=connectivity), W)
  return W, L


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("nd", [1, 2, 3])
def test_random_volumes_orders_dims_and_connectivities(edt, order, nd):
  rng = np.random.default_rng(nd * 10 + (order == "F"))
  for conn in range(1, nd + 1):
    for levels in (None, 4):
      img, mk, lab = wc.random_case(rng, SHAPES[nd], nlabels=3, levels=levels, block=2 if nd == 3 else 3)
      if order == "F":
        img, mk, lab = np.asfortranarray(img), np.asfortranarray(mk), np.asfortranarray(lab)
      _check(edt, img, mk, lab, conn, order)
      _check(edt, img, mk, None, conn, order)


@pytest.mark.parametrize("dtype", [None, np.bool_, np.uint8, np.int8, np.uint16, np.int16, np.uint32, np.int32,
                                   np.uint64, np.int64])
def test_every_label_width(edt, dtype):
  rng = np.random.default_rng(3 if dtype is None else np.dtype(dtype).num)
  img, mk, base = wc.random_case(rng, (13, 17, 18), nlabels=4, levels=6)
  if dtype is None:
    labels = None
  elif dtype == np.bool_:
    labels = base != 0
  elif np.dtype(dtype).kind == "i":
    labels = ((base.astype(np.int64) - 2) * (base != 0)).astype(dtype)          # negative labels too
  else:
    labels = (base.astype(np.uint64) * (np.iinfo(dtype).max // 7)).astype(dtype)
  for conn in (1, 3):
    _check(edt, img, mk, labels, conn)


@pytest.mark.parametrize("dtype", [np.bool_, np.uint8, np.int8, np.uint16, np.int16, np.uint32, np.int32, np.uint64,
                                   np.int64])
def test_every_marker_width(edt, dtype):
  """Markers compared as unsigned integers of their width: negative values and the all-ones value sort last,
  and the all-ones value survives as itself."""
  rng = np.random.default_rng(11)
  img, _, lab = wc.random_case(rng, (12, 30, 31), nlabels=2, levels=5)
  pick = rng.random(lab.shape) < 0.01
  if dtype == np.bool_:
    mk = pick
  else:
    info = np.iinfo(dtype)
    vals = np.array([1, 2, 7, info.max] + ([-1, info.min] if info.min < 0 else [info.max - 1, 3]), dtype=dtype)
    mk = np.where(pick, vals[rng.integers(0, vals.size, lab.shape)], dtype(0)).astype(dtype)
    mk[0, 0, 0], mk[-1, -1, -1] = vals[4] if info.min < 0 else vals[3], 1
  for conn in (1, 2):
    W, _ = _check(edt, img, mk, lab, conn)
  if dtype != np.bool_:
    assert np.isin(W, np.unique(mk)).all()


def test_special_altitudes_and_plateaus(edt):
  rng = np.random.default_rng(7)
  img, mk, lab = wc.random_case(rng, (15, 22, 20), nlabels=2, levels=3)
  special = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0], np.float32)
  where = rng.random(img.shape) < 0.15
  img = np.where(where, special[rng.integers(0, special.size, img.shape)], img).astype(np.float32)
  mk[0, 0, :] = 2                                  # seeds of every altitude, including NaN and +inf
  img[0, 0, :5] = special
  for conn in (1, 2, 3):
    W, L = _check(edt, img, mk, lab, conn)
  assert not np.isnan(L).any() and not (np.signbit(L) & (L == 0)).any()
  # float64 and integer images are converted to float32 once
  _check(edt, img.astype(np.float64), mk, lab, 2, want=wc.restate(img, mk, lab, 2))
  ints = rng.integers(-3, 4, img.shape).astype(np.int16)
  _check(edt, ints, mk, lab, 1, want=wc.restate(ints.astype(np.float32), mk, lab, 1))
  # a constant image: every component takes its least marker; an image of +inf: the same
  for value in (0.0, np.inf, np.nan):
    flat = np.full(img.shape, value, np.float32)
    W, L = _check(edt, flat, mk, lab, 1)


@pytest.mark.parametrize("name,img,mk,lab,conn", wc.seeded_at_tile_borders(),
                         ids=[c[0] for c in wc.seeded_at_tile_borders()])
def test_seeds_on_tile_borders_reach_both_sides(edt, name, img, mk, lab, conn):
  """A seed on a tile's face, edge or corner that is its structure's only contact with the tiles beyond it:
  both phases reach across."""
  W, L = _check(edt, img, mk, lab, conn)
  assert (W[lab != 0] == mk.max()).all()
  _check(edt, np.asfortranarray(img), np.asfortranarray(mk), np.asfortranarray(lab), conn, "F")
  _check(edt, -img, mk, lab, conn)


def test_markers_on_label_0_repeats_and_a_seed_beside_a_smaller_flood(edt):
  lab = np.zeros((20, 22, 24), np.uint16)
  lab[2:9, 2:20, 2:22] = 1
  lab[11:18, 2:20, 2:22] = 1             # the same label, cut off: no seed reaches it
  lab[:, :, 23] = 2
  img = np.zeros(lab.shape, np.float32)
  mk = np.zeros(lab.shape, np.uint32)
  mk[5, 10, 10] = 6
  mk[5, 10, 11] = 1                      # a seed beside a smaller-valued flood on a plateau: keeps its 6
  mk[3, 3, 3] = 1                        # a repeated marker value
  mk[10, 10, 10] = 3                     # on label 0: ignored
  mk[0, 0, 0] = 1
  W, L = _check(edt, img, mk, lab, 1)
  assert W[5, 10, 10] == 6 and (W[11:18] == 0).all() and (W[lab == 0] == 0).all() and (W[:, :, 23] == 0).all()
  assert np.isinf(L[11:18]).all() and np.isinf(L[lab == 0]).all()
  assert (W[2:9, 2:20, 2:22] == 1).sum() == 7 * 18 * 20 - 1


def test_mazes_take_many_rounds(edt):
  """A serpentine maze whose flood runs through hundreds of tile crossings, on noise and on a plateau."""
  rng = np.random.default_rng(5)
  maze = np.ascontiguousarray(wc.serpentine((64, 97, 9), period=4).T)       # (z, y, x)
  mk = np.zeros(maze.shape, np.uint8)
  mk[0, 0, 0] = 3
  mk[8, 96, 63] = 2
  for img in (rng.random(maze.shape).astype(np.float32), np.zeros(maze.shape, np.float32)):
    _check(edt, img, mk, maze, 1)
  spiral_img = rng.random((70, 70)).astype(np.float32)
  mk2 = np.zeros((70, 70), np.int64)
  mk2[0, 0], mk2[35, 35] = 5, 9
  lab2 = np.ascontiguousarray(wc.serpentine((70, 70), period=3).T)
  _check(edt, spiral_img, mk2, lab2, 2)


@pytest.mark.parametrize("order", ["C", "F"])
def test_stacks_are_the_per_volume_calls(edt, order):
  rng = np.random.default_rng(4)
  for shape, conn in (((4, 21, 19), 2), ((3, 7, 10, 9), 3), ((5, 70), 1), ((2, 9, 11, 12), 1)):
    cases = [wc.random_case(rng, shape[1:], levels=4) for _ in range(shape[0])]
    cases[1][1][...] = 0                                                      # no markers
    if order == "C":
      img, mk, lab = (np.stack([c[k] for c in cases]) for k in range(3))
      axis = 0
    else:
      img, mk, lab = (np.asfortranarray(np.stack([c[k].T for c in cases]).T) for k in range(3))
      axis = lab.ndim - 1
    W, L = edt.watershed(img, mk, lab, connectivity=conn, stacked=True, return_level=True)
    vol = (lambda a, i: np.asfortranarray(np.take(a, i, axis))) if order == "F" else (lambda a, i: a[i])
    for i in range(lab.shape[axis]):
      w1, l1 = _check(edt, vol(img, i), vol(mk, i), vol(lab, i), conn, order)
      assert np.array_equal(np.take(W, i, axis), w1) and _same_level(np.take(L, i, axis), l1)
    assert (np.take(W, 1, axis) == 0).all()


def test_device_residency_and_a_side_stream(edt):
  import torch
  rng = np.random.default_rng(9)
  img, mk, lab = wc.random_case(rng, (18, 23, 29), nlabels=3, levels=5)
  lab = lab.astype(np.int32)
  want_w, want_l = wc.restate(img, mk, lab, 2)
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    ti, tm, tl = (torch.from_numpy(a).cuda() for a in (img, mk.astype(np.int16), lab))
    W, L = edt.watershed(ti, tm, tl, connectivity=2, return_level=True)
  side.synchronize()
  assert W.is_cuda and W.dtype == torch.int16 and L.is_cuda and L.dtype == torch.float32
  assert np.array_equal(W.cpu().numpy().view(np.uint16), want_w) and _same_level(L.cpu().numpy(), want_l)
  # host markers and image are moved to the labels' device
  got = edt.watershed(img, mk, tl, connectivity=2)
  assert got.is_cuda and got.dtype == torch.uint16 and np.array_equal(got.cpu().numpy(), want_w)
  # an F-ordered device view: x is its first axis, as for a host F array
  f = lambda a: torch.from_numpy(np.asfortranarray(a)).cuda().permute(2, 1, 0).contiguous().permute(2, 1, 0)
  W, L = edt.watershed(f(img), f(mk), f(lab), connectivity=2, return_level=True)
  want_fw, want_fl = wc.restate(np.asfortranarray(img), np.asfortranarray(mk), np.asfortranarray(lab), 2, "F")
  assert W.stride() == f(lab).stride() and np.array_equal(W.cpu().numpy(), want_fw)
  assert _same_level(L.cpu().numpy(), want_fl)
  # no labels, the image as the volume; bool markers give uint8
  W = edt.watershed(ti, torch.from_numpy(mk != 0).cuda(), connectivity=3)
  assert W.dtype == torch.uint8 and np.array_equal(W.cpu().numpy(), wc.restate(img, mk != 0, None, 3)[0])
  stack = edt.watershed(ti[:5], tm[:5], tl[:5], stacked=True)
  each = np.stack([edt.watershed(img[i], mk[i].astype(np.int16), lab[i]) for i in range(5)])
  assert np.array_equal(stack.cpu().numpy(), each)
  empty = edt.watershed(torch.zeros((0, 3), device="cuda"), torch.zeros((0, 3), dtype=torch.int32, device="cuda"),
                        return_level=True)
  assert empty[0].is_cuda and tuple(empty[0].shape) == (0, 3) and empty[0].dtype == torch.int32


def test_two_touching_balls_split_at_the_neck(edt):
  mask, mk = wc.balls((40, 40, 60), [(20, 20, 18), (20, 20, 36)], [12, 7])
  W = edt.watershed(wc.minus_edt(mask), mk, mask)
  want, _ = wc.restate(wc.minus_edt(mask), mk, mask)
  assert np.array_equal(W, want)
  # the balls span x = 6 .. 43 on their axis and meet at x = 29 .. 30
  assert (W[20, 20, 6:31] == 1).all() and (W[20, 20, 31:44] == 2).all()


def test_a_256_cube(edt):
  """64 balls of -edt in a 256^3 volume, one marker each, against the numpy-frontier restatement."""
  import scipy.ndimage
  rng = np.random.default_rng(256)
  centres = rng.integers(20, 236, (64, 3))
  radii = rng.integers(10, 28, 64)
  mask, mk = wc.balls((256, 256, 256), centres, radii)
  img = -scipy.ndimage.distance_transform_edt(mask).astype(np.float32)
  for conn in (1, 3):
    _check(edt, img, mk, mask, conn, want=wc.flood(img, mk, mask, conn))


def test_past_2_to_the_32_voxels(edt):
  """A uint8-marker volume of more than 2^32 voxels with no labels: slabs of altitude 0 between walls of
  altitude 1 on every 64th z plane, one marker per slab.  Each slab takes its own marker, and each wall the
  smaller of the two it is reached from at level 1."""
  import torch
  shape = (1024, 2048, 2049)                                # (z, y, x): 4.30e9 voxels
  total = int(np.prod(shape))
  assert total > 1 << 32
  # markers, image, L, W and the result
  need = 14 * total + (2 << 30)
  free = torch.cuda.mem_get_info()[0]
  if free < need:
    pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 1e9, free / 1e9))
  z = np.arange(shape[0])
  want = np.where(z % 64 == 0, z // 64, z // 64 + 1)
  want[0] = 1
  try:
    img = torch.zeros(shape, dtype=torch.float32, device="cuda")
    img[64::64] = 1.0
    mk = torch.zeros(shape, dtype=torch.uint8, device="cuda")
    for k in range(shape[0] // 64):
      mk[64 * k + 1, (k * 131) % shape[1], shape[2] - 1 - k] = k + 1
    W = edt.watershed(img, mk)
    del img, mk
    want_t = torch.from_numpy(want.astype(np.uint8)).cuda()
    for z0 in range(0, shape[0], 64):
      assert not bool((W[z0:z0 + 64] != want_t[z0:z0 + 64, None, None]).any()), z0
  finally:
    # give the 60 GB back, so that the tests after this one see the card's memory free
    img = mk = W = None
    torch.cuda.synchronize()
    edt.release()
    torch.cuda.empty_cache()
