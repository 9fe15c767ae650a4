"""GPU tests: connected_components and extended_maxima equal the restatements in components_cases.py byte for
byte, over every label width and no labels, image dtypes, 1-D to 3-D, both memory orders, every connectivity,
stacks numbered volume by volume, device input on a side stream, components that cross tile faces, edges
and corners only once, a serpentine maze, an all-ones 256^3 volume, label noise, checkerboards, special
image values, h at and either side of a peak's dynamic, the edt -> extended_maxima -> watershed split, and
volumes past 2^31 and 2^32 voxels made of walled slabs whose components are known."""
import numpy as np
import pytest

import components_cases as cc
import watershed_cases as wc

pytestmark = pytest.mark.gpu

SHAPES = {1: (3000,), 2: (70, 45), 3: (19, 37, 26)}


def _check_cc(edt, lab, conn=1, order="C", want=None, how="csgraph"):
  got = edt.connected_components(lab, connectivity=conn)
  assert isinstance(got, np.ndarray) and got.dtype == np.int32 and got.shape == np.shape(lab)
  assert got.flags.f_contiguous if order == "F" else got.flags.c_contiguous
  want = cc.restate_cc(lab, conn, order, how) if want is None else want
  assert np.array_equal(got, want), (np.shape(lab), conn, order, int((got != want).sum()))
  return got


def _check_em(edt, img, h=0.0, lab=None, conn=1, order="C", want=None, recon="relax"):
  got = edt.extended_maxima(img, h, lab, connectivity=conn)
  assert isinstance(got, np.ndarray) and got.dtype == np.int32 and got.shape == np.shape(img)
  assert got.flags.f_contiguous if order == "F" else got.flags.c_contiguous
  want = cc.restate_em(img, h, lab, conn, order, recon) if want is None else want
  assert np.array_equal(got, want), (np.shape(img), h, conn, order, int((got != want).sum()))
  return got


def test_worked_examples(edt):
  a = np.array([[1, 1, 0, 2], [0, 1, 0, 2], [3, 0, 0, 1]], np.uint8)
  assert edt.connected_components(a).tolist() == [[1, 1, 0, 2], [0, 1, 0, 2], [3, 0, 0, 4]]
  d = np.array([[1, 0], [0, 1]], np.uint8)
  assert edt.connected_components(d).tolist() == [[1, 0], [0, 2]]
  assert edt.connected_components(d, connectivity=2).tolist() == [[1, 0], [0, 1]]
  x = np.array([0, 3, 1, 5, 2, 0], np.float32)
  for h, want in ((0.0, [0, 1, 0, 2, 0, 0]), (1.9, [0, 1, 0, 2, 0, 0]), (2.0, [0, 0, 0, 1, 0, 0])):
    assert edt.extended_maxima(x, h).tolist() == want, h
  y = np.array([0, 4, 3.5, 4, 0], np.float32)
  for h, want in ((0.0, [0, 1, 0, 2, 0]), (0.4, [0, 1, 0, 2, 0]), (0.5, [0, 1, 1, 1, 0]), (1.0, [0, 1, 1, 1, 0])):
    assert edt.extended_maxima(y, h).tolist() == want, h


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("nd", [1, 2, 3])
def test_random_volumes_orders_dims_and_connectivities(edt, order, nd):
  rng = np.random.default_rng(nd * 10 + (order == "F"))
  for conn in range(1, nd + 1):
    lab = cc.random_labels(rng, SHAPES[nd], nlabels=3, block=2 if nd == 3 else 3)
    img = cc.random_image(rng, SHAPES[nd], levels=5)
    if order == "F":
      lab, img = np.asfortranarray(lab), np.asfortranarray(img)
    _check_cc(edt, lab, conn, order)
    for h in (0.0, 1.0):
      _check_em(edt, img, h, lab, conn, order)
      _check_em(edt, img, h, None, conn, order)


@pytest.mark.parametrize("dtype", [np.bool_, np.uint8, np.int8, np.uint16, np.int16, np.uint32, np.int32,
                                   np.uint64, np.int64])
def test_every_label_width(edt, dtype):
  rng = np.random.default_rng(np.dtype(dtype).num)
  base = cc.random_labels(rng, (13, 17, 40), nlabels=4)
  if dtype == np.bool_:
    lab = base != 0
  elif np.dtype(dtype).kind == "i":
    lab = ((base.astype(np.int64) - 2) * (base != 0)).astype(dtype)             # negative labels too
  else:
    lab = (base.astype(np.uint64) * (np.iinfo(dtype).max // 7)).astype(dtype)
  img = cc.random_image(rng, lab.shape, levels=4)
  for conn in (1, 3):
    _check_cc(edt, lab, conn)
    _check_em(edt, img, 0.0, lab, conn)
    _check_em(edt, img, 2.0, lab, conn)


@pytest.mark.parametrize("dtype", [np.float64, np.float16, np.int16, np.uint8, np.int64, np.bool_])
def test_image_dtypes_are_converted_to_float32_once(edt, dtype):
  rng = np.random.default_rng(5)
  img = (rng.random((20, 30)) * 6).astype(dtype)
  f32 = img.astype(np.float32)
  for h in (0.0, 1.0):
    _check_em(edt, img, h, want=cc.restate_em(f32, h))


def test_special_image_values(edt):
  rng = np.random.default_rng(7)
  img = cc.random_image(rng, (15, 22, 20), levels=3)
  special = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1e-40, -1e-40, 1e-45], np.float32)
  where = rng.random(img.shape) < 0.2
  img = np.where(where, special[rng.integers(0, special.size, img.shape)], img).astype(np.float32)
  img[0, 0, :special.size] = special
  lab = cc.random_labels(rng, img.shape, nlabels=2)
  for conn in (1, 2, 3):
    for h in (0.0, 1e-45, 0.5, 2.0):
      _check_em(edt, img, h, lab, conn)
  # all NaN and all -inf: no maxima; all +inf: every component of the labels
  for value in (np.nan, -np.inf):
    assert not edt.extended_maxima(np.full((9, 9), value, np.float32)).any()
  flat = np.full(lab.shape, np.inf, np.float32)
  assert np.array_equal(edt.extended_maxima(flat, 1.0, lab), cc.restate_cc(lab))


def test_h_at_and_either_side_of_a_dynamic(edt):
  """A peak of 3 behind a pass of 1.25 on the way to 5: its dynamic is 1.75, exact in float32."""
  x = np.zeros((6, 9, 40), np.float32)
  x[3, 4, 5], x[3, 4, 6:20], x[3, 4, 20] = 3.0, 1.25, 5.0
  for h, n in ((np.nextafter(np.float32(1.75), np.float32(0)), 2), (1.75, 1), (np.nextafter(np.float32(1.75), np.float32(2)), 1)):
    got = _check_em(edt, x, float(h))
    assert got.max() == n, h
  # the same with the peak's value one ulp higher: it survives h = 1.75
  x[3, 4, 5] = np.nextafter(np.float32(3), np.float32(4))
  assert _check_em(edt, x, 1.75).max() == 2


@pytest.mark.parametrize("name,lab,conn", cc.crossing_tiles(), ids=[c[0] for c in cc.crossing_tiles()])
def test_components_that_cross_tiles_once(edt, name, lab, conn):
  got = _check_cc(edt, lab, conn)
  assert got.max() == 1
  img = np.where(lab != 0, 2.0, 0.0).astype(np.float32)
  assert _check_em(edt, img, 0.0, None, conn).max() == 1
  assert _check_em(edt, img, 0.5, lab, conn).max() == 1
  _check_cc(edt, np.asfortranarray(lab), conn, "F")


def test_a_serpentine_maze_and_checkerboards(edt):
  maze = np.ascontiguousarray(wc.serpentine((64, 97, 9), period=4).T)      # (z, y, x)
  got = _check_cc(edt, maze, 1)
  assert got.max() == 1
  ramp = np.cumsum(maze.reshape(-1)).reshape(maze.shape).astype(np.float32)
  _check_em(edt, ramp, 0.0, maze)
  _check_em(edt, ramp, 3.0, maze)
  for nd, shape in ((2, (40, 33)), (3, (12, 14, 17))):
    board = (np.indices(shape).sum(0) % 2).astype(np.uint8)
    for conn in range(1, nd + 1):
      got = _check_cc(edt, board, conn)
      assert got.max() == (1 if conn > 1 else board.sum())
      _check_em(edt, board.astype(np.float32), 0.0, None, conn)


@pytest.mark.parametrize("order", ["C", "F"])
def test_stacks_are_the_per_volume_calls(edt, order):
  rng = np.random.default_rng(4)
  for shape, conn in (((4, 21, 19), 2), ((3, 7, 10, 9), 3), ((5, 70), 1), ((2, 9, 11, 12), 1)):
    labs = [cc.random_labels(rng, shape[1:]) for _ in range(shape[0])]
    imgs = [cc.random_image(rng, shape[1:], levels=4) for _ in range(shape[0])]
    labs[1][...] = 0                                                         # a volume with no components
    if order == "C":
      lab, img, axis = np.stack(labs), np.stack(imgs), 0
    else:
      lab = np.asfortranarray(np.stack([a.T for a in labs]).T)
      img = np.asfortranarray(np.stack([a.T for a in imgs]).T)
      axis = lab.ndim - 1
    got = edt.connected_components(lab, connectivity=conn, stacked=True)
    em = edt.extended_maxima(img, 1.0, lab, connectivity=conn, stacked=True)
    vol = (lambda a, i: np.asfortranarray(np.take(a, i, axis))) if order == "F" else (lambda a, i: a[i])
    for i in range(lab.shape[axis]):
      assert np.array_equal(np.take(got, i, axis), _check_cc(edt, vol(lab, i), conn, order))
      assert np.array_equal(np.take(em, i, axis), _check_em(edt, vol(img, i), 1.0, vol(lab, i), conn, order))
    assert not np.take(got, 1, axis).any()


def test_device_residency_and_a_side_stream(edt):
  import torch
  rng = np.random.default_rng(9)
  lab = cc.random_labels(rng, (18, 23, 29)).astype(np.int32)
  img = cc.random_image(rng, lab.shape, levels=5)
  want_cc = cc.restate_cc(lab, 2)
  want_em = cc.restate_em(img, 1.0, lab, 2)
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    tl, ti = torch.from_numpy(lab).cuda(), torch.from_numpy(img).cuda()
    got = edt.connected_components(tl, connectivity=2)
    em = edt.extended_maxima(ti, 1.0, tl, connectivity=2)
  side.synchronize()
  assert got.is_cuda and got.dtype == torch.int32 and em.is_cuda and em.dtype == torch.int32
  assert np.array_equal(got.cpu().numpy(), want_cc) and np.array_equal(em.cpu().numpy(), want_em)
  # a host image is moved to the labels' device; a device image with host labels is a TypeError
  with pytest.raises(TypeError, match="image is a GPU array but the volume is a host array"):
    edt.extended_maxima(ti, 1.0, lab)
  assert np.array_equal(edt.extended_maxima(img, 1.0, tl, connectivity=2).cpu().numpy(), want_em)
  # an F-ordered device view: x is its first axis, as for a host F array
  f = lambda a: torch.from_numpy(np.asfortranarray(a)).cuda().permute(2, 1, 0).contiguous().permute(2, 1, 0)
  got = edt.connected_components(f(lab), connectivity=2)
  assert got.stride() == f(lab).stride()
  assert np.array_equal(got.cpu().numpy(), cc.restate_cc(np.asfortranarray(lab), 2, "F"))
  em = edt.extended_maxima(f(img), 0.0, connectivity=3)
  assert np.array_equal(em.cpu().numpy(), cc.restate_em(np.asfortranarray(img), 0.0, None, 3, "F"))
  stack = edt.connected_components(tl[:5], stacked=True)
  assert np.array_equal(stack.cpu().numpy(), np.stack([cc.restate_cc(lab[i]) for i in range(5)]))
  empty = edt.connected_components(torch.zeros((0, 3), dtype=torch.uint8, device="cuda"))
  assert empty.is_cuda and tuple(empty.shape) == (0, 3) and empty.dtype == torch.int32


def test_label_noise_and_an_all_ones_256_cube(edt):
  rng = np.random.default_rng(256)
  noise = rng.integers(0, 4, (256, 256, 256)).astype(np.uint32)
  for conn in (1, 3):
    _check_cc(edt, noise, conn, how="scipy")
  ones = np.ones((256, 256, 256), np.uint8)
  for conn in (1, 3):
    assert (edt.connected_components(ones, connectivity=conn) == 1).all()
  # one maximum on a constant image, one per block of blocks
  blocks = (np.indices((256, 256, 256)) // 32).sum(0).astype(np.float32) % 3
  _check_em(edt, blocks, 0.0, None, 1)


def test_the_split_pipeline(edt):
  """edt -> extended_maxima -> watershed equals the same pipeline built from the restatements."""
  mask, _ = wc.balls((48, 48, 72), [(24, 24, 20), (24, 24, 44), (10, 10, 60)], [13, 9, 6])
  dist = edt.edt(mask)
  for h in (0.0, 0.5, 2.0):
    markers = edt.extended_maxima(dist, h, mask)
    want = cc.restate_em(dist, h, mask)
    assert np.array_equal(markers, want), h
    split = edt.watershed(-dist, markers, mask)
    assert np.array_equal(split, wc.flood(-dist, want, mask, 1)[0]), h
  assert edt.extended_maxima(dist, 2.0, mask).max() == 3


def _walled(edt, shape, count):
  """Slabs of label 1 between walls of label 0 on every 64th z plane, one volume (count 0) or a stack: the
  components are the slabs, numbered in z order in every volume."""
  import torch
  z = np.arange(shape[0])
  want = np.where(z % 64 == 0, 0, z // 64 + 1)
  lab = torch.ones(((count,) if count else ()) + shape, dtype=torch.uint8, device="cuda")
  lab[..., ::64, :, :] = 0
  return lab, torch.from_numpy(want.astype(np.int64)).cuda()


@pytest.mark.parametrize("count", [0, 3])
def test_past_2_to_the_31_and_32_voxels(edt, count):
  """One volume of more than 2^31 voxels (int64 out), and a stack of three volumes of 1.43e9 voxels (more
  than 2^32 voxels in all, int32 out)."""
  import torch
  shape = (1024, 2048, 1025) if count == 0 else (1024, 1024, 1366)
  vol = int(np.prod(shape))
  total = vol * max(count, 1)
  assert (vol > 1 << 31) if count == 0 else (total > 1 << 32 and vol < 1 << 31)
  out_bytes = 8 if count == 0 else 4
  need = total * (1 + 4 + out_bytes) + (2 << 30)
  free = torch.cuda.mem_get_info()[0]
  if free < need:
    pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 1e9, free / 1e9))
  try:
    lab, want = _walled(edt, shape, count)
    got = edt.connected_components(lab, stacked=count > 0)
    assert got.dtype == (torch.int64 if count == 0 else torch.int32)
    del lab
    for v in range(max(count, 1)):
      g = got[v] if count else got
      for z0 in range(0, shape[0], 128):
        assert not bool((g[z0:z0 + 128] != want[z0:z0 + 128, None, None]).any()), (v, z0)
  finally:
    lab = got = g = None
    torch.cuda.synchronize()
    edt.release()
    torch.cuda.empty_cache()
