"""GPU tests: fill_holes and dust equal the restatements in holes_cases.py byte for byte, with equal fill counts,
over every label width and bool (negative signed labels included), 1-D to 3-D, both memory orders, every
connectivity, stacks, device input on a side stream, holes and components that cross tile faces, edges and
corners, a cell with a nucleus, a diagonal second label, bounds at and either side of a size, empty and uniform
volumes, a 256^3 volume with thousands of holes, and stacks past 2^31 and 2^32 voxels of walled slabs."""
import numpy as np
import pytest
import scipy.ndimage as ndi

import holes_cases as hc

pytestmark = pytest.mark.gpu

SHAPES = {1: (3000,), 2: (70, 45), 3: (19, 37, 26)}


def _check_fill(edt, lab, conn=1, max_size=None, order="C", how="scipy", stacked=False):
  got, n = edt.fill_holes(lab, connectivity=conn, max_size=max_size, return_fill_count=True, stacked=stacked)
  want, m = hc.restate_fill(lab, conn, max_size, order, how, stacked=stacked)
  assert isinstance(got, np.ndarray) and got.dtype == lab.dtype and got.shape == lab.shape
  assert got.flags.f_contiguous if order == "F" else got.flags.c_contiguous
  assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (lab.shape, conn, max_size, order,
                                                                     int((got != want).sum()))
  assert np.array_equal(n, m), (n, m)
  return got, n


def _check_dust(edt, lab, threshold, conn=1, invert=False, order="C", how="scipy", stacked=False):
  got = edt.dust(lab, threshold, connectivity=conn, invert=invert, stacked=stacked)
  want = hc.restate_dust(lab, threshold, conn, invert, order, how, stacked=stacked)
  assert isinstance(got, np.ndarray) and got.dtype == lab.dtype and got.shape == lab.shape
  assert got.flags.f_contiguous if order == "F" else got.flags.c_contiguous
  assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (lab.shape, threshold, conn, invert, order)
  return got


def test_worked_examples(edt):
  assert edt.fill_holes(np.array([1, 0, 0, 1, 0])).tolist() == [1, 1, 1, 1, 0]
  assert edt.fill_holes(np.array([2, 0, 1, 0, 1])).tolist() == [2, 0, 1, 1, 1]
  ring = np.array([[0, 1, 0], [1, 0, 1], [0, 1, 0]])
  assert edt.fill_holes(ring).tolist() == [[0, 1, 0], [1, 1, 1], [0, 1, 0]]
  assert edt.fill_holes(ring, connectivity=2).tolist() == ring.tolist()
  assert edt.fill_holes(np.array([1, 0, 0, 1]), max_size=1).tolist() == [1, 0, 0, 1]
  assert edt.fill_holes(np.array([1, 0, 0, 1]), return_fill_count=True)[1] == 2
  x = np.array([1, 1, 0, 2, 0, 1])
  assert edt.dust(x, 2).tolist() == [1, 1, 0, 0, 0, 0]
  assert edt.dust(x, 2, invert=True).tolist() == [0, 0, 0, 2, 0, 1]
  d = np.array([[1, 0], [0, 1]])
  assert edt.dust(d, 2).tolist() == [[0, 0], [0, 0]]
  assert edt.dust(d, 2, connectivity=2).tolist() == [[1, 0], [0, 1]]


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("nd", [1, 2, 3])
def test_random_volumes_orders_dims_and_connectivities(edt, order, nd):
  rng = np.random.default_rng(nd * 10 + (order == "F"))
  for conn in range(1, nd + 1):
    lab = hc.random_labels(rng, SHAPES[nd], nlabels=2 if nd < 3 else 1, p=0.6 if nd < 3 else 0.7)
    mask = hc.random_mask(rng, SHAPES[nd])
    if order == "F":
      lab, mask = np.asfortranarray(lab), np.asfortranarray(mask)
    _check_fill(edt, lab, conn, order=order)
    _check_fill(edt, lab, conn, max_size=3, order=order)
    got, _ = _check_fill(edt, mask, conn, order=order)
    assert np.array_equal(got, ndi.binary_fill_holes(mask, hc.structure(nd, conn)))
    for threshold in (2, 5):
      _check_dust(edt, lab, threshold, conn, order=order)
      _check_dust(edt, lab, threshold, conn, invert=True, order=order)


@pytest.mark.parametrize("dtype", [np.bool_, np.uint8, np.int8, np.uint16, np.int16, np.uint32, np.int32,
                                   np.uint64, np.int64])
def test_every_label_width(edt, dtype):
  rng = np.random.default_rng(np.dtype(dtype).num)
  base = hc.random_labels(rng, (13, 17, 40), nlabels=3, p=0.65)
  if dtype == np.bool_:
    lab = base != 0
  elif np.dtype(dtype).kind == "i":
    lab = np.array([0, -1, -2, 1], dtype)[base]                                  # negative labels too
  else:
    lab = (base.astype(np.uint64) * (np.iinfo(dtype).max // 7)).astype(dtype)
  for conn in (1, 3):
    _check_fill(edt, lab, conn)
    _check_fill(edt, lab, conn, how="flood")
    _check_dust(edt, lab, 4, conn)
    _check_dust(edt, lab, 4, conn, how="cc", invert=True)


@pytest.mark.parametrize("name,lab,conn", hc.crossing_holes(), ids=[c[0] for c in hc.crossing_holes()])
def test_holes_and_components_that_cross_tiles(edt, name, lab, conn):
  _, n = _check_fill(edt, lab, conn)
  assert (n == 0) == name.startswith("open_")
  _check_fill(edt, np.asfortranarray(lab), conn, order="F")
  # the structure as one component of label 1: kept at its size, dropped one voxel above it
  s = (lab == 0).astype(np.uint8)
  size = int(s.sum())
  if name.startswith("open_"):
    assert _check_dust(edt, s, size, conn).sum() == size
    assert _check_dust(edt, s, size + 1, conn).sum() == 0


def test_a_cell_with_a_nucleus(edt):
  for nd in (2, 3):
    lab, want = hc.cell_with_nucleus(nd)
    for conn in range(1, nd + 1):
      got, n = _check_fill(edt, lab, conn)
      assert np.array_equal(got, want) and n == 1


def test_a_second_label_touching_a_hole_diagonally(edt):
  lab = hc.diagonal_touch()
  assert _check_fill(edt, lab, 1)[0][2, 2] == 1
  assert _check_fill(edt, lab, 2)[0][2, 2] == 0


def test_bounds_at_and_either_side_of_a_size(edt):
  for size in (1, 7, 40):
    lab = hc.sized_hole(size)
    for bound, filled in ((size - 1, 0), (size, size), (size + 1, size), (0, 0), (lab.size, size)):
      assert _check_fill(edt, lab, 1, max_size=bound)[1] == filled, (size, bound)
    comp = (lab == 0).astype(np.uint8)                          # one component of `size` voxels
    for threshold, kept in ((size - 1, True), (size, True), (size + 1, False), (0, True), (lab.size + 1, False)):
      assert bool(_check_dust(edt, comp, threshold).any()) == kept, (size, threshold)
      assert bool(_check_dust(edt, comp, threshold, invert=True).any()) == (not kept), (size, threshold)


@pytest.mark.parametrize("order", ["C", "F"])
def test_stacks_are_the_per_volume_calls(edt, order):
  a = hc.stacked_slabs()
  if order == "F":
    a = np.asfortranarray(a.T)
  got, n = _check_fill(edt, a, 1, order=order, stacked=True)
  assert n.tolist() == [8, 0]
  rng = np.random.default_rng(4)
  for shape, conn in (((4, 21, 19), 2), ((3, 7, 10, 9), 3), ((5, 70), 1)):
    lab = np.stack([hc.random_labels(rng, shape[1:], nlabels=2) for _ in range(shape[0])])
    lab[1] = 0
    if order == "F":
      lab = np.asfortranarray(lab.T)
    _check_fill(edt, lab, conn, order=order, stacked=True)
    _check_dust(edt, lab, 3, conn, order=order, stacked=True)
  # per-slice 2-D filling of a 3-D stack is scipy's per slice
  mask = hc.random_mask(rng, (6, 30, 40))
  got = edt.fill_holes(mask, stacked=True)
  assert np.array_equal(got, np.stack([ndi.binary_fill_holes(m) for m in mask]))


def test_device_input_on_a_side_stream(edt):
  import torch
  rng = np.random.default_rng(9)
  lab = hc.random_labels(rng, (18, 23, 29), nlabels=2, p=0.7).astype(np.int32)
  want, m = hc.restate_fill(lab, 2)
  want_d = hc.restate_dust(lab, 3, 2)
  stack_want, stack_m = hc.restate_fill(lab[:5], 1, stacked=True)
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    tl = torch.from_numpy(lab).cuda()
    got, n = edt.fill_holes(tl, connectivity=2, return_fill_count=True)
    dusted = edt.dust(tl, 3, connectivity=2)
    sgot, sn = edt.fill_holes(tl[:5], return_fill_count=True, stacked=True)
  side.synchronize()
  assert got.is_cuda and got.dtype == torch.int32 and dusted.is_cuda and sn.is_cuda and sn.dtype == torch.int64
  assert np.array_equal(got.cpu().numpy(), want) and n == m
  assert np.array_equal(dusted.cpu().numpy(), want_d)
  assert np.array_equal(sgot.cpu().numpy(), stack_want) and np.array_equal(sn.cpu().numpy(), stack_m)
  f = torch.from_numpy(np.asfortranarray(lab)).cuda().permute(2, 1, 0).contiguous().permute(2, 1, 0)
  got = edt.fill_holes(f, connectivity=3)
  assert got.stride() == f.stride()
  assert np.array_equal(got.cpu().numpy(), hc.restate_fill(np.asfortranarray(lab), 3, order="F")[0])
  mask = torch.from_numpy(lab != 0).cuda()
  assert np.array_equal(edt.fill_holes(mask).cpu().numpy(), ndi.binary_fill_holes(lab != 0))


def test_empty_and_uniform_volumes(edt):
  for shape in ((0,), (0, 5), (3, 0, 2)):
    got, n = edt.fill_holes(np.zeros(shape, np.uint8), return_fill_count=True)
    assert got.shape == shape and n == 0
    assert edt.dust(np.zeros(shape, np.uint16), 3).shape == shape
  got, n = edt.fill_holes(np.zeros((0, 4, 4), np.uint8), return_fill_count=True, stacked=True)
  assert got.shape == (0, 4, 4) and n.shape == (0,)
  for value in (0, 5):
    lab = np.full((20, 33, 17), value, np.uint32)
    got, n = _check_fill(edt, lab, 3)
    assert n == 0 and np.array_equal(got, lab)
    _check_dust(edt, lab, lab.size)
    _check_dust(edt, lab, lab.size + 1)


def test_256_cube_with_thousands_of_holes(edt):
  rng = np.random.default_rng(256)
  n = 256
  lab = np.zeros((n, n, n), np.uint16)
  lab[(np.indices((n, n, n)) // 16).sum(0) % 2 == 0] = 1                      # a checkerboard of 16^3 blocks
  lab[lab == 1] += (np.indices((n, n, n))[0] // 64).astype(np.uint16)[lab == 1]
  holes = rng.random((n, n, n)) < 0.02
  lab[holes] = 0
  for conn in (1, 3):
    got, filled = _check_fill(edt, lab, conn)
    assert filled > 1000
    _check_dust(edt, lab, 8, conn)


def _walled(shape, count):
  """Slabs of label 1 with walls on every 64th z plane, and in each slab a cavity of 2x2x2 voxels: the
  cavities are the holes, and with a dust threshold above 8 only the 1-voxel specks on the walls go."""
  import torch
  lab = torch.ones(((count,) if count else ()) + shape, dtype=torch.uint8, device="cuda")
  lab[..., ::64, :, :] = 0
  z = torch.arange(32, shape[0] - 32, 64, device="cuda")
  for dz in (0, 1):
    for dy in (0, 1):
      lab[..., z + dz, 100 + dy, 200:202] = 0
  return lab, int(z.numel()) * 8


@pytest.mark.parametrize("count", [0, 3])
def test_past_2_to_the_31_and_32_voxels(edt, count):
  """One volume of more than 2^31 voxels, and a stack of three volumes of 1.43e9 voxels (more than 2^32 in
  all)."""
  import torch
  shape = (1024, 2048, 1025) if count == 0 else (1024, 1024, 1366)
  vol = int(np.prod(shape))
  total = vol * max(count, 1)
  need = total * (1 + 1 + 4 + 4 + 1) + (2 << 30)
  free = torch.cuda.mem_get_info()[0]
  if free < need:
    pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 1e9, free / 1e9))
  lab = got = None
  try:
    lab, holes = _walled(shape, count)
    got, n = edt.fill_holes(lab, return_fill_count=True, stacked=count > 0)
    if count:
      assert n.tolist() == [holes] * count
    else:
      assert n == holes
    # only the cavities change, to 1: the walls touch the faces and stay open
    assert int((got != lab).sum()) == holes * max(count, 1) and bool((got >= lab).all())
    del got
    lab[..., 64, 5, 7] = 2                                                      # a speck of its own label
    got = edt.dust(lab, 9, stacked=count > 0)
    assert int((got != lab).sum()) == max(count, 1)
  finally:
    lab = got = None
    torch.cuda.synchronize()
    edt.release()
    torch.cuda.empty_cache()
