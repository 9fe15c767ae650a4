"""GPU tests of local_thickness, bit for bit: against the threshold restatement on the CPU oracle at the
levels the call returns, for every label dtype (float labels with -0.0 and NaN payloads, bool), C and F
order, 1-D to 3-D, integer and non-integer anisotropy and both black_border values; against the maximum of
spherical_open calls at the same levels; stacks against per-volume calls (their default levels differ per
volume); the default levels against their formula in float64; device input on a non-default stream; and
the edge cases (a level of 0, one label without black border, an all-background volume)."""
import numpy as np
import pytest

import local_thickness_cases as lt
import morphology_cases as mc

pytestmark = pytest.mark.gpu

DTYPES = [np.bool_, np.uint8, np.int8, np.uint16, np.int16, np.uint32, np.int32, np.uint64, np.int64, np.float32,
          np.float64]


def labels_of(rng, dtype, shape):
  if dtype == np.bool_:
    return mc.balls(rng, shape, 6, 8.0, np.uint8) != 0
  if np.dtype(dtype).kind == "f":
    base = mc.touching(rng, shape, np.int32).astype(dtype)
    bits = np.uint32(0x7FC01234) if dtype == np.float32 else np.uint64(0x7FF8000000ABCDEF)
    base[base == 2] = np.array([bits]).view(dtype)[0]
    base[base == 3] = -1.5
    base[(base == 0) & (rng.random(shape) < 0.5)] = -0.0
    return base
  kind = ("voronoi", "balls", "touching")[DTYPES.index(dtype) % 3]
  return mc.seeded(rng, kind, shape, dtype)


def check(edt, arr, w=None, bb=False, sizes=6):
  got, levels = edt.local_thickness(arr, w, bb, sizes=sizes, return_sizes=True)
  assert got.dtype == np.float32 and got.shape == arr.shape
  if arr.ndim > 1:
    assert got.flags.f_contiguous == (arr.flags.f_contiguous and not arr.flags.c_contiguous)
  want = lt.threshold(arr, levels, w, bb)
  assert np.array_equal(got, want), (w, bb, int((got != want).sum()))
  if isinstance(sizes, int):
    np.testing.assert_array_max_ulp(levels, lt.default_levels(arr, sizes, w, bb), maxulp=4)
  return got, levels


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: np.dtype(d).name)
def test_dtypes_and_orders(edt, dtype, order):
  rng = np.random.default_rng(DTYPES.index(dtype))
  arr = labels_of(rng, dtype, (30, 27, 22))
  arr = np.asfortranarray(arr) if order == "F" else np.ascontiguousarray(arr)
  for bb in (False, True):
    check(edt, arr, None, bb, sizes=6)
    check(edt, arr, None, bb, sizes=[0.0, 1.0, 1.5, 2.5, 4.0, 9.0])


@pytest.mark.parametrize("w", [(1.0, 2.0, 1.0), (0.7, 1.3, 2.9), (3.0, 1.0, 0.5)])
def test_anisotropy(edt, w):
  rng = np.random.default_rng(7)
  arr = np.asfortranarray(mc.voronoi(rng, (26, 21, 24), 7, np.uint16))
  for bb in (False, True):
    check(edt, arr, w, bb, sizes=8)
    check(edt, np.ascontiguousarray(arr), w, bb, sizes=[0.9, 2.0, 2.6, 4.2, 11.0])


@pytest.mark.parametrize("shape", [(300,), (70, 45), (9, 300)], ids=["1d", "2d", "2d_tall"])
def test_one_and_two_dimensions(edt, shape):
  rng = np.random.default_rng(len(shape) * 3 + shape[0])
  w = (1.5,) if len(shape) == 1 else (1.0, 0.75)
  for kind in mc.KINDS:
    arr = mc.seeded(rng, kind, shape, np.uint32)
    for bb in (False, True):
      check(edt, arr, w, bb, sizes=10)
      check(edt, arr, None, bb, sizes=[0.5, 1.0, 2.0, 3.0, 17.0])


def test_equals_the_maximum_of_openings(edt):
  rng = np.random.default_rng(11)
  for arr, w in ((mc.voronoi(rng, (64, 70, 80), 40, np.uint32), (1.0, 1.0, 1.0)),
                 (mc.balls(rng, (48, 60, 52), 12, 14.0, np.uint8), (1.0, 0.8, 1.25))):
    for bb in (False, True):
      got, levels = edt.local_thickness(arr, w, bb, sizes=9, return_sizes=True)
      want = np.zeros(arr.shape, np.float32)
      for r in levels:
        want = np.maximum(want, np.where(edt.spherical_open(arr, r, w, bb) != 0, np.float32(r), np.float32(0)))
      assert np.array_equal(got, want), bb


def test_stacks_equal_per_volume_calls(edt):
  rng = np.random.default_rng(5)
  vols = [mc.balls(rng, (20, 24, 18), 4, 3.0 + 3 * i, np.uint16) for i in range(4)]
  vols.append(np.zeros((20, 24, 18), np.uint16))                  # no labelled voxel: R = h/2
  stack = np.stack(vols)
  for bb in (False, True):
    got, levels = edt.local_thickness(stack, (1.0, 2.0, 1.5), bb, sizes=7, return_sizes=True, stacked=True)
    assert levels.shape == (5, 7)
    for i, v in enumerate(vols):
      one, lv = edt.local_thickness(v, (1.0, 2.0, 1.5), bb, sizes=7, return_sizes=True)
      assert np.array_equal(got[i], one) and np.array_equal(levels[i], lv), (i, bb)
    assert len({tuple(row) for row in levels}) > 1                   # the volumes' levels differ
    got, lv = edt.local_thickness(stack, (1.0, 2.0, 1.5), bb, sizes=[1.0, 2.5, 4.0], return_sizes=True, stacked=True)
    assert list(lv) == [4.0, 2.5, 1.0]
    assert np.array_equal(got, np.stack([edt.local_thickness(v, (1.0, 2.0, 1.5), bb, sizes=[1.0, 2.5, 4.0])
                                         for v in vols]))


def test_known_answers(edt):
  got, levels = edt.local_thickness(lt.run_of_seven(), return_sizes=True)
  assert 3.5 < levels[0] < 4.0 and np.all(got[1:-1] == np.float32(levels[0]))
  arr, mid = lt.rod_between_balls()
  assert edt.local_thickness(arr, sizes=[0.5, 1.0, 2.0, 4.0])[mid] == 1.0
  line = lt.thin_line()
  got = edt.local_thickness(line, sizes=(0.5, 1.0, 2.0))
  assert np.all(got[line != 0] == 0.5) and not got[line == 0].any()


def test_edge_cases(edt):
  rng = np.random.default_rng(2)
  arr = mc.voronoi(rng, (20, 21, 22), 5, np.uint8)
  assert not edt.local_thickness(arr, sizes=[0.0]).any()           # level 0 covers nothing but gives 0
  one = np.full((12, 13, 9), 3, np.int32)
  got, levels = edt.local_thickness(one, (2.0, 1.0, 3.0), sizes=5, return_sizes=True)
  assert np.all(levels == 0.5) and np.all(got == 0.5)              # no finite D2: R = h/2, every voxel a seed
  got, levels = edt.local_thickness(one, (2.0, 1.0, 3.0), True, sizes=5, return_sizes=True)
  assert np.array_equal(got, lt.threshold(one, levels, (2.0, 1.0, 3.0), True)) and got.max() > 0.5
  empty = np.zeros((10, 11, 12), np.uint16)
  got, levels = edt.local_thickness(empty, sizes=4, return_sizes=True)
  assert not got.any() and np.all(levels == 0.5)


def test_device_input_on_a_side_stream(edt):
  torch = pytest.importorskip("torch")
  rng = np.random.default_rng(9)
  arr = mc.voronoi(rng, (33, 40, 28), 9, np.int32)
  want, want_levels = edt.local_thickness(arr, (1.0, 1.5, 2.0), True, sizes=6, return_sizes=True)
  want_given = edt.local_thickness(arr, (1.0, 1.5, 2.0), True, sizes=[3.0, 1.0, 2.0])
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    t = torch.from_numpy(arr).to("cuda")
    got, levels = edt.local_thickness(t, (1.0, 1.5, 2.0), True, sizes=6, return_sizes=True)
    given, given_levels = edt.local_thickness(t, (1.0, 1.5, 2.0), True, sizes=[3.0, 1.0, 2.0], return_sizes=True)
    ft = torch.from_numpy(np.asfortranarray(arr)).to("cuda").permute(2, 1, 0).contiguous().permute(2, 1, 0)
    got_f = edt.local_thickness(ft, (1.0, 1.5, 2.0), True, sizes=6)
    stack, stack_levels = edt.local_thickness(torch.stack([t, t.flip(0)]), (1.0, 1.5, 2.0), True, sizes=6,
                                              return_sizes=True, stacked=True)
  side.synchronize()
  assert got.is_cuda and levels.is_cuda and given_levels.is_cuda and got.dtype == torch.float32
  assert np.array_equal(got.cpu().numpy(), want) and np.array_equal(levels.cpu().numpy(), want_levels)
  assert np.array_equal(given.cpu().numpy(), want_given) and given_levels.cpu().tolist() == [3.0, 2.0, 1.0]
  assert not got_f.is_contiguous() and np.array_equal(got_f.cpu().numpy(), want)
  assert stack_levels.shape == (2, 6) and np.array_equal(stack[0].cpu().numpy(), want)
  assert np.array_equal(stack[1].cpu().numpy(), edt.local_thickness(arr[::-1].copy(), (1.0, 1.5, 2.0), True, sizes=6))
