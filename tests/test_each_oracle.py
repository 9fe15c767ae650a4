"""CPU tests that pin each_cases.py, the restatement the GPU tests of the per-label views compare with: `stats`
and `extract` against loops written a second, slower way, `extract` against the reference's own `each`, the
restated hash and its colliding key sets, and planted defects that the committed case volumes must notice."""
import numpy as np
import pytest

import each_cases as ec

SMALL = [((1,), np.uint8), ((6,), np.int8), ((4, 5), np.int16), ((6, 6, 6), np.int32), ((3, 5, 6), np.int64),
         ((2, 6, 5), np.uint64), ((5, 6, 4), np.bool_)]


def small_volume(shape, dtype, seed):
  rng = np.random.default_rng(seed)
  nbytes = np.dtype(dtype).itemsize
  keys = np.concatenate([[0, 0], ec.random_keys(5, nbytes, seed, signed=np.dtype(dtype).kind == "i")])
  return ec.as_labels(keys[rng.integers(0, keys.size, shape)], dtype).reshape(shape)


def total_order_less(a, b):
  """a < b for two float32 under the IEEE total order, from sign and magnitude."""
  ua, ub = int(np.float32(a).view(np.uint32)), int(np.float32(b).view(np.uint32))
  (sa, ma), (sb, mb) = (ua >> 31, ua & 0x7fffffff), (ub >> 31, ub & 0x7fffffff)
  if sa != sb:
    return sa > sb
  return ma > mb if sa else ma < mb


def stats_by_loops(labels, dt):
  """One Python loop over the voxels per key."""
  sx, sy, sz = ec.dims_of(labels.shape)
  width = 8 * (1 if labels.dtype == np.bool_ else labels.itemsize)
  flat = [int(v) & ((1 << width) - 1) for v in labels.ravel().tolist()]
  dist = np.asarray(dt, np.float32).ravel()
  rows = []
  for key in sorted(set(flat) - {0}):
    count, best, where, lo, hi = 0, None, None, [sx, sy, sz], [-1, -1, -1]
    for i, v in enumerate(flat):
      if v != key:
        continue
      count += 1
      if best is None or total_order_less(best, dist[i]):
        best, where = dist[i], i
      p = (i % sx, i // sx % sy, i // (sx * sy))
      lo = [min(a, b) for a, b in zip(lo, p)]
      hi = [max(a, b) for a, b in zip(hi, p)]
    rows.append((key, count, best, where, lo + hi))
  return {"keys": np.array([r[0] for r in rows], np.uint64), "count": np.array([r[1] for r in rows], np.int64),
          "max": np.array([r[2] for r in rows], np.float32), "argmax": np.array([r[3] for r in rows], np.int64),
          "box": np.array([r[4] for r in rows], np.int64).reshape(-1, 6)}


@pytest.mark.parametrize("kind", ec.DT_KINDS)
@pytest.mark.parametrize("shape,dtype", SMALL, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else np.dtype(v).name)
def test_stats_against_loops(shape, dtype, kind):
  lab = small_volume(shape, dtype, 3 + len(shape))
  dt = ec.distances(lab, kind, 7)
  if kind == "signed":
    dt.ravel()[::5] = -0.0                                       # -0.0 orders below +0.0
    dt.ravel()[1::5] = 0.0
  assert ec.mismatch(ec.stats(lab, dt), stats_by_loops(lab, dt)) == []


def test_stats_of_an_empty_volume():
  got = ec.stats(np.zeros((3, 4), np.uint16), np.ones((3, 4), np.float32))
  assert all(len(got[f]) == 0 for f in ec.FIELDS) and got["box"].shape == (0, 6)


@pytest.mark.parametrize("shape,dtype", SMALL[2:], ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else np.dtype(v).name)
def test_extract_against_loops(shape, dtype):
  rng = np.random.default_rng(5)
  lab = small_volume(shape, dtype, 9)
  dt = ec.distances(lab, "signed", 2)
  sx, sy, sz = ec.dims_of(shape)
  before = rng.uniform(1, 2, shape).astype(np.float32)
  keys = ec.keys_of(lab).reshape(sz, sy, sx)
  for key in [int(k) for k in np.unique(keys)[:3]] + [12345]:
    for erase in (False, True):
      lo = [int(rng.integers(0, n)) for n in (sx, sy, sz)]
      hi = [int(rng.integers(a, n)) for a, n in zip(lo, (sx, sy, sz))]
      want = before.copy().reshape(sz, sy, sx)
      for z in range(lo[2], hi[2] + 1):
        for y in range(lo[1], hi[1] + 1):
          for x in range(lo[0], hi[0] + 1):
            want[z, y, x] = dt.reshape(sz, sy, sx)[z, y, x] if keys[z, y, x] == key and not erase else 0.0
      got = ec.extract(lab, dt, key, lo + hi, erase, before)
      assert got.shape == shape and np.array_equal(got.view(np.uint32), want.reshape(shape).view(np.uint32))
  whole = ec.extract(lab, dt, int(np.unique(keys)[-1]))
  assert np.array_equal(whole, np.where(ec.keys_of(lab) == np.unique(keys)[-1], dt, np.float32(0)))


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint32, np.uint64])
def test_extract_equals_the_reference_each(reference, dtype, order):
  if reference is None:
    pytest.skip("the reference is not built (oracle/_ref)")
  lab = ec.voronoi_many((9, 8, 7), 12, 4, dtype)
  dt = ec.distances(lab, "ties", 1) + np.float32(0.25)           # the reference's images hold what dt holds
  lab_o, dt_o = (np.asfortranarray(lab), np.asfortranarray(dt)) if order == "F" else (lab, dt)
  seen = []
  for key, img in reference.each(lab_o, dt_o, in_place=False):
    assert np.array_equal(np.ascontiguousarray(img), ec.extract(lab, dt, int(key))), key
    seen.append(int(key))
  assert sorted(seen) == ec.stats(lab, dt)["keys"].tolist()


@pytest.mark.parametrize("defect", ec.DEFECTS)
def test_case_volumes_notice_a_planted_defect(defect):
  """`mismatch`, the comparison the GPU tests use, reports each planted defect on some committed volume, in the
  field the defect belongs to."""
  field = {"last_tie": "argmax", "exclusive_box": "box", "unsigned_max": "max", "sign_extend": "keys"}[defect]
  caught = [name for name, lab, dt in ec.case_volumes()
            if field in ec.mismatch(ec.stats(lab, dt, defect=defect), ec.stats(lab, dt))]
  assert len(caught) >= 3, (defect, caught)


def test_case_volumes_cover_the_list():
  cases = list(ec.case_volumes())
  names = [c[0] for c in cases]
  assert len(set(names)) == len(names)
  assert {len(lab.shape) for _, lab, _ in cases} == {1, 2, 3}
  assert {np.dtype(lab.dtype).itemsize for _, lab, _ in cases} == {1, 2, 4, 8}
  assert any(lab.size % 32 == 1 and lab.ravel()[-1] != 0 for _, lab, _ in cases)
  for _, lab, dt in cases:
    assert lab.flags.c_contiguous and dt.dtype == np.float32 and not np.isnan(dt).any()
  for kind, check in (("inf", np.isposinf), ("inf", np.isneginf), ("negative", lambda m: m < 0)):
    assert any(kind in name and check(ec.stats(lab, dt)["max"]).any() for name, lab, dt in cases), kind


def test_slot_hash_is_the_64_bit_finaliser():
  def scalar(k):
    m = (1 << 64) - 1
    k ^= k >> 33
    k = k * 0xff51afd7ed558ccd & m
    k ^= k >> 33
    k = k * 0xc4ceb9fe1a85ec53 & m
    k ^= k >> 33
    return k & 0xffffffff
  keys = [1, 2, 255, 1 << 32, (1 << 64) - 1, 0x8000000000000000, 123456789123456789]
  assert ec.slot_hash(np.array(keys, np.uint64)).tolist() == [scalar(k) for k in keys]
  assert ec.slot_hash(7).tolist() == [scalar(7)]


@pytest.mark.parametrize("nbytes,capacity,n", [(1, 16, 8), (2, 128, 64), (4, 128, 64), (8, 128, 64)])
def test_colliding_keys_collide_and_wrap(nbytes, capacity, n):
  for home in (capacity - 1, capacity - 2):
    keys = ec.colliding_keys(n, capacity, home, nbytes)
    assert keys.size == n == np.unique(keys).size and keys.min() > 0
    assert int(keys.max()) < 1 << (8 * nbytes)
    assert (ec.home_slot(keys, capacity) == home).all()
    # linear probing from `home` places them in home, home + 1, ...: past the end, so from slot 0 on
    slots = (home + np.arange(n)) % capacity
    assert slots.max() == capacity - 1 and slots.min() == 0 and (np.diff(slots) < 0).sum() == 1


def test_makers():
  lab = ec.stripes((6, 10, 64), 1, 32).ravel()
  assert all(np.unique(lab[i:i + 32]).size == 32 for i in range(0, lab.size, 32))
  lab = ec.stripes((6, 10, 64), 16, 64).ravel()
  assert all(np.unique(lab[i:i + 32]).size == 2 for i in range(0, lab.size, 32))
  lab = ec.stripes((6, 10, 64), 64, 5).ravel()
  assert all(np.unique(lab[i:i + 32]).size == 1 for i in range(0, lab.size, 32))
  keys = ec.random_keys(500, 8, 1, signed=True)
  lab = ec.singletons((4, 5, 25), keys, 2, np.int64)
  assert np.unique(lab).size == 500 and (lab < 0).any()
  lab = ec.voronoi_many((20, 21, 22), 700, 3, np.uint32)
  assert np.unique(lab[lab != 0]).size == 700 and 0.05 < (lab == 0).mean() < 0.15
  lab = ec.noise((4, 5, 6), keys[:100], 4, np.int64, background=0.5)
  assert np.unique(lab[lab != 0]).size == 100
