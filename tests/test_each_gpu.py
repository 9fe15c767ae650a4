"""GPU tests of the per-label views (csrc/edt_each.cuh: label_stats_kernel, label_argmax_kernel, label_extract_kernel
and the open-addressing table behind them) against the plain restatement in each_cases.py, for exact equality:

* the table through the C ABI at capacities the test chooses: one label, a full table, overflow, load factors up
  to 0.97, probe chains that wrap round the end of the table, 64-bit keys that differ only above bit 32, signed
  and bool labels, and the slot the restated hash predicts;
* the statistics on 1-D to 3-D shapes with ragged tails, warps of 1, 2 and 32 labels, and distances that are
  negative, infinite or constant over a plateau; a 2-D image of more than 2^31 pixels;
* label_stats_cuda through its table growth, on non-contiguous tensors, other float types and a side stream;
* edtb200_label_extract box by box: what is inside the box, and that nothing outside it is touched;
* each_cuda and each (numpy in and out), label by label."""
import ctypes

import numpy as np
import pytest

import each_cases as ec

pytestmark = pytest.mark.gpu

PATTERN = 0x7fc5a5a5                                             # a NaN no kernel writes


def device_bytes(arr):
  """A numpy array's bytes on the device (so that every label dtype travels the same way)."""
  import torch
  return torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).reshape(-1).copy()).cuda()


def label_bytes(lab):
  return 1 if lab.dtype == np.bool_ else lab.itemsize


def c_stats(edt, labels_np, dt_np, capacity, dims=None):
  """edtb200_label_stats on buffers pre-filled with 0x5a bytes: (return code, overflow word, raw table)."""
  import torch
  labels_np = np.ascontiguousarray(labels_np)
  lab, dt = device_bytes(labels_np), device_bytes(np.ascontiguousarray(dt_np, dtype=np.float32))
  sx, sy, sz = dims or ec.dims_of(labels_np.shape)
  buf = {name: torch.full((capacity * width,), 0x5a, dtype=torch.uint8, device="cuda")
         for name, width in (("keys", 8), ("count", 8), ("max", 4), ("argmax", 8), ("box", 24))}
  overflow = torch.full((4,), 0x5a, dtype=torch.uint8, device="cuda")
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  rc = edt._lib().edtb200_label_stats(lab.data_ptr(), label_bytes(labels_np), dt.data_ptr(), sx, sy, sz, capacity,
                                      buf["keys"].data_ptr(), buf["count"].data_ptr(), buf["max"].data_ptr(),
                                      buf["argmax"].data_ptr(), buf["box"].data_ptr(), overflow.data_ptr(), 0, stream)
  torch.cuda.synchronize()
  assert np.array_equal(lab.cpu().numpy(), labels_np.view(np.uint8).reshape(-1))          # inputs are const
  table = {"keys": buf["keys"].cpu().numpy().view(np.uint64), "count": buf["count"].cpu().numpy().view(np.int64),
           "max": buf["max"].cpu().numpy().view(np.float32), "argmax": buf["argmax"].cpu().numpy().view(np.int64),
           "box": buf["box"].cpu().numpy().view(np.int32).reshape(-1, 6)}
  return rc, int(overflow.cpu().numpy().view(np.int32)[0]), table


def check_table(edt, lab, dt, capacity):
  """The table at `capacity` holds exactly what the restatement says, without overflow."""
  rc, overflow, table = c_stats(edt, lab, dt, capacity)
  assert rc == 0 and overflow == 0
  want = ec.stats(lab, dt)
  assert ec.mismatch(ec.table_stats(table), want) == []
  return table, want


def with_every_key(shape, keys, dtype, seed):
  lab = ec.noise(shape, keys, seed, dtype)
  assert np.unique(ec.keys_of(lab)).size == len(keys)
  return lab


WIDTHS = [(1, np.uint8, 32), (2, np.uint16, 256), (4, np.uint32, 256), (8, np.uint64, 256)]
WIDTH_IDS = ["1byte", "2bytes", "4bytes", "8bytes"]


# ---- the table ---------------------------------------------------------------------------------

def test_slot_is_where_the_restated_hash_says(edt):
  rng = np.random.default_rng(1)
  keys = np.concatenate([rng.integers(1, 1 << 63, 40, dtype=np.uint64) * np.uint64(2) + np.uint64(1),
                         rng.integers(1, 1 << 16, 10, dtype=np.uint64)])
  for key in keys.tolist():
    lab = np.zeros((3, 7), np.uint64)
    lab[1, 2:5] = key
    rc, overflow, table = c_stats(edt, lab, np.ones(lab.shape, np.float32), 1024)
    assert rc == 0 and overflow == 0
    assert np.flatnonzero(table["keys"]).tolist() == ec.home_slot(key, 1024).tolist(), hex(key)


@pytest.mark.parametrize("nbytes,dtype,capacity", WIDTHS, ids=WIDTH_IDS)
def test_one_label_in_two_slots(edt, nbytes, dtype, capacity):
  lab = np.zeros((5, 6, 7), dtype)
  lab[1:4, 2:, 3] = (1 << (8 * nbytes)) - 3
  check_table(edt, lab, ec.distances(lab, "ties", 1), 2)


@pytest.mark.parametrize("nbytes,dtype,capacity", WIDTHS, ids=WIDTH_IDS)
def test_full_table(edt, nbytes, dtype, capacity):
  """As many labels as slots: every insert succeeds, no slot stays empty, and the lookups of the argmax
  pass end without an empty slot to stop at."""
  lab = with_every_key((8, 24, 40), ec.random_keys(capacity, nbytes, 2), dtype, 3)
  table, _ = check_table(edt, lab, ec.distances(lab, "ties", 4), capacity)
  assert (table["keys"] != 0).all()


@pytest.mark.parametrize("extra", ["one_more", "four_times"])
@pytest.mark.parametrize("nbytes,dtype,capacity", WIDTHS, ids=WIDTH_IDS)
def test_overflow(edt, nbytes, dtype, capacity, extra):
  """More labels than slots: overflow is raised, the call succeeds, and every filled slot holds a key of the
  volume, each at most once.  Nothing else is promised about such a table."""
  n = capacity + 1 if extra == "one_more" else 4 * capacity
  keys = ec.random_keys(n, nbytes, 5)
  lab = with_every_key((8, 24, 40), keys, dtype, 6)
  rc, overflow, table = c_stats(edt, lab, ec.distances(lab, "ties", 7), capacity)
  assert rc == 0 and overflow == 1
  filled = table["keys"][table["keys"] != 0]
  assert np.unique(filled).size == filled.size and np.isin(filled, keys).all()


@pytest.mark.parametrize("load", [0.5, 0.75, 0.97])
@pytest.mark.parametrize("nbytes,dtype,capacity", WIDTHS, ids=WIDTH_IDS)
def test_load_factor(edt, nbytes, dtype, capacity, load):
  keys = ec.random_keys(int(load * capacity), nbytes, 8, signed=True)
  lab = with_every_key((8, 24, 40), keys, dtype, 9)
  check_table(edt, lab, ec.distances(lab, "signed", 10), capacity)


@pytest.mark.parametrize("volume", ["noise", "singletons"])
@pytest.mark.parametrize("nbytes,dtype,capacity,n", [(1, np.int8, 16, 8), (2, np.int16, 128, 64), (4, np.int32, 128, 64),
                                                     (8, np.int64, 128, 64)], ids=WIDTH_IDS)
def test_colliding_keys_wrap_round_the_table(edt, nbytes, dtype, capacity, n, volume):
  """Keys that share one home slot near the end of the table: the probe chain runs past the last slot and on
  from slot 0.  In the noise volume many warps insert the same few keys at once; in the singletons volume one
  warp inserts 32 different colliding keys in one step."""
  for home in (capacity - 1, capacity - 2):
    keys = ec.colliding_keys(n, capacity, home, nbytes)
    if volume == "noise":
      lab = with_every_key((6, 20, 37), keys, dtype, 11)
    else:
      lab = np.zeros((3, 5, 64), dtype)
      lab.ravel()[64:64 + n] = ec.as_labels(keys, dtype)
      lab.ravel()[700:700 + n] = ec.as_labels(keys[::-1], dtype)
    table, _ = check_table(edt, lab, ec.distances(lab, "ties", 12), capacity)
    slots = np.flatnonzero(table["keys"])
    assert sorted(slots.tolist()) == sorted(((home + np.arange(n)) % capacity).tolist())
    # and the same keys among others, in a table that is nearly full
    more = np.union1d(keys, ec.random_keys(int(0.97 * capacity) - n, nbytes, 13))
    lab = with_every_key((6, 20, 37), more, dtype, 14)
    check_table(edt, lab, ec.distances(lab, "negative", 15), capacity)


def test_keys_that_differ_only_above_bit_32(edt):
  low = ec.random_keys(40, 4, 16)
  keys = np.concatenate([low, low | np.uint64(1 << 32), low | np.uint64(1 << 63), low << np.uint64(32)])
  lab = with_every_key((6, 20, 37), np.unique(keys), np.int64, 17)
  assert (lab < 0).any()
  check_table(edt, lab, ec.distances(lab, "ties", 18), 512)


@pytest.mark.parametrize("dtype", [np.int8, np.int16, np.int32, np.int64, np.bool_], ids=lambda d: np.dtype(d).name)
def test_signed_and_bool_labels_are_zero_extended(edt, dtype):
  if dtype == np.bool_:
    lab = np.random.default_rng(19).uniform(size=(5, 9, 33)) < 0.6
  else:
    lab = np.random.default_rng(19).integers(-3, 3, (5, 9, 33)).astype(dtype)
  table, want = check_table(edt, lab, ec.distances(lab, "signed", 20), 16)
  width = 8 * label_bytes(lab)
  assert want["keys"].tolist() == ([1] if dtype == np.bool_ else [1, 2, (1 << width) - 3, (1 << width) - 2, (1 << width) - 1])


# ---- statistics -------------------------------------------------------------------------------

CASES = list(ec.case_volumes())


@pytest.mark.parametrize("name,lab,dt", CASES, ids=[c[0] for c in CASES])
def test_case_volume(edt, name, lab, dt):
  """Shapes down to one voxel, ragged tails, every dtype, warps of 1 / 2 / 32 labels, one label under every
  block, negative / infinite / plateau distances: through the C ABI and through label_stats_cuda."""
  import torch
  n = len(ec.stats(lab, dt)["keys"])
  capacity = 2
  while capacity < n:
    capacity *= 2
  for cap in (capacity, 4 * capacity):
    check_table(edt, lab, dt, cap)
  if lab.dtype.kind == "u" and lab.itemsize > 1:
    lab = lab.view(np.dtype("i%d" % lab.itemsize))               # same bits in a dtype every torch has
  got = edt.label_stats_cuda(torch.from_numpy(lab).cuda(), torch.from_numpy(dt).cuda())
  assert ec.mismatch(python_stats(got, lab.ndim), ec.stats(lab, dt)) == []


def python_stats(stats, nd):
  """label_stats_cuda's dict (boxes in array axis order, nd wide) in the form each_cases.stats returns."""
  box = stats["box"].cpu().numpy().reshape(-1, 2 * nd)
  n = box.shape[0]
  lo = np.concatenate([box[:, :nd][:, ::-1], np.zeros((n, 3 - nd), np.int64)], axis=1)
  hi = np.concatenate([box[:, nd:][:, ::-1], np.zeros((n, 3 - nd), np.int64)], axis=1)
  return {"keys": stats["labels"].cpu().numpy().view(np.uint64), "count": stats["count"].cpu().numpy(),
          "max": stats["max"].cpu().numpy(), "argmax": stats["argmax"].cpu().numpy(),
          "box": np.concatenate([lo, hi], axis=1)}


@pytest.mark.parametrize("shape", [(40,), (7, 5), (3, 5, 7)], ids=lambda s: "%dd" % len(s))
def test_all_background(edt, shape):
  import torch
  lab, dt = np.zeros(shape, np.uint8), np.ones(shape, np.float32)
  table, want = check_table(edt, lab, dt, 4)
  assert len(want["keys"]) == 0 and not table["keys"].any()
  lt, dtt = torch.from_numpy(lab).cuda(), torch.from_numpy(dt).cuda()
  assert len(edt.label_stats_cuda(lt, dtt)["labels"]) == 0
  it = edt.each_cuda(lt, dtt)
  assert len(it) == 0 and list(it) == []
  it = edt.each(lab, dt)
  assert len(it) == 0 and list(it) == []


@pytest.mark.parametrize("fn", ["edt", "sdf"])
def test_distances_from_a_transform(edt, fn):
  """edt leaves zeros under the background; sdf over all voxels, with the background relabelled to a key of
  its own, puts negative distances under a label."""
  lab = ec.voronoi_many((40, 72, 65), 150, 21, np.uint32, background=0.2)
  dt = getattr(edt, fn)(np.asfortranarray(lab), anisotropy=(1, 2, 1.5), black_border=True)
  dt = np.ascontiguousarray(dt)
  if fn == "sdf":
    lab = np.where(lab == 0, np.uint32(0xfffffff0), lab)
    assert (dt[lab == 0xfffffff0] < 0).all()
  check_table(edt, lab, dt, 1024)


# ---- label_stats_cuda ----------------------------------------------------------------------------

@pytest.mark.parametrize("nlabels", [600, 2049, 20000])
def test_label_stats_cuda_grows_its_table(edt, nlabels):
  """More labels than half the first table (1024 slots): the call repeats until the table is at most half full."""
  import torch
  lab = ec.voronoi_many((64, 96, 100), nlabels, 22, np.int64, ec.random_keys(nlabels, 8, 23, signed=True))
  dt = ec.distances(lab, "signed", 24)
  got = edt.label_stats_cuda(torch.from_numpy(lab).cuda(), torch.from_numpy(dt).cuda())
  want = ec.stats(lab, dt)
  assert len(want["keys"]) == nlabels
  assert ec.mismatch(python_stats(got, 3), want) == []


def test_label_stats_cuda_inputs(edt):
  """Non-contiguous tensors, float16 / float64 distances (converted to float32), and a side stream."""
  import torch
  lab = ec.voronoi_many((24, 30, 66), 90, 25, np.int32, ec.random_keys(90, 4, 26, signed=True))
  dt = ec.distances(lab, "signed", 27)                           # multiples of 1/4: exact in float16
  lt, dtt = torch.from_numpy(lab).cuda(), torch.from_numpy(dt).cuda()
  want = ec.stats(lab, dt)
  for dtype in (torch.float16, torch.float64):
    assert ec.mismatch(python_stats(edt.label_stats_cuda(lt, dtt.to(dtype)), 3), want) == []
  got = edt.label_stats_cuda(lt.permute(2, 0, 1), dtt.permute(2, 0, 1))
  assert ec.mismatch(python_stats(got, 3), ec.stats(lab.transpose(2, 0, 1), dt.transpose(2, 0, 1))) == []
  got = edt.label_stats_cuda(lt[:, ::2], dtt[:, ::2])
  assert ec.mismatch(python_stats(got, 3), ec.stats(lab[:, ::2], dt[:, ::2])) == []
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    got = edt.label_stats_cuda(lt, dtt)
  side.synchronize()
  assert ec.mismatch(python_stats(got, 3), want) == []


def test_image_of_more_than_2_31_pixels(edt):
  """46 400 x 46 400 uint8: four rectangles, one before linear index 2^31, one a full-width band, one
  straddling 2^31 and one entirely past it.  dt = x + y, so every expected value follows from the corners."""
  import torch
  free, _ = torch.cuda.mem_get_info()
  if free < 24 << 30:
    pytest.skip("needs 24 GiB of free device memory, %.1f GiB are free" % (free / 2 ** 30))
  n = 46400
  rects = {3: (100, 200, 5, 300), 7: (20000, 20010, 0, n - 1), 200: (46270, 46290, 1000, 2000),
           255: (46300, n - 1, 40000, n - 1)}                    # key: y0 y1 x0 x1 (inclusive)
  assert 46270 * n + 1000 < 1 << 31 < 46290 * n and 46300 * n > 1 << 31
  lab = torch.zeros((n, n), dtype=torch.uint8, device="cuda")
  for key, (y0, y1, x0, x1) in rects.items():
    lab[y0:y1 + 1, x0:x1 + 1] = key
  ramp = torch.arange(n, dtype=torch.float32, device="cuda")
  dt = ramp[:, None] + ramp[None, :]
  got = edt.label_stats_cuda(lab, dt)
  got = {k: v.cpu() for k, v in got.items()}
  del lab, dt
  torch.cuda.empty_cache()
  want = {"keys": np.array(sorted(rects), np.uint64),
          "count": np.array([(r[1] - r[0] + 1) * (r[3] - r[2] + 1) for _, r in sorted(rects.items())], np.int64),
          "max": np.array([r[1] + r[3] for _, r in sorted(rects.items())], np.float32),
          "argmax": np.array([r[1] * n + r[3] for _, r in sorted(rects.items())], np.int64),
          "box": np.array([[r[2], r[0], 0, r[3], r[1], 0] for _, r in sorted(rects.items())], np.int64)}
  assert ec.mismatch(python_stats(got, 2), want) == []


# ---- extraction through the C ABI ----------------------------------------------------------------

def c_extract(edt, lab_dev, nbytes, dt_dev, dims, key, box, erase, out_dev):
  import torch
  cbox = None if box is None else (ctypes.c_int * 6)(*box)
  rc = edt._lib().edtb200_label_extract(lab_dev.data_ptr(), nbytes, dt_dev.data_ptr(), dims[0], dims[1], dims[2],
                                        ctypes.c_uint64(int(key)), cbox, int(erase), out_dev.data_ptr(), 0,
                                        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
  torch.cuda.synchronize()
  return rc


@pytest.mark.parametrize("dtype", [np.uint8, np.int16, np.int32, np.int64], ids=lambda d: np.dtype(d).name)
def test_extract_box_by_box(edt, dtype):
  """Inside the box out = (labels == key) ? dt : 0 bit for bit; outside it every word keeps what it held."""
  import torch
  shape = (5, 7, 1030)
  sx, sy, sz = ec.dims_of(shape)
  nbytes = np.dtype(dtype).itemsize
  lab = ec.voronoi_many(shape, 6, 28, dtype, ec.random_keys(6, nbytes, 29, signed=True), background=0.2)
  dt = ec.distances(lab, "inf", 30)
  dt[dt == 0] = -0.0                                             # a value whose bits a float compare would lose
  st = ec.stats(lab, dt)
  key, own = int(st["keys"][-1]), st["box"][-1].tolist()
  far = int(st["keys"][0])
  lab_dev, dt_dev = device_bytes(lab), device_bytes(dt)
  boxes = [None, (0, 0, 0, sx - 1, sy - 1, sz - 1), own, (4, 3, 2, 4, 3, 2)]
  boxes += [(3, 1, 1, 3 + bx - 1, 5, 3) for bx in (1, 31, 32, 33, 1025)]
  none = np.argwhere(ec.keys_of(lab) != key)[0]                  # a one-voxel box that holds none of the label
  boxes.append((int(none[2]), int(none[1]), int(none[0])) * 2)
  have = np.full(shape, PATTERN, np.uint32).view(np.float32)
  out = device_bytes(have)
  for i, box in enumerate(boxes):
    k = key if i % 2 == 0 else far
    assert c_extract(edt, lab_dev, nbytes, dt_dev, (sx, sy, sz), k, box, 0, out) == 0
    have = ec.extract(lab, dt, k, box, False, have)
    assert np.array_equal(out.cpu().numpy().view(np.uint32), have.view(np.uint32).ravel()), (i, box)
    if i < 2:                                                    # whole volume: start from the pattern again
      have = np.full(shape, PATTERN, np.uint32).view(np.float32)
      out = device_bytes(have)
  # erase a different box: zeros inside, the pattern or the earlier drawings outside
  for box in ((0, 2, 1, 40, 4, 2), (1000, 0, 0, 1029, 6, 4), (3, 3, 3, 3, 3, 3)):
    assert c_extract(edt, lab_dev, nbytes, dt_dev, (sx, sy, sz), key, box, 1, out) == 0
    have = ec.extract(lab, dt, key, box, True, have)
    assert np.array_equal(out.cpu().numpy().view(np.uint32), have.view(np.uint32).ravel()), box
  assert (have.view(np.uint32) == PATTERN).any()
  # the empty box returns 0 and touches nothing
  for box in ((5, 0, 0, 4, 6, 4), (0, 3, 0, 9, 2, 4), (0, 0, 2, 9, 6, 1)):
    assert c_extract(edt, lab_dev, nbytes, dt_dev, (sx, sy, sz), key, box, 0, out) == 0
    assert np.array_equal(out.cpu().numpy().view(np.uint32), have.view(np.uint32).ravel()), box
  assert np.array_equal(lab_dev.cpu().numpy(), lab.view(np.uint8).ravel())
  assert np.array_equal(dt_dev.cpu().numpy(), dt.view(np.uint8).ravel())


# ---- each_cuda and each --------------------------------------------------------------------------

def test_each_cuda_over_many_labels(edt):
  """in_place=True: after every step the one image equals the restatement everywhere -- the previous label
  is erased even where the boxes overlap or nest.  in_place=False: independent images."""
  import torch
  lab = ec.voronoi_many((32, 48, 50), 2049, 31, np.int32, ec.random_keys(2049, 4, 32, signed=True), background=0.3)
  lab[4:28, 6:40, 5] = lab.ravel()[np.flatnonzero(lab)[0]]       # one label whose box holds many others
  dt = ec.distances(lab, "signed", 33)
  lt, dtt = torch.from_numpy(lab).cuda(), torch.from_numpy(dt).cuda()
  want = ec.stats(lab, dt)["keys"]
  it = edt.each_cuda(lt, dtt, in_place=True)
  assert len(it) == len(want) >= 2049
  seen, first = [], None
  for key, img in it:
    first = img if first is None else first
    assert img is first
    bits = int(np.array([key], np.int32).view(np.uint32)[0])
    assert np.array_equal(img.cpu().numpy().view(np.uint32), ec.extract(lab, dt, bits).view(np.uint32)), key
    seen.append(bits)
  assert seen == want.tolist()
  images = [(key, img) for key, img in edt.each_cuda(lt[:8], dtt[:8], in_place=False)]
  assert len({img.data_ptr() for _, img in images}) == len(images)
  for key, img in images:
    bits = int(np.array([key], np.int32).view(np.uint32)[0])
    assert np.array_equal(img.cpu().numpy().view(np.uint32), ec.extract(lab[:8], dt[:8], bits).view(np.uint32)), key


def host_labels(kind):
  rng = np.random.default_rng(34)
  if kind == "F2":
    return np.asfortranarray(ec.voronoi_many((37, 45), 20, 35, np.uint16))
  if kind == "F3":
    return np.asfortranarray(ec.voronoi_many((17, 25, 33), 30, 36, np.uint32))
  if kind == "strided":
    return ec.voronoi_many((18, 26, 34), 30, 37, np.int16, ec.random_keys(30, 2, 38))[::2, :, 1::2].transpose(1, 0, 2)
  if kind in ("float32", "float64"):
    values = np.array([-0.0, 0.0, 1.5, -2.25, np.nan, np.inf, 3.0], dtype=kind)
    return values[rng.integers(0, values.size, (9, 14, 11))]
  if kind == "bool":
    return rng.uniform(size=(9, 14, 11)) < 0.5
  return ec.voronoi_many((9, 14, 11), 25, 39, np.int64, ec.random_keys(25, 8, 40, signed=True))


@pytest.mark.parametrize("in_place", [False, True])
@pytest.mark.parametrize("kind", ["F2", "F3", "strided", "float32", "float64", "bool", "int64"])
def test_each_on_host_arrays(edt, kind, in_place):
  """Keys come back in the array's own dtype, in ascending order of their raw bits (floats by value: -0.0 is
  background, NaN a key like any other), and every image is dt masked to that key."""
  lab = host_labels(kind)
  if kind == "strided":
    assert not lab.flags.c_contiguous and not lab.flags.f_contiguous
  dt = ec.distances(np.ascontiguousarray(lab), "signed", 41)
  if kind.startswith("F"):
    dt = np.asfortranarray(dt)
  folded = np.ascontiguousarray(lab + 0 if lab.dtype.kind == "f" else lab)     # -0.0 + 0 is +0.0
  want = ec.stats(folded, dt)["keys"]
  it = edt.each(lab, dt, in_place=in_place)
  assert len(it) == len(want) > 0
  seen = []
  for key, img in it:
    assert np.asarray(key).dtype == lab.dtype and img.dtype == np.float32 and img.shape == lab.shape
    bits = int(ec.keys_of(np.array([key], lab.dtype))[0])
    assert np.array_equal(np.ascontiguousarray(img).view(np.uint32), ec.extract(folded, dt, bits).view(np.uint32)), key
    seen.append(bits)
  assert seen == want.tolist()
