"""Every operation past 2^31 and 2^32 voxels, against walled tiles whose answers are known
(tests/large_index_cases.py; the identity each comparison rests on is checked on the CPU by
tests/test_large_index_oracle.py).

A big volume is a lattice of K = 7 tile variants with walls; inside every tile it must equal, bit for
bit, the same call on the variant alone, translated.  Stacks of small volumes are the lattice (B, 1, 1)
without walls: every volume must equal its variant's single-volume call.  Volumes are assembled and
compared on the device, one slab of tiles at a time.

Each test skips, with the figure, when the device has less free memory than the peak measured for it
(the drop in cudaMemGetInfo's free memory over the test, polled from a thread, printed with -s), plus a
margin.  Which later-pass kernel each call ran is recorded; the last test asserts the tile and window
kernels ran past 2^31 voxels and the long-line kernel past 2^32."""
import functools
import gc
import threading
import traceback

import numpy as np
import pytest

import large_index_cases as lc

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GB = 1 << 30
K = 7
W3, W2 = (1.0, 2.0, 1.0), (1.0, 2.0)
SHAPE3, TILE3 = (528, 2048, 2048), (16, 32, 64)            # 2.21e9 voxels
SHAPE4G = (1040, 2048, 2048)                               # 4.36e9 voxels
SHAPE2, TILE2 = (46368, 46368), (48, 48)                   # 2.15e9 pixels
RAN = []                                                   # (what, later-pass kernel, voxels)


def counts(shape, tile):
  assert all(s % t == 0 for s, t in zip(shape, tile)), (shape, tile)
  return tuple(s // t for s, t in zip(shape, tile))


def need(gbytes):
  free, _ = torch.cuda.mem_get_info()
  if free < gbytes * GB:
    pytest.skip("needs %.0f GB of free device memory, %.1f GB free" % (gbytes, free / GB))


@pytest.fixture(autouse=True)
def peak(edt):
  """Print the test's peak device memory (GB below the free memory at its start) and give it all back."""
  torch.cuda.synchronize()
  start = torch.cuda.mem_get_info()[0]
  low, done = [start], threading.Event()

  def poll():
    while not done.wait(0.002):
      low[0] = min(low[0], torch.cuda.mem_get_info()[0])
  th = threading.Thread(target=poll, daemon=True)
  th.start()
  yield
  torch.cuda.synchronize()
  done.set()
  th.join()
  low[0] = min(low[0], torch.cuda.mem_get_info()[0])
  print("\npeak %.1f GB of %.1f GB free" % ((start - low[0]) / GB, start / GB))
  torch.cuda.empty_cache()
  edt.release()


def released(test):
  """Run the test so that a failure keeps none of its device memory: pytest keeps a failed test's
  traceback, and with it every frame's tensors, to the end of the session, and the next tests would skip
  for want of memory.  The failure is re-raised as an AssertionError carrying the original traceback's text."""
  @functools.wraps(test)
  def run(*args, **kwargs):
    try:
      return test(*args, **kwargs)
    except Exception as e:                   # pytest's skip is not an Exception
      msg = "%s: %s\n%s" % (type(e).__name__, e, traceback.format_exc())
    gc.collect()
    torch.cuda.empty_cache()
    raise AssertionError(msg)
  return run


def ran(what, n):
  RAN.append((what, edt_b200().last_later_launch()["kernel"], n))


def edt_b200():
  import edt_b200 as mod
  return mod


def labels_of(shape, tile, t, dtype, seed):
  pool = torch.from_numpy(lc.label_pool(np.random.default_rng(seed), K, tile, t, dtype)).cuda()
  return pool, lc.assemble(pool, counts(shape, tile))


def stack_of(pool, count):
  return lc.stack(pool, count)


def answers(fn, pool):
  return torch.stack([fn(pool[k]) for k in range(K)])


# ---- single volumes past 2^31 voxels ----------------------------------------------------------------

@pytest.mark.parametrize("dtype", [np.uint8, np.int32])
@released
def test_transforms_beyond_2_31(edt, dtype):
  """edt_cuda unsigned and signed, unbounded (tile kernel) and at max_distance 2 and 8 (window kernel),
  on 528 x 2048 x 2048 labels of 1 and 4 bytes (the X pass's run-start planes)."""
  need({np.uint8: 22, np.int32: 28}[dtype])     # measured peaks: 19.6 and 25.6 GB
  pool, lab = labels_of(SHAPE3, TILE3, 1, dtype, 11)
  assert lab.numel() > 2**31
  out = torch.empty(SHAPE3, dtype=torch.float32, device="cuda")
  for border, sqrt, signed, d in ((True, False, False, None), (False, True, True, None), (False, False, False, 2.0),
                                  (True, True, True, 8.0)):
    kw = dict(sqrt=sqrt, signed=signed, max_distance=d)
    edt.edt_cuda(lab, W3, border, out=out, **kw)
    ran("edt_cuda %s %s" % (dtype.__name__, kw), lab.numel())
    # the window kernel takes radii up to EDTB200_BOUNDED_WINDOW_MAX = 2 rows; at 8 the Z pass is the tile
    # kernel's, then the cut
    assert RAN[-1][1] == ("window" if d == 2.0 else "tile"), RAN[-1]
    want = answers(lambda v: edt.edt_cuda(v, W3, border, **kw), pool)
    lc.assert_tiles(out, want, counts(SHAPE3, TILE3), 1, what="edt_cuda %s" % kw)


@pytest.mark.parametrize("op", ["erode", "open", "dilate", "close"])
@released
def test_morphology_beyond_2_31(edt, op):
  """The four spherical operations at radius 2 on 528 x 2048 x 2048 one-byte labels."""
  need(25)                                   # measured peaks: 20.7 to 22.8 GB
  pool, lab = labels_of(SHAPE3, TILE3, 1, np.uint8, 14)
  fn = getattr(edt, "spherical_" + op)
  kw = {} if op == "dilate" else {"black_border": op != "close"}
  out = fn(lab, 2.0, W3, **kw)
  ran("spherical_" + op, lab.numel())
  lc.assert_tiles(out, answers(lambda v: fn(v, 2.0, W3, **kw), pool), counts(SHAPE3, TILE3), 1, what=op)


@pytest.mark.parametrize("op", ["erode", "dilate"])
@released
def test_parabolic_beyond_2_31(edt, op):
  """parabolic_erode / _dilate of 528 x 2048 x 2048 samples whose walls hold the least (greatest) value."""
  need(21)                                   # measured peak: 18.4 GB
  pool = torch.from_numpy(lc.value_pool(np.random.default_rng(15), K, TILE3, 1, op)).cuda()
  f = lc.assemble(pool, counts(SHAPE3, TILE3))
  fn = getattr(edt, "parabolic_" + op)
  out = fn(f, W3)
  lc.assert_tiles(out, answers(lambda v: fn(v, W3), pool), counts(SHAPE3, TILE3), 1, what=op)


@released
def test_parabolic_sites_beyond_2_31(edt):
  """parabolic_erode(return_indices=True) on a 46368^2 image: values and translated sites."""
  # measured peak: 64.1 GB.  Lines of 46368 samples exceed kParabolicExactN = 23170, so both passes run the
  # brute-force site kernel, O(n^2) per line: this test takes about 280 s of the file's 320 s on an H100
  need(68)
  pool = torch.from_numpy(lc.value_pool(np.random.default_rng(16), K, TILE2, 1, "erode")).cuda()
  f = lc.assemble(pool, counts(SHAPE2, TILE2))
  out, idx = edt.parabolic_erode(f, W2, return_indices=True)
  del f
  small = [edt.parabolic_erode(pool[k], W2, return_indices=True) for k in range(K)]
  cn = counts(SHAPE2, TILE2)
  lc.assert_tiles(out, torch.stack([s[0] for s in small]), cn, 1, what="values")
  lc.assert_tiles(idx, torch.stack([s[1] for s in small]), cn, 1, sites=True, what="sites")


@pytest.mark.parametrize("k", [1, 2])
@released
def test_nearest_labels_beyond_2_31(edt, k):
  """nearest_labels at max_distance 2.5 on a 46368^2 image of one-byte labels with walls of 3."""
  need({1: 25, 2: 45}[k])                    # measured peaks: 22.1 and 42.1 GB
  pool, lab = labels_of(SHAPE2, TILE2, 3, np.uint8, 17)
  dist, near = edt.nearest_labels(lab, 2.5, W2, k=k)
  del lab
  small = [edt.nearest_labels(pool[j], 2.5, W2, k=k) for j in range(K)]
  cn = counts(SHAPE2, TILE2)
  lc.assert_tiles(dist, torch.stack([s[0] for s in small]), cn, 3, what="distances k=%d" % k)
  lc.assert_tiles(near, torch.stack([s[1] for s in small]), cn, 3, what="labels k=%d" % k)


@released
def test_medial_axis_beyond_2_31(edt):
  """medial_axis(return_distance=True) on 528 x 2048 x 2048 one-byte labels (integer weights)."""
  need(50)                                   # measured peak: 46.5 GB
  pool, lab = labels_of(SHAPE3, TILE3, 1, np.uint8, 18)
  medial, dist = edt.medial_axis(lab, W3, return_distance=True)
  del lab
  small = [edt.medial_axis(pool[k], W3, return_distance=True) for k in range(K)]
  cn = counts(SHAPE3, TILE3)
  lc.assert_tiles(medial, torch.stack([s[0] for s in small]), cn, 1, what="medial")
  lc.assert_tiles(dist, torch.stack([s[1] for s in small]), cn, 1, what="distances")


# ---- one volume past 2^32 voxels: the Z pass on the long-line kernel --------------------------------

@pytest.mark.parametrize("dtype", ["uint8", "uint32"])
@released
def test_transforms_beyond_2_32(edt, dtype):
  """edt_cuda unsigned and sdf on 1040 x 2048 x 2048 labels of 1 and 4 bytes: n * line_stride of the Z
  pass is past 2^32, beyond the tile kernel's 32-bit offsets, so the Z pass runs on the long-line kernel."""
  need({"uint8": 57, "uint32": 69}[dtype])   # measured peaks: 53.7 and 65.9 GB
  # uint32 labels are assembled as int32 (wall -1, i.e. 0xffffffff) and viewed
  pool, lab = labels_of(SHAPE4G, TILE3, 1, np.uint8 if dtype == "uint8" else np.int32, 19)
  pool, lab = pool.view(getattr(torch, dtype)), lab.view(getattr(torch, dtype))
  assert lab.numel() >= 2**32
  out = torch.empty(SHAPE4G, dtype=torch.float32, device="cuda")
  for border, sqrt, signed in ((True, False, False), (False, True, True)):
    edt.edt_cuda(lab, W3, border, sqrt=sqrt, signed=signed, out=out)
    ran("edt_cuda %s sqrt=%s signed=%s" % (dtype, sqrt, signed), lab.numel())
    assert RAN[-1][1] == "long", RAN[-1]
    want = answers(lambda v: edt.edt_cuda(v, W3, border, sqrt=sqrt, signed=signed), pool)
    lc.assert_tiles(out, want, counts(SHAPE4G, TILE3), 1, what="sqrt=%s signed=%s" % (sqrt, signed))


# ---- stacks whose flat index passes 2^31 and 2^32 ---------------------------------------------------

def check_stack(got, want, vnd, what):
  """got: lead + (count,) + volume; want: (K,) + lead + volume; vnd: the volume's dimensions."""
  lc.assert_stack(got, want, got.dim() - vnd - 1, what)


STACK31 = 140000                                             # x 128^2: 2.29e9 voxels


@pytest.mark.parametrize("op", ["edt", "feature_transform", "feature_indices", "expand_labels", "parabolic_erode", "nearest_labels",
                                "medial_axis", "spherical_open"])
@released
def test_stack_beyond_2_31(edt, op):
  """140000 volumes of 128^2, each the single-volume call on its variant."""
  # measured peaks: 12.7, 64.0, 64.0, 64.1, 59.9, 46.9, 40.5 and 17.0 GB
  need({"edt": 15, "feature_transform": 67, "feature_indices": 67, "expand_labels": 67, "parabolic_erode": 63, "nearest_labels": 50,
        "medial_axis": 43, "spherical_open": 19}[op])
  rng = np.random.default_rng(20)
  if op == "parabolic_erode":
    pool = torch.from_numpy(lc.value_pool(rng, K, (128, 128), 0, "erode")).cuda()
  else:
    pool = torch.from_numpy(lc.label_pool(rng, K, (128, 128), 0, np.uint8)).cuda()
  st = stack_of(pool, STACK31)
  assert st.numel() > 2**31
  w = (2.0, 1.0)
  calls = {
    "edt": lambda v, s: (edt.edt_cuda(v, w, True, sqrt=True, stacked=s),),
    "feature_transform": lambda v, s: edt.feature_transform(v, w, return_distances=True, stacked=s),
    "feature_indices": lambda v, s: (edt.feature_transform(v, w, stacked=s),),
    "expand_labels": lambda v, s: (edt.expand_labels(v, 2.5, w, stacked=s),),
    "parabolic_erode": lambda v, s: edt.parabolic_erode(v, w, return_indices=True, stacked=s),
    "nearest_labels": lambda v, s: edt.nearest_labels(v, 2.5, w, k=2, stacked=s),
    "medial_axis": lambda v, s: edt.medial_axis(v, w, return_distance=True, stacked=s),
    "spherical_open": lambda v, s: (edt.spherical_open(v, 2.0, w, True, stacked=s),),
  }[op]
  got = calls(st, True)
  if op in ("edt", "spherical_open"):
    ran("stacked " + op, st.numel())
  del st
  small = [calls(pool[k], False) for k in range(K)]
  for j, g in enumerate(got):
    check_stack(g, torch.stack([s[j] for s in small]), 2, "%s output %d" % (op, j))


@released
def test_stack_surface_distances_beyond_2_31(edt):
  """surface_distances of two stacks of 140000 volumes of 128^2 whose surfaces are few voxels (large
  boxes, b = a with a few voxels relabelled), so the values stay small while the flat index passes 2^31:
  every volume's segments are its variant pair's, bit for bit."""
  need(17)                                   # measured peak: 14.5 GB (1.18e8 distances)
  pa, pb = (torch.from_numpy(p).cuda() for p in lc.block_pool(np.random.default_rng(21), K, (128, 128), np.uint8))
  keys = np.arange(1, 6, dtype=np.uint8)
  a, b = stack_of(pa, STACK31), stack_of(pb, STACK31)
  assert a.numel() > 2**31
  got = edt.surface_distances(a, b, (2.0, 1.0), labels=keys, stacked=True)
  del a, b
  nseg = 2 * keys.size
  lens = got.offsets.diff().view(STACK31, nseg)
  assert int(got.offsets[-1]) == got.values.numel() > 0
  for k in range(K):
    want = edt.surface_distances(pa[k], pb[k], (2.0, 1.0), labels=keys)
    vols = torch.arange(k, STACK31, K, device="cuda")
    assert bool((lens[vols] == want.offsets.diff().view(1, nseg)).all()), k
    n = want.values.numel()
    step = max(1, (1 << 26) // max(1, n))       # volumes compared at a time
    for v0 in range(0, vols.numel() if n else 0, step):
      at = got.offsets[vols[v0:v0 + step] * nseg].view(-1, 1) + torch.arange(n, device="cuda").view(1, -1)
      bad = int((got.values[at].view(torch.int32) != want.values.view(1, -1).view(torch.int32)).sum())
      assert bad == 0, "variant %d: %d distances differ" % (k, bad)
  print("\n%d surface distances" % got.values.numel())


STACK32 = 260                                                # x 256^3: 4.36e9 voxels


@pytest.mark.parametrize("op", ["edt", "spherical_open"])
@released
def test_stack_beyond_2_32(edt, op):
  """260 volumes of 256^3 (a Z pass of n = 256 on the tile kernel, flat indices past 2^32)."""
  need({"edt": 25, "spherical_open": 48}[op])     # measured peaks: 22.5 and 44.8 GB
  pool = torch.from_numpy(lc.label_pool(np.random.default_rng(22), K, (256, 256, 256), 0, np.uint8)).cuda()
  st = stack_of(pool, STACK32)
  assert st.numel() >= 2**32
  if op == "edt":
    fn = lambda v, s: edt.edt_cuda(v, W3, False, sqrt=True, signed=True, stacked=s)
  else:
    fn = lambda v, s: edt.spherical_open(v, 2.0, W3, True, stacked=s)
  got = fn(st, True)
  ran("stacked %s 2^32" % op, st.numel())
  del st
  check_stack(got, answers(lambda v: fn(v, False), pool), 3, op)


def test_kernel_coverage():
  """The tile and window kernels ran past 2^31 voxels, and the long-line kernel past 2^32."""
  print("\n" + "\n".join("%-50s %-6s %.2e" % r for r in RAN))
  kinds = {(kernel, n >= 2**32) for _, kernel, n in RAN if n > 2**31}
  assert ("tile", False) in kinds or ("tile", True) in kinds, RAN
  assert any(kernel == "window" for kernel, _ in kinds), RAN
  assert ("long", True) in kinds, RAN
