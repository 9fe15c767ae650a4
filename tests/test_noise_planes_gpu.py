"""GPU tests (-m gpu) of the plane-writing X pass (first_axis_planes_kernel) word by word: through
edtb200_noise_planes, f as bits and every word of the run-start and settled planes against the
restatement of tests/noise_planes_cases.py, exactly -- in every instance the transform can launch,
at every chunk count a slice may be cut into, on grids with fewer CTAs than items, and after the Y
pass that reads the planes, skips settled tiles and refreshes the Z pass's settled plane.

Every word of the planes buffer and every distance starts as a sentinel, so a word the kernel leaves
unwritten fails; the words past the buffer must keep theirs.  The instances and march shapes reached
are collected in HIT and BEYOND, and the last test fails if a reachable one was never run.
"""
import ctypes

import numpy as np
import pytest

import noise_cases as nc
import noise_planes_cases as npc
from test_first_axis_gpu import change_rows, later_ctas
from test_run_planes_gpu import runs_volume

pytestmark = pytest.mark.gpu

INFO = ("label_bytes", "k", "plain", "planes", "nchunks", "items", "grid", "reads", "settled", "refresh")
SQRT = 1
DTYPES = (np.uint32, np.int32, np.uint64, np.int64)
TORCH_VIEW = {4: np.int32, 8: np.int64}
GUARD = 64                                   # sentinel words past f and past the planes
F_SENTINEL = np.uint32(0x7fc0dead)           # a NaN no pass writes
P_SENTINEL = np.uint32(0xa5a5a5a5)
SXS = (4, 36, 128, 132, 256, 260, 508, 512)
DEPTHS = (1, 3, 6, 8, 9, 17)
WEIGHTS = [(1.0, 1.0, 1.0), (1.0, 2.0, 3.0), (1.5, 1.0, 2.5), (1.0, 2.0, 1.0), (1.0, 2.0, 2.0),
           (1.0, 1.33355, 1.33355), (1.33355, 1.0, 0.5), (2.0, 1.0, 3.0)]
HIT = set()          # (label bytes, K, planes) of every run
BEYOND = set()       # (label bytes, planes, nst < S) of runs with more items than CTAs
PLANS = set()        # (reads, settled, refresh) of the Y passes run


def run(edt, lab, ndim, w, border, passes=1, nchunks=0, ctas=0, flags=0):
  """edtb200_noise_planes on lab ((count, sz, sy, sx) or (count, sy, sx)): (f, planes, info)."""
  import torch
  vol, depth = npc.slices(lab, ndim)
  n, sy, sx = vol.shape
  count = lab.shape[0]
  flat = np.ascontiguousarray(lab).reshape(-1)
  lab_t = torch.from_numpy(flat.view(TORCH_VIEW[flat.dtype.itemsize])).cuda()
  words = npc.buffer_words(sx, sy, n * sy, ndim)
  f_t = torch.from_numpy(np.full(flat.size + GUARD, F_SENTINEL).view(np.int32)).cuda()
  p_t = torch.from_numpy(np.full(words + GUARD, P_SENTINEL).view(np.int32)).cuda()
  info = (ctypes.c_int * len(INFO))()
  lib = edt._lib()
  wxyz = [float(v) for v in w] + [1.0] * (3 - len(w))      # the weight of a missing axis is not read
  rc = lib.edtb200_noise_planes(lab_t.data_ptr(), flat.dtype.itemsize, ndim, sx, sy, depth if ndim == 3 else 1,
                                count, *wxyz, int(border), flags, passes, nchunks, ctas, f_t.data_ptr(),
                                p_t.data_ptr(), ctypes.cast(info, ctypes.c_void_p), 0, ctypes.c_void_p(None))
  assert rc == 0, lib.edtb200_last_error()
  torch.cuda.synchronize()
  f = f_t.cpu().numpy().view(np.uint32)
  planes = p_t.cpu().numpy().view(np.uint32)
  got = dict(zip(INFO, (int(v) for v in info)))
  assert np.all(f[flat.size:] == F_SENTINEL), "the pass wrote past f"
  assert np.all(planes[words:] == P_SENTINEL), "the pass wrote past the planes"
  assert got["label_bytes"] == flat.dtype.itemsize and got["plain"] == 1 and got["planes"] == ndim - 1, got
  assert got["k"] == (1 if sx <= 128 else 2 if sx <= 256 else 4), got
  HIT.add((got["label_bytes"], got["k"], got["planes"]))
  if got["items"] > got["grid"]:
    nst = -(-sy // got["nchunks"]) + 2
    BEYOND.add((got["label_bytes"], got["planes"], nst < (3 if got["label_bytes"] == 8 else 4)))
  return f[:flat.size].view(np.float32).reshape(n, sy, sx), planes[:words], got


def assert_words(got, want, what):
  if not np.array_equal(got, want):
    bad = np.argwhere(got != want)
    first = tuple(bad[0])
    raise AssertionError("%s: %d words differ; first at %s: got %#x want %#x" % (
      what, len(bad), first, int(got[first]), int(want[first])))


def check(edt, oracle, lab, ndim, w, border, passes=1, nchunks=0, ctas=0, flags=0, x=None, what=()):
  """One run against the restatement (x: the X pass's, when known); returns (info, x)."""
  vol, _ = npc.slices(lab, ndim)
  n, sy, sx = vol.shape
  what = tuple(what) + (lab.dtype.name, lab.shape, ndim, w, border, passes, nchunks, ctas, flags)
  f, planes, info = run(edt, lab, ndim, w, border, passes, nchunks, ctas, flags)
  if x is None:
    x = npc.restate(oracle, lab, ndim, w, border)
  want = x
  if passes == 2:
    assert info["reads"] == (sx >= 32), (what, info)
    if info["reads"]:
      nc.assert_planes_plan(edt, info["settled"])
    PLANS.add((info["reads"], info["settled"], info["refresh"]))
    want = npc.restate_after_y(oracle, lab, ndim, w, border, x, sqrt=bool(flags & SQRT) and ndim == 2,
                               refreshes=bool(info["refresh"]))
  assert_words(f.view(np.uint32), want["f"].view(np.uint32), what + ("f",))
  got = npc.split(planes, sx, sy, n * sy, ndim)
  for name in want:
    if name != "f":
      assert_words(got[name], want[name], what + (name,))
  if passes == 2 and ndim == 3:
    assert np.all(got["settled_z"] & x["settled_z"] == x["settled_z"]), what     # only bits that were clear are set
    tz = npc.square(w[2])
    words = got["settled_z"].reshape(n, sy)
    for s in range(npc.wpr(sx)):
      on = (words >> np.uint32(s)) & 1 == 1
      assert np.all(want["f"][:, :, s * npc.SEG:(s + 1) * npc.SEG][on] <= tz), (what, s)   # every set bit is true
  return info, x


def volume(kind, shape, dtype, seed):
  """Labels of one pattern: noise, planted_rows, runs (runs_volume) or a settled pattern."""
  if kind == "noise":
    return nc.noise(shape, dtype, seed)
  if kind == "planted":
    return nc.planted_rows(shape, dtype, seed)
  if kind == "runs":                         # runs along y, and along z through the whole stack
    return runs_volume((int(np.prod(shape[:-2])),) + shape[-2:], dtype, seed).reshape(shape)
  return npc.settled_pattern(shape, dtype, np.random.default_rng(seed), kind)


KINDS = ("noise", "planted", "runs", "all", "none", "some")


@pytest.mark.parametrize("dtype", DTYPES, ids=[d.__name__ for d in DTYPES])
def test_widths_shapes_and_patterns(edt, oracle, dtype):
  """Every row length of SXS (K = 1..4, the last word full or partial), 2-D stacks and 3-D stacks of
  volumes of every depth of DEPTHS, the patterns, weights and borders taking turns; the X pass alone
  and with the Y pass."""
  for i, sx in enumerate(SXS):
    for j, (ndim, shape) in enumerate(((2, (5, 11, sx)), (3, (2, DEPTHS[i % 6], 13, sx)),
                                       (3, (3, DEPTHS[(i + 3) % 6], 6, sx)))):
      seed = 1000 * i + 10 * j + dtype().itemsize
      lab = volume(KINDS[(i + j) % len(KINDS)], shape, dtype, seed)
      w = WEIGHTS[(i + 2 * j) % len(WEIGHTS)]
      border = (i + j) % 2
      _, x = check(edt, oracle, lab, ndim, w, border)
      check(edt, oracle, lab, ndim, w, border, passes=2, x=x, flags=SQRT if (i + j) % 4 == 3 else 0)


@pytest.mark.parametrize("sy", (2, 3, 7, 67, 134, 201, 400))
def test_every_chunk_count(edt, oracle, sy):
  """Every chunk count from 1 to sy (chunks of one row) on volumes planted at every chunk cut, 2-D and
  3-D, 4- and 8-byte labels; the count the launch picks itself; the Y pass after 1, 2, 3, that count
  and sy chunks."""
  for ndim, shape, dtype in ((3, (1, 9, sy, 132), np.uint32), (2, (6, sy, 36), np.int64)):
    lab = nc.planted_rows(shape, dtype, sy + ndim)
    w, border = ((1.0, 1.0, 2.0), 0) if ndim == 3 else ((1.0, 2.0), 1)
    info, x = check(edt, oracle, lab, ndim, w, border, what=("own count",))
    own = info["nchunks"]
    assert 1 <= own <= max(1, sy * 3 // 200), info
    for n in range(1, sy + 1):
      check(edt, oracle, lab, ndim, w, border, nchunks=n, x=x)
    for n in sorted({1, min(2, sy), min(3, sy), own, sy}):
      check(edt, oracle, lab, ndim, w, border, passes=2, nchunks=n, x=x)


def test_more_items_than_ctas(edt, oracle):
  """Grids of 1, 2, 3 and items - 1 CTAs, so that CTAs march item after item: the ring slot and
  phase carried over, and the prefetch of the next item's stages while the last ones are read (sy = 1
  and 2: fewer stages per item than the ring holds); 3-D and 2-D stacks, 4- and 8-byte labels."""
  cases = []
  for dtype in (np.uint32, np.int64):
    for sy in (1, 2, 5, 67):
      cases.append((3, (7, 3, sy, 132), dtype))
      cases.append((2, (41, sy, 260), dtype))
  for k, (ndim, shape, dtype) in enumerate(cases):
    lab = volume(("planted", "runs", "noise")[k % 3], shape, dtype, 77 + k)
    sy = shape[-2]
    w, border = WEIGHTS[k % len(WEIGHTS)], k % 2
    x = npc.restate(oracle, lab, ndim, w, border)
    for nchunks in sorted({1, min(2, sy), sy}):
      items = (-(-shape[0] * shape[1] // nc.BAND) * nchunks if ndim == 3 else -(-shape[0] * nchunks // nc.BAND))
      for ctas in sorted({c for c in (1, 2, 3, items - 1) if 1 <= c < items}):
        info, _ = check(edt, oracle, lab, ndim, w, border, nchunks=nchunks, ctas=ctas, x=x)
        assert info["items"] == items and info["grid"] == ctas, info
      if items > 1:
        check(edt, oracle, lab, ndim, w, border, passes=2, nchunks=nchunks, ctas=1, x=x)


@pytest.mark.parametrize("ndim", (2, 3))
def test_weights_and_borders(edt, oracle, ndim):
  """Integer and non-integer weights, w_z below, equal to and above w_y, a weight whose square rounds
  in float32 (1.33355), both borders, the X pass and the Y pass, sqrt in the last pass."""
  shape = (2, 5, 20, 132) if ndim == 3 else (4, 20, 132)
  for k, kind in enumerate(("planted", "runs", "some")):
    lab = volume(kind, shape, np.uint32 if k % 2 else np.int64, 500 + k)
    for w in WEIGHTS:
      for border in (0, 1):
        _, x = check(edt, oracle, lab, ndim, w, border)
        for flags in (0, SQRT):
          check(edt, oracle, lab, ndim, w, border, passes=2, flags=flags, x=x)


def test_run_statistic_equals_the_plain_kernels(edt, oracle):
  """The run statistic the planes kernel publishes steers the next tile pass as the plain X kernel's
  does, at 0.90 and 0.89 label changes per voxel (the edge of label noise), 2-D and 3-D; so the
  planes kernel counts every row's changes once, its leading and trailing rows not again."""
  import torch
  rng = np.random.default_rng(61)
  for ndim, nrows in ((2, 40), (3, 9 * 12)):
    for changes, ctas in ((90, 2), (89, 3)):
      rows = change_rows(rng, 100, nrows, changes)
      lab = rows.reshape((1, 9, 12, 100) if ndim == 3 else (1, nrows, 100))
      for nchunks in (0, 3):
        check(edt, oracle, lab, ndim, (1.0, 1.0, 1.0), 0, nchunks=nchunks, what=("stat",))
        assert later_ctas(edt, oracle, rng) == ctas, (ndim, changes, nchunks, "planes kernel")
      lab_t = torch.from_numpy(rows.view(np.int32)).cuda()
      f_t = torch.empty(rows.size, dtype=torch.float32, device="cuda")
      lib = edt._lib()
      assert lib.edtb200_pass_first(lab_t.data_ptr(), 4, 100, nrows, 1, 1.0, 0, 0, f_t.data_ptr(), 0,
                                    ctypes.c_void_p(None)) == 0, lib.edtb200_last_error()
      torch.cuda.synchronize()
      assert later_ctas(edt, oracle, rng) == ctas, (ndim, changes, "vector kernel")


@pytest.fixture(autouse=True)
def _record_run(request):
  yield
  RAN.add(request.node.originalname)


RAN = set()
PRODUCERS = {"test_widths_shapes_and_patterns", "test_every_chunk_count", "test_more_items_than_ctas",
             "test_weights_and_borders"}


def test_every_instance_and_march_was_run():
  """Every (label bytes, K, planes) the transform can launch the planes kernel with, runs with more
  items than CTAs for both label widths and plane counts (with fewer stages per item than the ring
  holds among them), and Y passes that skipped settled tiles and refreshed settled_z.  Meaningful
  only after the tests above have run in this process; skipped otherwise."""
  if not PRODUCERS <= RAN:
    pytest.skip("the producing tests of this file did not run before this one: %s" % sorted(PRODUCERS - RAN))
  want = {(b, k, p) for b in (4, 8) for k in (1, 2, 4) for p in (1, 2)}
  print("\nplanes kernel instances run (%d of %d):" % (len(HIT & want), len(want)), sorted(HIT))
  print("more items than CTAs:", sorted(BEYOND))
  print("Y pass plans (reads, settled, refresh):", sorted(PLANS))
  assert HIT == want, (sorted(want - HIT), sorted(HIT - want))
  assert {(b, p) for b, p, _ in BEYOND} == {(b, p) for b in (4, 8) for p in (1, 2)}, sorted(BEYOND)
  assert any(short for _, _, short in BEYOND), sorted(BEYOND)
  assert {(0, 0, 0), (1, 0, 0), (1, 1, 1), (1, 1, 0)} <= PLANS, sorted(PLANS)
