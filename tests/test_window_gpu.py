"""GPU tests (-m gpu) of the bounded transforms' window kernel (edt_bounded.cuh).

One pass at a time through edtb200_pass_window, against the restatement of tests/window_cases.py bit for
bit, distances and site codes, at every radius up to the kernel's launch limit of 128 rows, across the
edges of its 64-row by 32-line tiles; which variant ran (label bytes, sites, epilogue, exact arithmetic) is
collected in HIT and the last test fails if one was never run.

Then whole calls with every later pass forced onto the window (EDTB200_BOUNDED_RMAX=128, read on every
call): the bounded transforms against the oracle's unbounded transform cut at B, the bounded feature
transform against the site contract, the spherical morphology (the select kernel) against
morphology_cases, and all of them against the same calls with no pass windowed (EDTB200_BOUNDED_RMAX=-1).
"""
import ctypes
import math

import numpy as np
import pytest

import morphology_cases as mc
import window_cases as wc
from feature_cases import check_sites

pytestmark = pytest.mark.gpu

WIDTHS = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}
LENGTHS = (1, 2, 63, 64, 65, 127, 128, 129, 200, 257)
LINES = (1, 31, 32, 33, 65)
RADII = (0, 1, 2, 3, 31, 32, 33, 63, 64, 65, 127, 128)
WEIGHTS = (1.0, 0.7, 2.5, 1.333549976348877)
BORDERS = ((0, 0), (1, 0), (0, 1), (1, 1))
FLAGS = (0, wc.SQRT, wc.SIGNED, wc.SQRT | wc.SIGNED)
HIT = set()            # (label bytes, sites, epilogue, exact arithmetic)
RADII_RUN = set()


def geometry(n, lines, axis):
  """A (z, y, x) shape whose pass along `axis` has lines of n rows, `lines` of them side by side."""
  if axis == 1:
    return (2 if lines <= 33 else 1, n, lines)
  sy, sx = {1: (1, 1), 31: (1, 31), 32: (4, 8), 33: (3, 11), 65: (5, 13)}[lines]
  return (n, sy, sx)


def run_window(edt, lab, f, axis, w, d, lo, hi, flags, sites):
  """edtb200_pass_window on C-ordered (z, y, x) arrays: (fout, codes or None, the launch)."""
  import torch
  lab = np.ascontiguousarray(lab)
  nbytes = lab.dtype.itemsize
  lt = torch.from_numpy(lab.view(np.dtype("i%d" % nbytes) if nbytes > 1 else np.uint8)).cuda()
  fin = torch.from_numpy(np.ascontiguousarray(f, dtype=np.float32)).cuda()
  fout = torch.full_like(fin, float("nan"))
  codes = torch.full(fin.shape, 7, dtype=torch.int32, device="cuda") if sites else None
  sz, sy, sx = lab.shape
  lib = edt._lib()
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  rc = lib.edtb200_pass_window(lt.data_ptr(), nbytes, axis, sx, sy, sz, float(w), int(lo), int(hi), flags, float(d),
                               fin.data_ptr(), fout.data_ptr(), codes.data_ptr() if sites else None, 0, stream)
  assert rc == 0, lib.edtb200_last_error()
  torch.cuda.synchronize()
  v = edt.last_later_launch()
  assert v["kernel"] == "window" and v["epilogue"] == int(flags != 0), v
  HIT.add((nbytes, bool(sites), bool(flags), v["all_double"] == 0))
  RADII_RUN.add(v["tx"])
  return fout.cpu().numpy(), (codes.cpu().numpy() if sites else None), v


def check_window(edt, lab, f, axis, w, d, lo, hi, flags, sites, what):
  got, codes, v = run_window(edt, lab, f, axis, w, d, lo, hi, flags, sites)
  assert v["tx"] == wc.plan(w, d)[1], (what, v)
  want = wc.window_pass(lab, f, axis, w, d, lo, hi, flags)
  bad = got.view(np.uint32) != want.view(np.uint32)
  if bad.any():
    first = tuple(np.argwhere(bad)[0])
    raise AssertionError("%s %s: %d voxels differ; first at %s: got %r want %r" % (
      what, v, int(bad.sum()), first, got[first], want[first]))
  if sites:
    wc.check_codes(lab, f, axis, w, d, lo, hi, codes)
  return v


@pytest.mark.parametrize("nbytes", sorted(WIDTHS))
def test_pass_every_length_and_radius(edt, nbytes):
  """Every pass length against every radius: partial last row tiles with large halos, halos longer than
  the line (R >= n) and halos crossing two row tiles (R > 64), with 1, 31, 32, 33 and 65 lines across."""
  rng = np.random.default_rng(300 + nbytes)
  k = 0
  for n in LENGTHS:
    for r in RADII:
      k += 1
      axis = 1 + k % 2
      lines = LINES[(k // 2) % len(LINES)]
      w = WEIGHTS[k % len(WEIGHTS)]
      kind = wc.PROFILES[k % len(wc.PROFILES)]
      labeling = ("one_run", "runs", "specks")[(k // 3) % 3]
      flags = FLAGS[(k // 4) % 4]
      sites = (k // 5) % 2 == 0
      lo, hi = BORDERS[(k // 7) % 4]
      shape = geometry(n, lines, axis)
      d, b = wc.distance_for(w, r)
      lab = wc.labels(rng, labeling, shape, axis, WIDTHS[nbytes])
      f = wc.profile(rng, kind, shape, axis, w, r, b)
      check_window(edt, lab, f, axis, w, d, lo, hi, flags, sites,
                   (nbytes, n, r, axis, lines, w, kind, labeling, flags, sites, lo, hi))


@pytest.mark.parametrize("nbytes", sorted(WIDTHS))
def test_pass_every_variant(edt, nbytes):
  """Each (sites, epilogue, arithmetic) variant on the adversarial lines: winners at R and R + 1 rows,
  heights at B and next to it, border terms tied with samples, the ends of every window tile."""
  rng = np.random.default_rng(400 + nbytes)
  for sites in (False, True):
    for flags in FLAGS:
      for kind, w in (("sparse", 1.0), ("tiny", 0.7), ("at_bound", 2.5), ("border_ties", 1.0), ("tile_edges", 0.7),
                      ("real", 1.333549976348877)):
        for r, n, axis, lines in ((3, 200, 2, 33), (64, 257, 1, 65), (128, 200, 2, 32)):
          lo, hi = BORDERS[(r + len(kind)) % 4]
          shape = geometry(n, lines, axis)
          d, b = wc.distance_for(w, r)
          lab = wc.labels(rng, ("one_run", "runs", "specks")[r % 3], shape, axis, WIDTHS[nbytes])
          f = wc.profile(rng, kind, shape, axis, w, r, b)
          check_window(edt, lab, f, axis, w, d, lo, hi, flags, sites, (nbytes, sites, flags, kind, r))


def test_pass_high_label_bits(edt):
  """8-byte labels 1 and 1 + 2^40 in alternating runs: the runs end where only the high bits change."""
  rng = np.random.default_rng(9)
  for r in (2, 33, 128):
    d, b = wc.distance_for(1.0, r)
    shape = (129, 4, 8)
    lab = np.broadcast_to(np.where((np.arange(129) // 7) % 2 == 1, np.uint64(1 + (1 << 40)), np.uint64(1))
                          .reshape(-1, 1, 1), shape).copy()
    f = wc.profile(rng, "sparse", shape, 2, 1.0, r, b)
    check_window(edt, lab, f, 2, 1.0, d, 0, 0, 0, True, ("high bits", r))
    low = lab.astype(np.uint32).astype(np.uint64)                     # what the low bits alone would give
    assert not np.array_equal(wc.window_pass(low, f, 2, 1.0, d, 0, 0), wc.window_pass(lab, f, 2, 1.0, d, 0, 0))


def test_pass_bound_edges(edt):
  """Own-row heights at B, one float32 either side of it and +inf: kept, cut, kept, +inf."""
  for w in (1.0, 0.7):
    for r in (0, 1, 32, 128):
      d, b = wc.distance_for(w, r)
      above, below = np.nextafter(b, np.float32(np.inf)), np.nextafter(b, np.float32(0))
      col = np.array([b, above, below, np.inf] * 20, np.float32)
      f = np.ascontiguousarray(np.broadcast_to(col.reshape(-1, 1, 1), (80, 2, 16)))
      lab = np.ones(f.shape, np.uint32)
      got, _, _ = run_window(edt, lab, f, 2, w, d, 0, 0, 0, False)
      if r == 0:
        assert np.array_equal(got[:4, 0, 0], [b, np.inf, below, np.inf]), (w, r, got[:4, 0, 0])
      check_window(edt, lab, f, 2, w, d, 0, 0, 0, True, ("bound edges", w, r))


# ---- whole calls with every later pass windowed ------------------------------------------------------

FUNCS = {"edtsq": (False, False), "edt": (True, False), "sdfsq": (False, True), "sdf": (True, True)}
SHAPES = {2: (150, 131), 3: (20, 37, 140)}


def volume(rng, shape, order):
  """Blocky labels with background, long runs along every axis and a few specks."""
  small = rng.integers(0, 4, tuple(max(1, s // 9) + 1 for s in shape))
  lab = small
  for ax, s in enumerate(shape):
    lab = np.repeat(lab, 9, axis=ax).take(np.arange(s), axis=ax)
  lab = (lab * (rng.random(shape) > 0.003)).astype(np.uint16)
  return np.asfortranarray(lab) if order == "F" else np.ascontiguousarray(lab)


def same_bits(a, b):
  a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
  return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def cut(unbounded, sq, d):
  sq = np.asarray(sq, np.float32)
  keep = np.abs(sq).astype(np.float64) <= d * d
  return np.where(keep, unbounded, np.where(np.signbit(sq), -np.inf, np.inf)).astype(np.float32)


def whole_radii(nd):
  return RADII if nd == 2 else (0, 1, 3, 33, 65, 128)


def later_radius(arr, w, d):
  """R of the last later pass (the slowest axis in memory)."""
  ax = 0 if arr.flags.c_contiguous and not arr.flags.f_contiguous else arr.ndim - 1
  return wc.plan(w[ax], d)[1]


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("nd", [2, 3])
def test_transforms_windowed(edt, oracle, monkeypatch, nd, order):
  rng = np.random.default_rng(nd * 10 + (order == "F"))
  arr = volume(rng, SHAPES[nd], order)
  w = (1.0,) * nd
  for bb in (False, True):
    sq = {s: (oracle.sdfsq(arr, w, bb) if s else oracle.edtsq(arr, w, bb)) for s in (False, True)}
    unb = {fn: getattr(oracle, fn)(arr, w, bb) for fn in FUNCS}
    for r in whole_radii(nd):
      d = float(r)
      for fn, (_, signed) in FUNCS.items():
        monkeypatch.setenv("EDTB200_BOUNDED_RMAX", "128")
        got = np.asarray(getattr(edt, fn)(arr, anisotropy=w, black_border=bb, max_distance=d))
        launch = edt.last_later_launch()
        assert launch["kernel"] == "window" and launch["tx"] == r, (fn, r, launch)
        assert same_bits(got, cut(unb[fn], sq[signed], d)), (fn, bb, r)
        monkeypatch.setenv("EDTB200_BOUNDED_RMAX", "-1")
        other = np.asarray(getattr(edt, fn)(arr, anisotropy=w, black_border=bb, max_distance=d))
        assert edt.last_later_launch()["kernel"] != "window"
        assert same_bits(other, got), (fn, bb, r)


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("nd", [2, 3])
def test_transforms_windowed_anisotropic(edt, oracle, monkeypatch, nd, order):
  """Real and dyadic weights: every later axis has its own radius, up to 128."""
  rng = np.random.default_rng(nd * 20 + (order == "F"))
  arr = volume(rng, SHAPES[nd], order)
  for w in ((0.7, 1.3, 2.5)[:nd], (0.5, 1.25, 1.0)[:nd]):
    sq = oracle.sdfsq(arr, w, True)
    unb = oracle.sdf(arr, w, True)
    for d in (0.6, 2.6, 40.3, 63.9 * min(w)):
      monkeypatch.setenv("EDTB200_BOUNDED_RMAX", "128")
      got = np.asarray(edt.sdf(arr, anisotropy=w, black_border=True, max_distance=d))
      assert edt.last_later_launch()["tx"] == later_radius(arr, w, d)
      assert same_bits(got, cut(unb, sq, d)), (w, d)
      monkeypatch.setenv("EDTB200_BOUNDED_RMAX", "-1")
      assert same_bits(edt.sdf(arr, anisotropy=w, black_border=True, max_distance=d), got), (w, d)


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("nd", [2, 3])
def test_feature_transform_windowed(edt, oracle, monkeypatch, nd, order):
  rng = np.random.default_rng(nd * 30 + (order == "F"))
  shape = {2: (70, 133), 3: (12, 30, 131)}[nd]
  arr = volume(rng, shape, order)
  w = (1.0,) * nd
  for signed in (False, True):
    for bb in (False, True):
      sq = oracle.sdfsq(arr, w, bb) if signed else oracle.edtsq(arr, w, bb)
      udist, uidx = (np.asarray(a) for a in edt.feature_transform(arr, w, bb, signed=signed, return_distances=True))
      inside_any = False
      for r in (0, 2, 33, 65, 128):
        d = float(r)
        monkeypatch.setenv("EDTB200_BOUNDED_RMAX", "128")
        dist, idx = (np.asarray(a) for a in edt.feature_transform(arr, w, bb, signed=signed, return_distances=True,
                                                                   max_distance=d))
        launch = edt.last_later_launch()
        assert launch["kernel"] == "window" and launch["tx"] == r, (r, launch)
        assert same_bits(dist, cut(udist, sq, d)), (signed, bb, r)
        inside = np.abs(sq).astype(np.float64) <= d * d
        inside_any |= bool((inside & (np.abs(sq) > 0)).any())
        assert (idx[:, ~inside] == -1).all(), "a site outside the band"
        check_sites(arr, np.where(inside[None], idx, uidx), np.abs(sq), w, bb, signed)
        monkeypatch.setenv("EDTB200_BOUNDED_RMAX", "-1")
        dist2, idx2 = (np.asarray(a) for a in edt.feature_transform(arr, w, bb, signed=signed, return_distances=True,
                                                                     max_distance=d))
        assert same_bits(dist2, dist) and (idx2[:, ~inside] == -1).all()
      assert inside_any


FNS = {"erode": "spherical_erode", "open": "spherical_open", "dilate": "spherical_dilate", "close": "spherical_close"}


def morph(edt, op, arr, r, w, bb, **kw):
  fn = getattr(edt, FNS[op])
  return fn(arr, r, w, **kw) if op == "dilate" else fn(arr, r, w, bb, **kw)


def same_labels(got, exp):
  got, exp = np.asarray(got), np.asarray(exp)
  return got.dtype == exp.dtype and got.shape == exp.shape and np.array_equal(mc._raw(got), mc._raw(exp))


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("nd", [2, 3])
def test_morphology_windowed(edt, monkeypatch, nd, order):
  """The select kernel in the last pass's store, at radii up to 128."""
  rng = np.random.default_rng(nd * 40 + (order == "F"))
  shape = {2: (140, 133), 3: (14, 30, 135)}[nd]
  arr = mc.seeded(rng, "voronoi", shape, np.uint32)
  arr = np.asfortranarray(arr) if order == "F" else np.ascontiguousarray(arr)
  for r in (1.0, 3.0, 33.0, 64.0, 128.0):
    for op in mc.OPS:
      bb = op != "dilate" and r != 33.0
      monkeypatch.setenv("EDTB200_BOUNDED_RMAX", "128")
      got = morph(edt, op, arr, r, None, bb)
      launch = edt.last_later_launch()
      assert launch["kernel"] == "window" and launch["tx"] == int(r), (op, r, launch)
      assert same_labels(got, mc.threshold(op, arr, r, None, bb and op != "dilate")), (op, r)
      monkeypatch.setenv("EDTB200_BOUNDED_RMAX", "-1")
      assert same_labels(morph(edt, op, arr, r, None, bb), got), (op, r)


@pytest.mark.parametrize("order", ["C", "F"])
def test_morphology_windowed_stacks(edt, monkeypatch, order):
  """Stacks of volumes: a z window must stop at the boundary between two volumes of the stack."""
  rng = np.random.default_rng(50 + (order == "F"))
  vols = [mc.seeded(rng, kind, (20, 24, 70), np.uint16) for kind in ("voronoi", "balls", "touching")]
  stack = np.ascontiguousarray(np.stack(vols)) if order == "C" else np.asfortranarray(np.stack(vols, axis=-1))
  for r in (2.0, 19.0, 33.0, 128.0):
    for op in mc.OPS:
      monkeypatch.setenv("EDTB200_BOUNDED_RMAX", "128")
      got = morph(edt, op, stack, r, None, True, stacked=True)
      assert edt.last_later_launch()["kernel"] == "window", (op, r)
      per = [mc.threshold(op, v, r, None, op != "dilate") for v in vols]
      exp = np.stack(per) if order == "C" else np.stack(per, axis=-1)
      assert same_labels(got, exp), (op, r)
      monkeypatch.setenv("EDTB200_BOUNDED_RMAX", "-1")
      assert same_labels(morph(edt, op, stack, r, None, True, stacked=True), got), (op, r)


@pytest.fixture(autouse=True)
def _record_run(request):
  yield
  RAN.add(request.node.name)


RAN = set()
PRODUCERS = {"test_pass_every_variant[%d]" % b for b in WIDTHS} | {"test_pass_every_length_and_radius[%d]" % b for b in WIDTHS}


def test_every_reachable_variant_was_run():
  """Every (label bytes, sites, epilogue, exact) variant of the window kernel, and every radius of RADII,
  was launched by the pass tests above.  Meaningful only after those tests have run in this process (the
  file's order); skipped otherwise."""
  if not PRODUCERS <= RAN:
    pytest.skip("the variant-producing tests of this file did not run before this one: %s" % sorted(PRODUCERS - RAN))
  want = {(b, s, e, x) for b in WIDTHS for s in (False, True) for e in (False, True) for x in (False, True)}
  print("\nwindow variants run (%d of %d): %s" % (len(HIT & want), len(want), sorted(HIT)))
  assert HIT == want, sorted(want - HIT)
  assert set(RADII) <= RADII_RUN, sorted(set(RADII) - RADII_RUN)
