"""GPU tests of the bounded transforms (max_distance=d): every result against the library's own
unbounded call with the band applied -- where(|S| <= d*d, unbounded, +-inf), S the unbounded squared
value, compared bit for bit -- and the feature transform's sites through the site contract of
feature_cases.check_sites inside the band, -1 outside it.
"""
import math

import numpy as np
import pytest

from feature_cases import brute_sites, check_sites, memory_order

pytestmark = pytest.mark.gpu

WINDOW_MAX = 2           # EDTB200_BOUNDED_WINDOW_MAX (edtb200_transform_bounded)
SITES_WINDOW_MAX = 32    # EDTB200_BOUNDED_SITES_WINDOW_MAX (edtb200_feature_transform_bounded)
DTYPES = [np.bool_, np.uint8, np.int16, np.uint32, np.int64, np.float32]
SHAPES = {1: (203,), 2: (37, 70), 3: (19, 23, 41)}
ANISO = {"int": (1.0, 2.0, 3.0), "real": (0.7, 1.3, 2.9), "dyadic": (0.5, 1.25, 2.0)}
FUNCS = {"edtsq": (False, False), "edt": (True, False), "sdfsq": (False, True), "sdf": (True, True)}


def same_bits(a, b):
  a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
  return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def band(sq, d):
  """Where the unbounded squared value sq (signed: negative on background) is kept under bound d."""
  return np.abs(np.asarray(sq, np.float32)).astype(np.float64) <= d * d


def cut(unbounded, sq, d):
  sq = np.asarray(sq, np.float32)
  return np.where(band(sq, d), unbounded, np.where(np.signbit(sq), -np.inf, np.inf)).astype(np.float32)


def volume(rng, shape, dtype, order):
  """Blocky labels with background and long runs, so that windows meet run ends and faces."""
  small = rng.integers(0, 4, tuple(max(1, s // 5) + 1 for s in shape))
  lab = small
  for ax, s in enumerate(shape):
    lab = np.repeat(lab, 5, axis=ax).take(np.arange(s), axis=ax)
  lab = lab * (rng.random(shape) > 0.02)
  if dtype == np.bool_:
    lab = lab > 1
  arr = lab.astype(dtype)
  return np.asfortranarray(arr) if order == "F" else np.ascontiguousarray(arr)


def plan(edt, arr, aniso, d):
  """(radius, windowed) of edtb200_bounded_plan for this array (x-fastest axes)."""
  import ctypes
  nd = arr.ndim
  dims = list(arr.shape)
  w = list(aniso[:nd])
  if memory_order(arr) == "C":
    dims.reverse(); w.reverse()
  dims += [1] * (3 - nd); w += [1.0] * (3 - nd)
  r = (ctypes.c_int64 * 3)()
  win = (ctypes.c_int * 3)()
  assert edt._lib().edtb200_bounded_plan(nd, *dims, *w, d, r, win) == 0
  return list(r), list(win)


def fallback_distance(edt, arr, aniso, bit):
  """A d whose plan (bit 1: the transform's, 2: the feature transform's) takes the window kernel on
  one later axis and the unbounded kernel on another (in 2-D: the unbounded kernel on the only later
  axis)."""
  for d in np.arange(0.5, 120.0, 0.25):
    _, win = plan(edt, arr, aniso, float(d))
    if arr.ndim == 2 and not win[1] & bit:
      return float(d)
    if arr.ndim == 3 and (win[1] & bit) != (win[2] & bit):
      return float(d)
  return None


def distances(edt, arr, aniso):
  out = [0.0, 0.5, 1.0, 2.5, 7.9, math.inf]
  if arr.ndim >= 2:
    out += sorted(d for d in {fallback_distance(edt, arr, aniso, 1), fallback_distance(edt, arr, aniso, 2)} if d)
  return out


def run(edt, fn, arr, aniso, border, d):
  kw = {} if d is None else {"max_distance": d}
  return np.asarray(getattr(edt, fn)(arr, anisotropy=aniso, black_border=border, **kw))


@pytest.mark.parametrize("aniso", sorted(ANISO))
@pytest.mark.parametrize("border", [False, True])
@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("ndim", [1, 2, 3])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda t: np.dtype(t).name)
def test_transform_is_the_cut_unbounded_transform(edt, dtype, ndim, order, border, aniso):
  rng = np.random.default_rng(ndim * 100 + len(aniso) + border)
  arr = volume(rng, SHAPES[ndim], dtype, order)
  w = ANISO[aniso][:ndim]
  sq = {False: run(edt, "edtsq", arr, w, border, None), True: run(edt, "sdfsq", arr, w, border, None)}
  for d in distances(edt, arr, w):
    for fn, (_, signed) in FUNCS.items():
      unb = run(edt, fn, arr, w, border, None)
      got = run(edt, fn, arr, w, border, d)
      want = cut(unb, sq[signed], d)
      assert got.flags.f_contiguous == arr.flags.f_contiguous or ndim == 1
      assert same_bits(got, want), (fn, d, int((got.view(np.uint32) != want.view(np.uint32)).sum()))


def check_bounded_features(edt, arr, w, border, signed, d):
  dist, idx = edt.feature_transform(arr, w, border, signed=signed, return_distances=True, max_distance=d)
  udist, uidx = edt.feature_transform(arr, w, border, signed=signed, return_distances=True)
  sq = run(edt, "sdfsq" if signed else "edtsq", arr, w, border, None)
  dist, idx, udist, uidx = (np.asarray(a) for a in (dist, idx, udist, uidx))
  assert same_bits(dist, cut(udist, sq, d)), d
  inside = band(sq, d)
  assert (idx[:, ~inside] == -1).all(), "a site outside the band"
  sites = np.where(inside[None], idx, uidx)
  check_sites(arr, sites, np.abs(sq), w, border, signed)


@pytest.mark.parametrize("aniso", sorted(ANISO))
@pytest.mark.parametrize("signed", [False, True])
@pytest.mark.parametrize("border", [False, True])
@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_feature_transform_in_the_band(edt, ndim, order, border, signed, aniso):
  rng = np.random.default_rng(7 + ndim)
  w = ANISO[aniso][:ndim]
  for dtype in (np.uint8, np.int64, np.float32):
    arr = volume(rng, SHAPES[ndim], dtype, order)
    for d in distances(edt, arr, w):
      check_bounded_features(edt, arr, w, border, signed, d)


def test_attained_distance_and_one_below(edt):
  rng = np.random.default_rng(3)
  arr = volume(rng, (24, 26, 28), np.uint32, "C")
  sq = run(edt, "edtsq", arr, (1, 1, 1), False, None)
  for s in (1.0, 4.0, 9.0):
    assert (sq == s).any()
    d = math.sqrt(s)
    got = run(edt, "edtsq", arr, (1, 1, 1), False, d)
    assert (got[sq == s] == s).all()
    assert same_bits(got, cut(sq, sq, d))
    below = math.nextafter(d, 0.0)
    got = run(edt, "edtsq", arr, (1, 1, 1), False, below)
    assert np.isinf(got[sq == s]).all()
    assert same_bits(got, cut(sq, sq, below))


def test_zero_radius_pass(edt):
  arr = np.ones((40, 30, 30), np.uint8)
  arr[20, 15, 15] = 0
  w = (30.0, 6.0, 6.0)                                      # z weight 30 with d = 24: R_z = 0
  r, win = plan(edt, arr, w, 24.0)
  assert r[2] == 0 and win[2] == 3
  for border in (False, True):
    unb = run(edt, "edtsq", arr, w, border, None)
    got = run(edt, "edtsq", arr, w, border, 24.0)
    assert edt.last_later_launch()["kernel"] == "window" and edt.last_later_launch()["tx"] == 0
    assert same_bits(got, cut(unb, unb, 24.0))
  check_bounded_features(edt, arr[:12, :10, :10], w, True, False, 24.0)


def test_rounding_edges(edt):
  import os
  g = np.load(os.path.join(os.path.dirname(__file__), "golden", "rounding_edges.npz"))
  for name in g["names"]:
    name = str(name)
    arr, w, border = g[name + "_labels"], tuple(g[name + "_aniso"]), bool(g[name + "_border"])
    for fn in ("edtsq", "sdf"):
      unb = run(edt, fn, arr, w, border, None)
      sq = run(edt, "sdfsq" if fn == "sdf" else "edtsq", arr, w, border, None)
      finite = np.abs(sq[np.isfinite(sq)])
      ds = (1.0, 2.5, 7.9, 30.0) + ((float(np.sqrt(np.float64(np.median(finite)))),) if finite.size else ())
      for d in ds:
        got = run(edt, fn, arr, w, border, d)
        assert same_bits(got, cut(unb, sq, d)), (name, fn, d)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint32])
def test_window_maximum_and_one_beyond(edt, dtype):
  rng = np.random.default_rng(11)
  arr = volume(rng, (64, 48, 40), dtype, "C")
  unb = run(edt, "edt", arr, (1, 1, 1), True, None)
  sq = run(edt, "edtsq", arr, (1, 1, 1), True, None)
  got = run(edt, "edt", arr, (1, 1, 1), True, float(WINDOW_MAX))
  launch = edt.last_later_launch()
  assert launch["kernel"] == "window" and launch["tx"] == WINDOW_MAX and launch["epilogue"] == 1
  assert same_bits(got, cut(unb, sq, float(WINDOW_MAX)))
  got = run(edt, "edt", arr, (1, 1, 1), True, float(WINDOW_MAX + 1))
  assert edt.last_later_launch()["kernel"] in ("tile", "long")
  assert same_bits(got, cut(unb, sq, float(WINDOW_MAX + 1)))
  small = np.ascontiguousarray(arr[:, :20, :16])
  for d in (float(SITES_WINDOW_MAX), float(SITES_WINDOW_MAX + 1)):
    check_bounded_features(edt, small, (1, 1, 1), True, False, d)
    edt.edtsq(small)                                        # records a tile launch
    edt.feature_transform(small, (1, 1, 1), True, max_distance=d)
    launch = edt.last_later_launch()                        # the long-line site pass records none
    assert (launch["kernel"], launch["tx"]) == ("window", SITES_WINDOW_MAX) if d == SITES_WINDOW_MAX else \
        launch["kernel"] == "tile"


@pytest.mark.parametrize("name", ["cfg2", "cfg2b", "cfg3", "balls", "voronoi", "ones_nobb"])
def test_workloads(edt, name):
  import torch
  from edt_b200.workloads import generate
  lab, w, border = generate(name, 256, "cuda")
  sq = edt.edt_cuda(lab, w, border)
  full = edt.edt_cuda(lab, w, border, sqrt=True)
  for d in (2.5, 8.0, 24.0):
    got = edt.edt_cuda(lab, w, border, max_distance=d)
    want = torch.where(sq.double() <= d * d, sq, torch.full_like(sq, float("inf")))
    assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (name, d)
    dist, idx = edt.feature_transform(lab, w, border, return_distances=True, max_distance=d)
    inside = sq.double() <= d * d
    want = torch.where(inside, full, torch.full_like(full, float("inf")))
    assert torch.equal(dist.view(torch.int32), want.view(torch.int32)), (name, d)
    assert bool((idx[:, ~inside] == -1).all()) and bool((idx[:, inside] >= -1).all())
    # the site of every voxel in the band is at its distance (summed in double and rounded once, as the
    # passes do, for the integer weights of these workloads)
    p = torch.stack(torch.meshgrid(*[torch.arange(s, device="cuda") for s in lab.shape], indexing="ij"))
    ww = torch.tensor(w, device="cuda", dtype=torch.float64).view(3, 1, 1, 1)
    val = (((idx.double() - p.double()) * ww) ** 2).sum(0).float()
    assert torch.equal(val[inside], sq[inside]), (name, d)


def test_device_input_on_a_side_stream(edt):
  import torch
  rng = np.random.default_rng(5)
  arr = volume(rng, (30, 31, 33), np.int32, "C")
  host_sq = run(edt, "sdfsq", arr, (1.0, 2.0, 0.5), False, None)
  host_unb = run(edt, "sdf", arr, (1.0, 2.0, 0.5), False, None)
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    t = torch.as_tensor(arr, device="cuda")
    got = edt.sdf(t, anisotropy=(1.0, 2.0, 0.5), max_distance=3.0)
    tf = t.permute(2, 1, 0)                                  # an F-ordered view
    got_f = edt.edtsq(tf, anisotropy=(0.5, 2.0, 1.0), max_distance=3.0)
    dist, idx = edt.feature_transform(t, (1.0, 2.0, 0.5), signed=True, return_distances=True, max_distance=3.0)
  side.synchronize()
  assert same_bits(got.cpu().numpy(), cut(host_unb, host_sq, 3.0))
  assert same_bits(dist.cpu().numpy(), cut(host_unb, host_sq, 3.0))
  unb_f = run(edt, "edtsq", np.asfortranarray(arr.transpose(2, 1, 0)), (0.5, 2.0, 1.0), False, None)
  assert same_bits(got_f.cpu().numpy(), cut(unb_f, unb_f, 3.0))
  check_sites(arr, np.where(band(host_sq, 3.0)[None], idx.cpu().numpy(),
                            np.asarray(edt.feature_transform(arr, (1.0, 2.0, 0.5), signed=True))),
              np.abs(host_sq), (1.0, 2.0, 0.5), False, True)


@pytest.mark.parametrize("signed", [False, True])
@pytest.mark.parametrize("border", [False, True])
def test_brute_force(edt, border, signed):
  rng = np.random.default_rng(17)
  arr = rng.integers(0, 3, (5, 6, 4)).astype(np.uint16)
  w = (1.0, 1.5, 0.75)
  want_sq, _ = brute_sites(arr, w, border, signed)
  want_sq = np.where(signed & (arr == 0), -want_sq, want_sq).astype(np.float32)
  for d in (0.0, 0.8, 1.2, 2.0, 3.5):
    got = run(edt, "sdfsq" if signed else "edtsq", arr, w, border, d)
    assert same_bits(got, cut(want_sq, want_sq, d)), d
    check_bounded_features(edt, arr, w, border, signed, d)
