"""CPU tests of the bounded transforms (max_distance): the plan of edtb200_bounded_plan against a
Python restatement of the cut B and the window radii R_k, the argument checks of
edtb200_transform_bounded and edtb200_feature_transform_bounded, and the Python rejections.

As in test_stack_arguments.py, every rejection comes before any device is touched, and a fully valid
call stops at the device probe: device 64 is a "bad device" everywhere.  Nothing here launches a
kernel or copies a byte.
"""
import ctypes
import math

import numpy as np
import pytest

from abi_checks import ABI_VERSION, EINVAL

WINDOW_MAX = 2           # EDTB200_BOUNDED_WINDOW_MAX (edtb200_transform_bounded)
SITES_WINDOW_MAX = 32    # EDTB200_BOUNDED_SITES_WINDOW_MAX (edtb200_feature_transform_bounded)
CAP = 1 << 62

_LABELS = np.zeros(512, np.uint64)
_OUT = np.zeros(512, np.uint64)
L, O = _LABELS.ctypes.data, _OUT.ctypes.data


def f32(x):
  return float(np.float32(x))


def restated_plan(ndim, w, d):
  """B = the largest float32 with (double)B <= d*d; R_k = the largest r >= 0 with
  (double)fl32(w_k*w_k) * r * r < nextafterf(B, +inf) (capped at 2^62); on the later axes, bit 0 of
  windowed where R_k <= the transform's window maximum, bit 1 where R_k <= the feature transform's."""
  lim = d * d
  if lim >= float(np.finfo(np.float32).max):
    b = np.finfo(np.float32).max
  else:
    b = np.float32(lim)
    if float(b) > lim:
      b = np.nextafter(b, np.float32(-np.inf))
  with np.errstate(over="ignore"):                  # nextafter(FLT_MAX) is +inf
    above = float(np.nextafter(np.float32(b), np.float32(np.inf)))
  radius, windowed = [0, 0, 0], [0, 0, 0]
  for k in range(ndim):
    w2 = float(np.float32(np.float32(w[k]) * np.float32(w[k])))
    lo, hi = 0, CAP
    while lo < hi:
      mid = lo + (hi - lo + 1) // 2
      if w2 * float(mid) * float(mid) < above:
        lo = mid
      else:
        hi = mid - 1
    radius[k] = lo
    windowed[k] = int(k >= 1 and lo <= WINDOW_MAX) | int(k >= 1 and lo <= SITES_WINDOW_MAX) << 1
  return radius, windowed


def plan(edt, ndim, w, d, sizes=(8, 8, 8)):
  r = (ctypes.c_int64 * 3)()
  win = (ctypes.c_int * 3)()
  rc = edt._lib().edtb200_bounded_plan(ndim, *sizes, *w, d, r, win)
  return rc, list(r), list(win)


def test_symbols_and_version(edt):
  lib = edt._lib()
  for name in ("edtb200_transform_bounded", "edtb200_feature_transform_bounded", "edtb200_bounded_plan"):
    assert hasattr(lib, name)
  assert lib.edtb200_version() == ABI_VERSION


def _ds_around(b):
  """d at the square root of B (a float32) and one double either side of it."""
  s = math.sqrt(float(b))
  return [s, math.nextafter(s, 0.0), math.nextafter(s, math.inf)]


WEIGHTS = [
  (1.0, 1.0, 1.0), (1.0, 1.0, 30.0), (2.0, 3.0, 5.0),           # integer
  (0.7, 1.3, 2.9), (0.1, 1.0, 4.4),                              # real
  (0.5, 0.25, 1.5), (0.75, 2.5, 0.125),                          # dyadic
]
DS = [0.0, 0.5, 1.0, 2.5, 7.9, 8.0, 16.0, 17.0, 24.0, 1e3, 1e20, 1e200, math.inf]
DS += _ds_around(np.float32(64.0)) + _ds_around(np.float32(2.5 * 2.5)) + _ds_around(np.nextafter(np.float32(49), 0))


@pytest.mark.parametrize("w", WEIGHTS)
@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_plan_matches_restatement(edt, w, ndim):
  for d in DS:
    rc, radius, windowed = plan(edt, ndim, w, d)
    assert rc == 0
    want_r, want_w = restated_plan(ndim, w, d)
    assert (radius, windowed) == (want_r, want_w), (w, ndim, d)


def test_plan_edges(edt):
  # d = 0: no neighbour is in reach
  assert plan(edt, 3, (1.0, 1.0, 1.0), 0.0)[1:] == ([0, 0, 0], [0, 3, 3])
  # the z weight of 30 with d = 24: R_z = 0, a real window
  assert plan(edt, 3, (1.0, 1.0, 30.0), 24.0)[1:] == ([24, 24, 0], [0, 2, 3])
  # an attained distance is inside: d = 3 with unit weights reaches 3 rows, one float below does not
  assert plan(edt, 2, (1.0, 1.0, 1.0), 3.0)[1][1] == 3
  assert plan(edt, 2, (1.0, 1.0, 1.0), float(np.nextafter(np.float32(3.0), 0)))[1][1] == 2
  # the window maxima and one beyond them
  assert plan(edt, 2, (1.0, 1.0, 1.0), float(WINDOW_MAX))[1:] == ([WINDOW_MAX, WINDOW_MAX, 0], [0, 3, 0])
  assert plan(edt, 2, (1.0, 1.0, 1.0), float(WINDOW_MAX + 1))[2] == [0, 2, 0]
  assert plan(edt, 2, (1.0, 1.0, 1.0), float(SITES_WINDOW_MAX))[2] == [0, 2, 0]
  assert plan(edt, 2, (1.0, 1.0, 1.0), float(SITES_WINDOW_MAX + 1))[2] == [0, 0, 0]
  # no bound: the cap
  assert plan(edt, 3, (1.0, 1.0, 1.0), math.inf)[1:] == ([CAP] * 3, [0, 0, 0])
  assert plan(edt, 3, (1.0, 1.0, 1.0), 1e200)[1:] == ([CAP] * 3, [0, 0, 0])


@pytest.mark.parametrize("d", [-1.0, -0.0 - 1e-300, math.nan, -math.inf])
def test_plan_rejects_bad_distance(edt, d):
  assert plan(edt, 3, (1.0, 1.0, 1.0), d)[0] == EINVAL
  assert b"max_distance" in edt._lib().edtb200_last_error()


def test_plan_argument_order(edt):
  lib = edt._lib()
  r = (ctypes.c_int64 * 3)()
  win = (ctypes.c_int * 3)()
  assert lib.edtb200_bounded_plan(4, 8, 8, 8, 1.0, 1.0, 1.0, 1.0, r, win) == EINVAL
  assert b"ndim" in lib.edtb200_last_error()
  assert lib.edtb200_bounded_plan(3, -1, 8, 8, 1.0, 1.0, 1.0, math.nan, r, win) == EINVAL
  assert b"negative size" in lib.edtb200_last_error()
  assert lib.edtb200_bounded_plan(3, 8, 8, 8, 1.0, 1.0, 1.0, math.nan, None, None) == EINVAL
  assert b"max_distance" in lib.edtb200_last_error()
  assert lib.edtb200_bounded_plan(3, 8, 8, 8, 1.0, 1.0, 1.0, 1.0, None, win) == EINVAL
  assert b"null pointer" in lib.edtb200_last_error()


def _transform(labels=L, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, border=0, flags=0, out=O, device=64, d=1.0):
  return (labels, label_bytes, ndim, sx, sy, sz, 1.0, 1.0, 1.0, border, flags, out, device, None, d)


def _feature(labels=L, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, border=0, flags=0, idx="all", device=64, d=1.0):
  idx = (ctypes.c_void_p * 3)(O, O, O) if idx == "all" else idx
  return (labels, label_bytes, ndim, sx, sy, sz, 1.0, 1.0, 1.0, border, flags, None, idx, device, None, d)


@pytest.mark.parametrize("args, needle", [
  (dict(label_bytes=3, d=math.nan), b"label_bytes"),
  (dict(ndim=0, d=math.nan), b"ndim"),
  (dict(sx=-1, d=math.nan), b"negative size"),
  (dict(labels=None, d=math.nan), b"null pointer"),
  (dict(d=math.nan), b"max_distance"),
  (dict(d=-2.0), b"max_distance"),
  (dict(d=3.0), b"bad device"),
  (dict(d=0.0), b"bad device"),
])
def test_transform_bounded_checks(edt, args, needle):
  lib = edt._lib()
  assert lib.edtb200_transform_bounded(*_transform(**args)) == EINVAL
  assert needle in lib.edtb200_last_error()


def test_transform_bounded_empty_is_a_no_op(edt):
  assert edt._lib().edtb200_transform_bounded(*_transform(sx=0, d=math.nan)) == 0


@pytest.mark.parametrize("args, needle", [
  (dict(label_bytes=3, d=math.nan), b"label_bytes"),
  (dict(ndim=4, d=math.nan), b"ndim"),
  (dict(labels=None, d=math.nan), b"null pointer"),
  (dict(idx=(ctypes.c_void_p * 3)(O, None, O), d=math.nan), b"null index plane 1"),
  (dict(d=math.nan), b"max_distance"),
  (dict(d=-0.5), b"max_distance"),
  (dict(d=2.0), b"bad device"),
])
def test_feature_bounded_checks(edt, args, needle):
  lib = edt._lib()
  assert lib.edtb200_feature_transform_bounded(*_feature(**args)) == EINVAL
  assert needle in lib.edtb200_last_error()


VOL = np.zeros((4, 5, 6), np.uint8)


@pytest.mark.parametrize("fn", ["edt", "edtsq", "sdf", "sdfsq"])
@pytest.mark.parametrize("kwargs, needle", [
  (dict(max_distance=-1.0), "zero or more"),
  (dict(max_distance=math.nan), "zero or more"),
  (dict(max_distance=2.0, voxel_graph=np.zeros((4, 5, 6), np.uint8)), "voxel_graph"),
  (dict(max_distance=2.0, devices=[0, 1]), "devices"),
  (dict(max_distance=2.0, stacked=True), "stacked"),
  (dict(max_distance=2.0, max_device_bytes=1 << 20), "max_device_bytes"),
  (dict(max_distance=math.inf, stacked=True), "stacked"),
])
def test_python_rejections(edt, fn, kwargs, needle):
  with pytest.raises(ValueError, match=needle):
    getattr(edt, fn)(VOL, **kwargs)


def test_python_rejections_other_entry_points(edt):
  with pytest.raises(ValueError, match="stacked"):
    edt.feature_transform(VOL, max_distance=1.0, stacked=True)
  with pytest.raises(ValueError, match="max_device_bytes"):
    edt.feature_transform(VOL, max_distance=1.0, max_device_bytes=0)
  with pytest.raises(ValueError, match="zero or more"):
    edt.feature_transform(VOL, max_distance=-3)
  with pytest.raises(ValueError, match="zero or more"):
    edt.edt1dsq(np.zeros(5, np.uint8), max_distance=math.nan)
  with pytest.raises(ValueError, match="voxel_graph"):
    edt.edt2d(np.zeros((3, 3), np.uint8), voxel_graph=np.zeros((3, 3), np.uint8), max_distance=1.0)
  with pytest.raises(ValueError, match="max_device_bytes"):
    edt.edt3dsq(VOL, max_device_bytes=0, max_distance=1.0)
