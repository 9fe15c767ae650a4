"""CPU tests: the argument checks of edtb200_morphology, in their documented order, and the Python
rejections of spherical_erode, spherical_open, spherical_dilate and spherical_close.

As in test_surface_arguments.py, every rejection comes with a return code and a message before any
device is touched, and a fully valid call stops at the device probe (abi_checks.expect_probe).  Nothing here
launches a kernel or copies a byte.
"""
import ctypes
import inspect
import re

import numpy as np
import pytest

from abi_checks import (ABI_VERSION, BIG, BOTH, EINVAL, ELIMIT, HEADER, LABELS_FLOAT, LABELS_ON_DEVICE, PROBE, SIGNED,
                        SQRT, check_case, no_device_use)

ERODE, DILATE, OPEN, CLOSE = 0, 1, 2, 3

_IN = np.zeros(512, np.uint64)
_OUT = np.zeros(512, np.uint64)
IN, OUT = _IN.ctypes.data, _OUT.ctypes.data


def _args(labels=IN, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, count=2, w=(1.0, 1.0, 1.0), op=ERODE, radius=2.0,
          black_border=0, flags=BOTH, out=OUT, device=63, stream=None):
  return (labels, label_bytes, ndim, sx, sy, sz, count, w[0], w[1], w[2], op, radius, black_border, flags, out,
          device, stream)


CASES = [
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes"),
  ("label_bytes_16", dict(label_bytes=16), EINVAL, "label_bytes"),
  ("ndim_0", dict(ndim=0), EINVAL, "ndim"),
  ("ndim_4", dict(ndim=4), EINVAL, "ndim"),
  ("negative_size", dict(sy=-1), EINVAL, "negative size"),
  ("axis_too_long", dict(sx=BIG), ELIMIT, "axis longer than 2^30"),
  ("negative_count", dict(count=-1), EINVAL, "negative count"),
  ("op_negative", dict(op=-1), EINVAL, "op must be"),
  ("op_4", dict(op=4), EINVAL, "op must be"),
  ("radius_negative", dict(radius=-0.5), EINVAL, "radius must be finite"),
  ("radius_nan", dict(radius=float("nan")), EINVAL, "radius must be finite"),
  ("radius_inf", dict(radius=float("inf")), EINVAL, "radius must be finite"),
  ("radius_minus_inf", dict(radius=float("-inf")), EINVAL, "radius must be finite"),
  ("flag_sqrt", dict(flags=BOTH | SQRT), EINVAL, "residency flags"),
  ("flag_signed", dict(flags=SIGNED), EINVAL, "residency flags"),
  ("float_1_byte", dict(label_bytes=1, flags=BOTH | LABELS_FLOAT), EINVAL, "4- or 8-byte"),
  ("float_2_byte", dict(label_bytes=2, flags=LABELS_FLOAT), EINVAL, "4- or 8-byte"),
  ("too_many_voxels", dict(count=1 << 60), ELIMIT, "too many voxels"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_out", dict(out=None), EINVAL, "null pointer"),
  # order: label width, ndim, sizes, count, op, radius, flags, float width, stack size, emptiness,
  # pointers, device
  ("label_bytes_before_ndim", dict(label_bytes=3, ndim=4), EINVAL, "label_bytes"),
  ("ndim_before_size", dict(ndim=5, sx=-1), EINVAL, "ndim"),
  ("size_before_count", dict(sx=BIG, count=-1), ELIMIT, "axis longer"),
  ("count_before_op", dict(count=-1, op=9), EINVAL, "negative count"),
  ("op_before_radius", dict(op=9, radius=-1.0), EINVAL, "op must be"),
  ("radius_before_flags", dict(radius=-1.0, flags=SQRT), EINVAL, "radius must be finite"),
  ("flags_before_float_width", dict(flags=SQRT | LABELS_FLOAT, label_bytes=2), EINVAL, "residency flags"),
  ("float_width_before_empty", dict(flags=LABELS_FLOAT, label_bytes=1, sz=0), EINVAL, "4- or 8-byte"),
  ("radius_before_empty", dict(radius=-1.0, count=0), EINVAL, "radius must be finite"),
  ("op_before_pointers", dict(op=7, labels=None), EINVAL, "op must be"),
  ("no_volumes", dict(count=0, labels=None, out=None), 0, ""),
  ("empty_volume", dict(sz=0, labels=None, out=None, flags=0), 0, ""),
  ("valid", dict(), PROBE, ""),
  ("valid_host", dict(flags=0), PROBE, ""),
  ("valid_mixed", dict(flags=LABELS_ON_DEVICE), PROBE, ""),
  ("valid_float_4", dict(flags=BOTH | LABELS_FLOAT), PROBE, ""),
  ("valid_float_8", dict(label_bytes=8, flags=LABELS_FLOAT), PROBE, ""),
  ("valid_every_op", dict(op=CLOSE, black_border=1), PROBE, ""),
  ("valid_dilate", dict(op=DILATE), PROBE, ""),
  ("valid_open", dict(op=OPEN), PROBE, ""),
  ("valid_radius_0", dict(radius=0.0), PROBE, ""),
  ("valid_huge_radius", dict(radius=1e300), PROBE, ""),
  ("valid_2d_ignores_sz", dict(ndim=2, sz=-1), PROBE, ""),
  ("valid_1d_ignores_sy_sz", dict(ndim=1, sy=-1, sz=BIG), PROBE, ""),
]


@pytest.mark.parametrize("case,overrides,rc,msg", CASES, ids=[c[0] for c in CASES])
def test_morphology_argument_check(edt, case, overrides, rc, msg):
  check_case(edt, edt._lib().edtb200_morphology, _args, overrides, rc, msg)


def test_morphology_is_an_addition_at_the_same_version(edt):
  lib = edt._lib()
  assert lib.edtb200_version() == ABI_VERSION
  assert "edtb200_morphology" in set(re.findall(r"\b(edtb200_[a-z0-9_]+)\s*\(", HEADER))
  version_comment = HEADER[:HEADER.index("#define EDTB200_VERSION")]
  assert "edtb200_morphology" in version_comment
  for name, value in (("ERODE", 0), ("DILATE", 1), ("OPEN", 2), ("CLOSE", 3)):
    assert re.search(r"#define EDTB200_%s\s+%d\b" % (name, value), HEADER), name
  assert hasattr(ctypes.CDLL(edt.library_path()), "edtb200_morphology")
  assert lib.edtb200_morphology.argtypes[11] is ctypes.c_double


# ---- Python ---------------------------------------------------------------------------------------------

FNS = ["spherical_erode", "spherical_open", "spherical_dilate", "spherical_close"]


def test_exported(edt):
  for name in FNS:
    assert name in edt.__all__ and callable(getattr(edt, name))
    params = inspect.signature(getattr(edt, name)).parameters
    assert list(params)[:3] == ["labels", "radius", "anisotropy"]
    for kw in ("device", "stacked"):
      assert params[kw].kind is inspect.Parameter.KEYWORD_ONLY, (name, kw)
    assert params["stacked"].default is False
    assert ("black_border" in params) == (name != "spherical_dilate")


@pytest.mark.parametrize("name", FNS)
@pytest.mark.parametrize("radius", [-1.0, -1e-300, float("nan"), float("inf"), float("-inf")])
def test_rejects_bad_radius(no_device_use, name, radius):
  with pytest.raises(ValueError, match="radius must be finite"):
    getattr(no_device_use, name)(np.ones((4, 5), np.uint8), radius)


@pytest.mark.parametrize("name", FNS)
def test_rejects_bad_radius_before_anything_else(no_device_use, name):
  with pytest.raises(ValueError, match="radius"):
    getattr(no_device_use, name)(np.ones((2, 2, 2, 2, 2), np.complex64), -1.0)


@pytest.mark.parametrize("name", FNS)
@pytest.mark.parametrize("dtype", [np.float16, np.complex64, np.object_, np.dtype("U3"), np.dtype("V4")])
def test_rejects_unsupported_dtype(no_device_use, name, dtype):
  with pytest.raises(TypeError, match="unsupported label dtype"):
    getattr(no_device_use, name)(np.zeros((3, 4), dtype), 1.0)


@pytest.mark.parametrize("name", FNS)
def test_rejects_dimension_counts(no_device_use, name):
  fn = getattr(no_device_use, name)
  with pytest.raises(TypeError, match="1-D to 3-D"):
    fn(np.uint8(3), 1.0)
  with pytest.raises(TypeError, match="1-D to 3-D"):
    fn(np.ones((2, 2, 2, 2), np.uint8), 1.0)
  with pytest.raises(TypeError, match="2-D to 4-D"):
    fn(np.ones(5, np.uint8), 1.0, stacked=True)
  with pytest.raises(TypeError, match="2-D to 4-D"):
    fn(np.ones((2, 2, 2, 2, 2), np.uint8), 1.0, stacked=True)


@pytest.mark.parametrize("name", FNS)
def test_rejects_anisotropy_of_the_wrong_length(no_device_use, name):
  fn = getattr(no_device_use, name)
  with pytest.raises(ValueError, match="one entry per volume axis"):
    fn(np.ones((4, 5), np.uint8), 1.0, (1.0, 2.0, 3.0))
  with pytest.raises(ValueError, match="one entry per volume axis"):
    fn(np.ones((3, 4, 5), np.uint8), 1.0, (1.0, 2.0, 3.0), stacked=True)


@pytest.mark.parametrize("name", FNS)
@pytest.mark.parametrize("order", ["C", "F"])
def test_empty_arrays_need_no_device(no_device_use, name, order):
  fn = getattr(no_device_use, name)
  for shape, stacked in (((0,), False), ((3, 0, 2), False), ((0, 4, 4), True), ((2, 3, 0, 1), True)):
    arr = np.zeros(shape, np.int32, order=order)
    got = fn(arr, 2.0, stacked=stacked)
    assert isinstance(got, np.ndarray) and got.shape == shape
    assert got.dtype == (np.bool_ if name in ("spherical_dilate", "spherical_close") else np.int32)
    if len(shape) > 1 and order == "F":
      assert got.flags.f_contiguous


def test_the_public_max_distance_fence_stays(edt):
  with pytest.raises(ValueError, match="max_distance cannot be combined with stacked=True"):
    edt.edtsq(np.ones((2, 3, 4), np.uint8), max_distance=2.0, stacked=True)
