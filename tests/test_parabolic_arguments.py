"""CPU tests: the argument checks of edtb200_parabolic in their documented order, and the Python
rejections of parabolic_erode and parabolic_dilate -- each before any device is touched.  A fully valid
call stops at the device probe (abi_checks.expect_probe)."""
import ctypes
import inspect
import re

import numpy as np
import pytest

from abi_checks import (ABI_VERSION, BIG, BOTH, EINVAL, ELIMIT, HEADER, INF, LABELS_FLOAT, LABELS_ON_DEVICE, NAN,
                        PROBE, SQRT, check_case, no_device_use)

ERODE, DILATE = 0, 1

_IN = np.zeros(512, np.float32)
_OUT = np.zeros(512, np.float32)
IN, OUT = _IN.ctypes.data, _OUT.ctypes.data


def _args(f=IN, ndim=3, sx=4, sy=4, sz=4, count=2, w=(1.0, 1.0, 1.0), op=ERODE, flags=BOTH, out=OUT, device=63,
          stream=None):
  return (f, ndim, sx, sy, sz, count, w[0], w[1], w[2], op, flags, out, device, stream)


CASES = [
  ("ndim_0", dict(ndim=0), EINVAL, "ndim"),
  ("ndim_4", dict(ndim=4), EINVAL, "ndim"),
  ("negative_size", dict(sy=-1), EINVAL, "negative size"),
  ("axis_too_long", dict(sx=BIG), ELIMIT, "axis longer than 2^30"),
  ("negative_count", dict(count=-1), EINVAL, "negative count"),
  ("op_negative", dict(op=-1), EINVAL, "op must be"),
  ("op_2", dict(op=2), EINVAL, "op must be"),
  ("weight_zero", dict(w=(1.0, 0.0, 1.0)), EINVAL, "weight of axis 1"),
  ("weight_negative", dict(w=(-1.0, 1.0, 1.0)), EINVAL, "weight of axis 0"),
  ("weight_nan", dict(w=(1.0, 1.0, NAN)), EINVAL, "weight of axis 2"),
  ("weight_inf", dict(w=(INF, 1.0, 1.0)), EINVAL, "weight of axis 0"),
  ("flag_sqrt", dict(flags=BOTH | SQRT), EINVAL, "residency flags"),
  ("flag_float", dict(flags=LABELS_FLOAT), EINVAL, "residency flags"),
  ("too_many_voxels", dict(count=1 << 60), ELIMIT, "too many voxels"),
  ("null_f", dict(f=None), EINVAL, "null pointer"),
  ("null_out", dict(out=None), EINVAL, "null pointer"),
  ("overlap", dict(out=IN + 4), EINVAL, "overlaps"),
  ("overlap_host", dict(out=IN + 4, flags=0), EINVAL, "overlaps"),
  # order: ndim, sizes, count, op, weights, flags, stack size, emptiness, pointers, device
  ("ndim_before_size", dict(ndim=5, sx=-1), EINVAL, "ndim"),
  ("size_before_count", dict(sx=BIG, count=-1), ELIMIT, "axis longer"),
  ("count_before_op", dict(count=-1, op=9), EINVAL, "negative count"),
  ("op_before_weights", dict(op=9, w=(0.0, 0.0, 0.0)), EINVAL, "op must be"),
  ("weights_before_flags", dict(w=(1.0, NAN, 1.0), flags=SQRT), EINVAL, "weight of axis 1"),
  ("weights_before_empty", dict(w=(0.0, 1.0, 1.0), count=0), EINVAL, "weight of axis 0"),
  ("flags_before_empty", dict(flags=SQRT, count=0), EINVAL, "residency flags"),
  ("no_volumes", dict(count=0, f=None, out=None), 0, ""),
  ("empty_volume", dict(sz=0, f=None, out=None, flags=0), 0, ""),
  ("valid", dict(), PROBE, ""),
  ("valid_host", dict(flags=0), PROBE, ""),
  ("valid_mixed", dict(flags=LABELS_ON_DEVICE), PROBE, ""),
  ("valid_mixed_overlap", dict(flags=LABELS_ON_DEVICE, out=IN + 4), PROBE, ""),
  ("valid_in_place", dict(out=IN), PROBE, ""),
  ("valid_dilate", dict(op=DILATE), PROBE, ""),
  ("valid_huge_weight", dict(w=(1e20, 3e38, 1.0)), PROBE, ""),
  ("valid_tiny_weight", dict(w=(1e-30, 1e-45, 1.0)), PROBE, ""),
  ("valid_2d_ignores_sz_wz", dict(ndim=2, sz=-1, w=(1.0, 1.0, NAN)), PROBE, ""),
  ("valid_1d_ignores_sy_sz", dict(ndim=1, sy=-1, sz=BIG, w=(2.0, 0.0, -1.0)), PROBE, ""),
]


@pytest.mark.parametrize("case,overrides,rc,msg", CASES, ids=[c[0] for c in CASES])
def test_parabolic_argument_check(edt, case, overrides, rc, msg):
  check_case(edt, edt._lib().edtb200_parabolic, _args, overrides, rc, msg)


def test_parabolic_is_an_addition_at_the_same_version(edt):
  lib = edt._lib()
  assert lib.edtb200_version() == ABI_VERSION
  assert "edtb200_parabolic" in set(re.findall(r"\b(edtb200_[a-z0-9_]+)\s*\(", HEADER))
  assert "edtb200_parabolic" in HEADER[:HEADER.index("#define EDTB200_VERSION")]
  for name, value in (("PARABOLIC_ERODE", 0), ("PARABOLIC_DILATE", 1)):
    assert re.search(r"#define EDTB200_%s\s+%d\b" % (name, value), HEADER), name
  assert hasattr(ctypes.CDLL(edt.library_path()), "edtb200_parabolic")


# ---- Python ---------------------------------------------------------------------------------------------

FNS = ["parabolic_erode", "parabolic_dilate"]


def test_exported(edt):
  for name in FNS:
    assert name in edt.__all__ and callable(getattr(edt, name))
    params = inspect.signature(getattr(edt, name)).parameters
    assert list(params)[:2] == ["f", "anisotropy"]
    for kw in ("device", "stacked"):
      assert params[kw].kind is inspect.Parameter.KEYWORD_ONLY, (name, kw)
    assert params["stacked"].default is False and params["anisotropy"].default is None


@pytest.mark.parametrize("name", FNS)
@pytest.mark.parametrize("w", [0.0, -1.0, NAN, INF, -INF])
def test_rejects_bad_weights(no_device_use, name, w):
  with pytest.raises(ValueError, match="finite and > 0"):
    getattr(no_device_use, name)(np.ones((4, 5), np.float32), (1.0, w))


@pytest.mark.parametrize("name", FNS)
def test_rejects_anisotropy_of_the_wrong_length(no_device_use, name):
  fn = getattr(no_device_use, name)
  with pytest.raises(ValueError, match="one entry per volume axis"):
    fn(np.ones((4, 5), np.float32), (1.0, 2.0, 3.0))
  with pytest.raises(ValueError, match="one entry per volume axis"):
    fn(np.ones((3, 4, 5), np.float32), (1.0, 2.0, 3.0), stacked=True)


@pytest.mark.parametrize("name", FNS)
@pytest.mark.parametrize("dtype", [np.complex64, np.object_, np.dtype("U3"), np.dtype("V4")])
def test_rejects_non_real_dtypes(no_device_use, name, dtype):
  with pytest.raises(TypeError, match="real or bool"):
    getattr(no_device_use, name)(np.zeros((3, 4), dtype))


@pytest.mark.parametrize("name", FNS)
def test_rejects_dimension_counts(no_device_use, name):
  fn = getattr(no_device_use, name)
  with pytest.raises(TypeError, match="1-D to 3-D"):
    fn(np.float32(3))
  with pytest.raises(TypeError, match="1-D to 3-D"):
    fn(np.ones((2, 2, 2, 2), np.float32))
  with pytest.raises(TypeError, match="2-D to 4-D"):
    fn(np.ones(5, np.float32), stacked=True)
  with pytest.raises(TypeError, match="2-D to 4-D"):
    fn(np.ones((2, 2, 2, 2, 2), np.float32), stacked=True)


@pytest.mark.parametrize("name", FNS)
@pytest.mark.parametrize("order", ["C", "F"])
def test_empty_arrays_need_no_device(no_device_use, name, order):
  fn = getattr(no_device_use, name)
  for shape, stacked in (((0,), False), ((3, 0, 2), False), ((0, 4, 4), True), ((2, 3, 0, 1), True)):
    arr = np.zeros(shape, np.int16, order=order)
    got = fn(arr, stacked=stacked)
    assert isinstance(got, np.ndarray) and got.shape == shape and got.dtype == np.float32
    if len(shape) > 1 and order == "F":
      assert got.flags.f_contiguous
  assert fn([]).shape == (0,)


@pytest.mark.parametrize("name", FNS)
def test_docstrings_give_the_definition_and_the_worked_uses(edt, name):
  doc = getattr(edt, name).__doc__
  for text in ("fl32(fl64(fl64(w2 * (i-j)^2) + g(j)))", "w2 = float32(w * w)", "NaN", "+0.0", "overflows",
               "-inf", "parabolic_erode(np.where(mask, np.inf, 0), w) == edtsq(mask, w)",
               "parabolic_dilate(np.where(medial, r * r, -np.inf)) > 0", "anisotropy = s / sqrt(2 t)"):
    assert text in doc, text
