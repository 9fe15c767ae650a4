"""CPU tests: the argument checks of edtb200_local_thickness, in their documented order, and the Python
rejections of local_thickness.

As in test_morphology_arguments.py, every rejection comes with a return code and a message before any
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

MAX_SIZES = 4096

_IN = np.zeros(512, np.uint64)
_OUT = np.zeros(512, np.uint64)
_LEVELS = np.zeros(64, np.float64)
IN, OUT, LEVELS = _IN.ctypes.data, _OUT.ctypes.data, _LEVELS.ctypes.data
_SIZES = np.array([2.0, 0.5, 1.0], np.float64)
SIZES = _SIZES.ctypes.data
_BAD = {name: np.array([1.0, v], np.float64) for name, v in
        (("nan", np.nan), ("inf", np.inf), ("minus_inf", -np.inf), ("negative", -0.25))}


def _args(labels=IN, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, count=2, w=(1.0, 1.0, 1.0), black_border=0,
          flags=BOTH, sizes=SIZES, nsizes=3, out=OUT, sizes_out=None, device=63, stream=None):
  return (labels, label_bytes, ndim, sx, sy, sz, count, w[0], w[1], w[2], black_border, flags, sizes, nsizes, out,
          sizes_out, device, stream)


def _bad(name):
  return _BAD[name].ctypes.data


CASES = [
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes"),
  ("ndim_0", dict(ndim=0), EINVAL, "ndim"),
  ("ndim_4", dict(ndim=4), EINVAL, "ndim"),
  ("negative_size", dict(sy=-1), EINVAL, "negative size"),
  ("axis_too_long", dict(sx=BIG), ELIMIT, "axis longer than 2^30"),
  ("negative_count", dict(count=-1), EINVAL, "negative count"),
  ("weight_zero", dict(w=(1.0, 0.0, 1.0)), EINVAL, "weight of axis 1"),
  ("weight_negative", dict(w=(-1.0, 1.0, 1.0)), EINVAL, "weight of axis 0"),
  ("weight_nan", dict(w=(1.0, 1.0, float("nan"))), EINVAL, "weight of axis 2"),
  ("nsizes_0", dict(nsizes=0), EINVAL, "nsizes must be 1 to 4096"),
  ("nsizes_negative", dict(nsizes=-3, sizes=None), EINVAL, "nsizes must be"),
  ("nsizes_above_limit", dict(nsizes=MAX_SIZES + 1, sizes=None), EINVAL, "nsizes must be"),
  ("size_nan", dict(sizes=_bad("nan"), nsizes=2), EINVAL, "sizes[1] must be finite"),
  ("size_inf", dict(sizes=_bad("inf"), nsizes=2), EINVAL, "sizes[1] must be finite"),
  ("size_minus_inf", dict(sizes=_bad("minus_inf"), nsizes=2), EINVAL, "sizes[1] must be finite"),
  ("size_negative", dict(sizes=_bad("negative"), nsizes=2), EINVAL, "sizes[1] must be finite"),
  ("flag_sqrt", dict(flags=BOTH | SQRT), EINVAL, "residency flags"),
  ("flag_signed", dict(flags=SIGNED), EINVAL, "residency flags"),
  ("float_1_byte", dict(label_bytes=1, flags=BOTH | LABELS_FLOAT), EINVAL, "4- or 8-byte"),
  ("too_many_voxels", dict(count=1 << 60), ELIMIT, "too many voxels"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_out", dict(out=None), EINVAL, "null pointer"),
  ("out_overlaps_labels", dict(out=IN + 8, flags=0), EINVAL, "out overlaps labels"),
  ("sizes_out_overlaps_out", dict(sizes_out=OUT + 16), EINVAL, "sizes_out overlaps out"),
  ("sizes_out_overlaps_labels", dict(sizes_out=IN), EINVAL, "sizes_out overlaps labels"),
  # order: label width, ndim, sizes, count, weights, nsizes, radii, flags, float width, stack size,
  # emptiness, pointers and overlap, device
  ("label_bytes_before_ndim", dict(label_bytes=3, ndim=4), EINVAL, "label_bytes"),
  ("ndim_before_size", dict(ndim=5, sx=-1), EINVAL, "ndim"),
  ("size_before_count", dict(sx=BIG, count=-1), ELIMIT, "axis longer"),
  ("count_before_weights", dict(count=-1, w=(0.0, 1.0, 1.0)), EINVAL, "negative count"),
  ("weights_before_nsizes", dict(w=(0.0, 1.0, 1.0), nsizes=0), EINVAL, "weight of axis 0"),
  ("nsizes_before_radii", dict(nsizes=0, sizes=_bad("nan")), EINVAL, "nsizes must be"),
  ("radii_before_flags", dict(sizes=_bad("negative"), nsizes=2, flags=SQRT), EINVAL, "sizes[1]"),
  ("flags_before_float_width", dict(flags=SQRT | LABELS_FLOAT, label_bytes=2), EINVAL, "residency flags"),
  ("float_width_before_stack", dict(flags=LABELS_FLOAT, label_bytes=1, count=1 << 60), EINVAL, "4- or 8-byte"),
  ("stack_before_empty", dict(count=1 << 60, sz=1), ELIMIT, "too many voxels"),
  ("radii_before_empty", dict(sizes=_bad("inf"), nsizes=2, count=0), EINVAL, "sizes[1]"),
  ("empty_before_pointers", dict(count=0, labels=None, out=None), 0, ""),
  ("empty_volume", dict(sz=0, labels=None, out=None, flags=0), 0, ""),
  ("pointers_before_overlap", dict(labels=None, sizes_out=OUT), EINVAL, "null pointer"),
  ("valid", dict(), PROBE, ""),
  ("valid_default_levels", dict(sizes=None, nsizes=25), PROBE, ""),
  ("valid_sizes_out", dict(sizes=None, nsizes=4, sizes_out=LEVELS), PROBE, ""),
  ("valid_host", dict(flags=0, sizes_out=LEVELS), PROBE, ""),
  ("valid_mixed", dict(flags=LABELS_ON_DEVICE), PROBE, ""),
  ("valid_float_8", dict(label_bytes=8, flags=LABELS_FLOAT), PROBE, ""),
  ("valid_max_sizes", dict(sizes=None, nsizes=MAX_SIZES), PROBE, ""),
  ("valid_level_0", dict(sizes=_LEVELS.ctypes.data, nsizes=1), PROBE, ""),
  ("valid_2d_ignores_sz_and_wz", dict(ndim=2, sz=-1, w=(1.0, 1.0, 0.0)), PROBE, ""),
  ("valid_1d_ignores_sy_sz", dict(ndim=1, sy=-1, sz=BIG, w=(2.0, -1.0, 0.0)), PROBE, ""),
]


@pytest.mark.parametrize("case,overrides,rc,msg", CASES, ids=[c[0] for c in CASES])
def test_local_thickness_argument_check(edt, case, overrides, rc, msg):
  check_case(edt, edt._lib().edtb200_local_thickness, _args, overrides, rc, msg)


def test_local_thickness_is_an_addition_at_the_same_version(edt):
  lib = edt._lib()
  assert lib.edtb200_version() == ABI_VERSION
  assert "edtb200_local_thickness" in set(re.findall(r"\b(edtb200_[a-z0-9_]+)\s*\(", HEADER))
  version_comment = HEADER[:HEADER.index("#define EDTB200_VERSION")]
  assert "edtb200_local_thickness" in version_comment
  assert re.search(r"#define EDTB200_THICKNESS_MAX_SIZES\s+%d\b" % MAX_SIZES, HEADER)
  assert edt.THICKNESS_MAX_SIZES == MAX_SIZES
  assert hasattr(ctypes.CDLL(edt.library_path()), "edtb200_local_thickness")
  proto = re.search(r"int edtb200_local_thickness\(([^)]*)\)", HEADER).group(1)
  assert len(proto.split(",")) == len(lib.edtb200_local_thickness.argtypes) == 18


# ---- Python ---------------------------------------------------------------------------------------------

def test_exported(edt):
  assert "local_thickness" in edt.__all__
  params = inspect.signature(edt.local_thickness).parameters
  assert list(params)[:3] == ["labels", "anisotropy", "black_border"]
  for kw, default in (("sizes", 25), ("return_sizes", False), ("device", 0), ("stacked", False)):
    assert params[kw].kind is inspect.Parameter.KEYWORD_ONLY and params[kw].default == default, kw
  assert "radius" in edt.local_thickness.__doc__.lower() and "twice" in edt.local_thickness.__doc__


@pytest.mark.parametrize("sizes,match", [
  ([], "non-empty 1-D"), (np.zeros((2, 2)), "non-empty 1-D"), (2.5, "non-empty 1-D"),
  ([1.0, float("nan")], "finite and zero or more"), ([1.0, -0.5], "finite and zero or more"),
  ([float("inf")], "finite and zero or more"), (0, "1 to 4096"), (-3, "1 to 4096"), (MAX_SIZES + 1, "1 to 4096"),
  (np.arange(MAX_SIZES + 1, dtype=np.float64), "at most 4096 distinct"),
])
def test_rejects_bad_sizes(no_device_use, sizes, match):
  with pytest.raises(ValueError, match=match):
    no_device_use.local_thickness(np.ones((4, 5), np.uint8), sizes=sizes)


@pytest.mark.parametrize("sizes", [True, "abc", ["a", "b"], [1j]])
def test_rejects_sizes_of_the_wrong_type(no_device_use, sizes):
  with pytest.raises(TypeError, match="sizes must be an integer or a 1-D sequence"):
    no_device_use.local_thickness(np.ones((4, 5), np.uint8), sizes=sizes)


def test_rejects_bad_sizes_before_anything_else(no_device_use):
  with pytest.raises(ValueError, match="every size must be finite"):
    no_device_use.local_thickness(np.ones((2, 2, 2, 2, 2), np.complex64), (0.0, 1.0, 2.0, 3.0), sizes=[-1.0])


@pytest.mark.parametrize("w", [(0.0, 1.0), (1.0, -2.0), (float("nan"), 1.0), (float("inf"), 1.0)])
def test_rejects_bad_weights(no_device_use, w):
  with pytest.raises(ValueError, match="finite and > 0"):
    no_device_use.local_thickness(np.ones((4, 5), np.uint8), w)


def test_rejects_anisotropy_of_the_wrong_length(no_device_use):
  with pytest.raises(ValueError, match="one entry per volume axis"):
    no_device_use.local_thickness(np.ones((4, 5), np.uint8), (1.0, 2.0, 3.0))


@pytest.mark.parametrize("dtype", [np.float16, np.complex64, np.object_, np.dtype("U3"), np.dtype("V4")])
def test_rejects_unsupported_dtype(no_device_use, dtype):
  with pytest.raises(TypeError, match="unsupported label dtype"):
    no_device_use.local_thickness(np.zeros((3, 4), dtype))


def test_rejects_dimension_counts_and_flags(no_device_use):
  fn = no_device_use.local_thickness
  with pytest.raises(TypeError, match="1-D to 3-D"):
    fn(np.uint8(3))
  with pytest.raises(TypeError, match="1-D to 3-D"):
    fn(np.ones((2, 2, 2, 2), np.uint8))
  with pytest.raises(TypeError, match="2-D to 4-D"):
    fn(np.ones(5, np.uint8), stacked=True)
  with pytest.raises(TypeError, match="return_sizes must be True or False"):
    fn(np.ones((2, 2), np.uint8), return_sizes=1)


@pytest.mark.parametrize("order", ["C", "F"])
def test_empty_arrays_need_no_device(no_device_use, order):
  fn = no_device_use.local_thickness
  for shape, stacked in (((0,), False), ((3, 0, 2), False), ((0, 4, 4), True), ((2, 3, 0, 1), True),
                         ((3, 0, 5), True)):
    arr = np.zeros(shape, np.int32, order=order)
    # the slowest axis in memory counts the volumes (C where the array is both)
    count = (shape[0] if arr.flags.c_contiguous else shape[-1]) if stacked else 1
    got, levels = fn(arr, (2.0,) * (len(shape) - stacked), sizes=4, stacked=stacked, return_sizes=True)
    assert isinstance(got, np.ndarray) and got.shape == shape and got.dtype == np.float32
    if len(shape) > 1 and order == "F":
      assert got.flags.f_contiguous
    assert levels.shape == ((count, 4) if stacked else (4,)) and np.all(levels == 1.0)
    got, levels = fn(arr, sizes=[1.0, 3.0, 1.0], stacked=stacked, return_sizes=True)
    assert got.shape == shape and list(levels) == [3.0, 1.0]
