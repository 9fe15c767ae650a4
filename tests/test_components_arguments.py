"""CPU tests: the argument checks of edtb200_connected_components and edtb200_extended_maxima in their
documented order and the header's parameter names, and the Python rejections of connected_components and
extended_maxima -- each before any device is touched.  A fully valid call stops at the device probe
(abi_checks.expect_probe)."""
import inspect
import re

import numpy as np
import pytest

from abi_checks import (ABI_VERSION, BIG, BOTH, EINVAL, ELIMIT, HEADER, LABELS_FLOAT, LABELS_ON_DEVICE, PROBE, SQRT,
                        check_case, header_doc, no_device_use, prototypes)

_LAB = np.zeros(128, np.uint32)          # 2 volumes of 4 x 4 x 4
_IMG = np.zeros(128, np.float32)
_OUT = np.zeros(128, np.int64)
LAB, IMG, OUT = (a.ctypes.data for a in (_LAB, _IMG, _OUT))


def _cc_args(labels=LAB, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, count=2, connectivity=1, flags=BOTH, out=OUT,
             out_bytes=4, device=63, stream=None):
  return (labels, label_bytes, ndim, sx, sy, sz, count, connectivity, flags, out, out_bytes, device, stream)


def _em_args(labels=LAB, label_bytes=4, image=IMG, ndim=3, sx=4, sy=4, sz=4, count=2, h=0.5, connectivity=1,
             flags=BOTH, out=OUT, out_bytes=4, device=63, stream=None):
  return (labels, label_bytes, image, ndim, sx, sy, sz, count, h, connectivity, flags, out, out_bytes, device, stream)


# the checks both entry points make in the same order after their own
SHARED = [
  ("ndim_0", dict(ndim=0), EINVAL, "ndim must be 1, 2 or 3"),
  ("ndim_4", dict(ndim=4), EINVAL, "ndim must be 1, 2 or 3"),
  ("negative_size", dict(sy=-1), EINVAL, "negative size"),
  ("axis_too_long", dict(sz=BIG), ELIMIT, "axis longer than 2^30"),
  ("negative_count", dict(count=-1), EINVAL, "negative count"),
  ("connectivity_0", dict(connectivity=0), EINVAL, "connectivity must be 1 to ndim (3)"),
  ("connectivity_4", dict(connectivity=4), EINVAL, "connectivity must be 1 to ndim (3)"),
  ("connectivity_3_in_2d", dict(ndim=2, connectivity=3), EINVAL, "connectivity must be 1 to ndim (2)"),
  ("flag_sqrt", dict(flags=BOTH | SQRT), EINVAL, "only the residency flags"),
  ("flag_float", dict(flags=LABELS_FLOAT), EINVAL, "only the residency flags"),
  ("out_bytes_2", dict(out_bytes=2), EINVAL, "out_bytes must be 4 or 8"),
  ("out_bytes_0", dict(out_bytes=0), EINVAL, "out_bytes must be 4 or 8"),
  ("too_many_voxels", dict(count=1 << 60), ELIMIT, "too many voxels"),
  ("volume_of_2_to_the_32", dict(sx=1 << 12, sy=1 << 10, sz=1 << 10, count=1, out_bytes=8), ELIMIT,
   "volumes of fewer than 2^32 voxels"),
  ("int32_volume_of_2_to_the_31", dict(sx=1 << 11, sy=1 << 10, sz=1 << 10, count=1), EINVAL,
   "out_bytes 4 needs volumes of fewer than 2^31 voxels"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_out", dict(out=None), EINVAL, "null pointer"),
  ("out_overlaps_labels", dict(out=LAB + 8), EINVAL, "out overlaps labels"),
  ("out_overlaps_labels_host", dict(out=LAB - 256 + 4, flags=0), EINVAL, "out overlaps labels"),
  # order: ndim, sizes, count, connectivity, flags, out_bytes, stack size, volume size, output width,
  # emptiness, pointers, overlap, device
  ("ndim_before_size", dict(ndim=5, sx=-1), EINVAL, "ndim"),
  ("size_before_count", dict(sx=BIG, count=-1), ELIMIT, "axis longer"),
  ("count_before_connectivity", dict(count=-1, connectivity=0), EINVAL, "negative count"),
  ("connectivity_before_flags", dict(connectivity=9, flags=SQRT), EINVAL, "connectivity must be"),
  ("flags_before_out_bytes", dict(flags=SQRT, out_bytes=3), EINVAL, "only the residency flags"),
  ("out_bytes_before_stack", dict(out_bytes=3, count=1 << 60), EINVAL, "out_bytes must be"),
  ("stack_before_volume", dict(sx=1 << 30, sy=1 << 30, sz=1, count=1 << 10), ELIMIT, "too many voxels"),
  ("volume_before_width", dict(sx=1 << 12, sy=1 << 10, sz=1 << 10, count=1), ELIMIT, "fewer than 2^32"),
  ("volume_limit_before_empty", dict(sx=1 << 12, sy=1 << 10, sz=1 << 10, count=0, out=None), ELIMIT, "2^32"),
  ("no_volumes", dict(count=0, labels=None, out=None), 0, ""),
  ("empty_volume", dict(sz=0, labels=None, out=None, flags=0), 0, ""),
  ("pointers_before_overlap", dict(labels=None, out=LAB), EINVAL, "null pointer"),
  ("overlap_before_device", dict(out=LAB, device=64), EINVAL, "out overlaps labels"),
  ("valid", dict(), PROBE, ""),
  ("valid_host", dict(flags=0), PROBE, ""),
  ("valid_int64", dict(out_bytes=8), PROBE, ""),
  ("valid_int64_volume_of_2_to_the_31", dict(sx=1 << 11, sy=1 << 10, sz=1 << 10, count=1, out_bytes=8,
                                             flags=LABELS_ON_DEVICE), PROBE, ""),
  ("valid_int32_stack_past_2_to_the_32", dict(sx=1 << 10, sy=1 << 10, sz=1 << 10, count=8, flags=LABELS_ON_DEVICE),
   PROBE, ""),
  ("valid_8_byte_labels", dict(label_bytes=8, count=1), PROBE, ""),
  ("valid_connectivity_3", dict(connectivity=3), PROBE, ""),
  ("valid_mixed_output_on_labels", dict(out=LAB, flags=LABELS_ON_DEVICE), PROBE, ""),
  ("valid_1d", dict(ndim=1, sy=-1, sz=-1), PROBE, ""),
  ("valid_2d_connectivity_2", dict(ndim=2, sz=-1, connectivity=2), PROBE, ""),
]

CC_CASES = [
  ("label_bytes_0", dict(label_bytes=0), EINVAL, "label_bytes must be 1, 2, 4 or 8"),
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes must be 1, 2, 4 or 8"),
  ("label_width_before_ndim", dict(label_bytes=5, ndim=0), EINVAL, "label_bytes must be"),
] + SHARED

EM_CASES = [
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes must be 0 (no labels), 1, 2, 4 or 8"),
  ("label_bytes_16", dict(label_bytes=16), EINVAL, "label_bytes must be 0"),
  ("label_width_before_ndim", dict(label_bytes=5, ndim=0), EINVAL, "label_bytes must be"),
  ("h_negative", dict(h=-0.5), EINVAL, "h must be finite and >= 0"),
  ("h_nan", dict(h=float("nan")), EINVAL, "h must be finite and >= 0"),
  ("h_inf", dict(h=float("inf")), EINVAL, "h must be finite and >= 0"),
  ("count_before_h", dict(count=-1, h=-1.0), EINVAL, "negative count"),
  ("h_before_connectivity", dict(h=-1.0, connectivity=0), EINVAL, "h must be"),
  ("too_many_tiles", dict(ndim=1, sx=1, count=1 << 32, labels=None, label_bytes=0), ELIMIT, "fewer than 2^32 tiles"),
  ("tiles_only_with_h", dict(ndim=1, sx=1, count=1 << 32, label_bytes=0, h=0.0, image=None), EINVAL, "null pointer"),
  ("tiles_before_empty", dict(ndim=1, sx=1, count=1 << 33, label_bytes=0, image=None, out=None), ELIMIT, "tiles"),
  ("null_image", dict(image=None), EINVAL, "null pointer"),
  ("out_overlaps_image", dict(out=IMG + 4), EINVAL, "out overlaps image"),
  ("valid_no_labels", dict(label_bytes=0, labels=None), PROBE, ""),
  ("valid_no_labels_ignores_the_pointer", dict(label_bytes=0, labels=OUT + 1), PROBE, ""),
  ("valid_h_0", dict(h=0.0), PROBE, ""),
  ("valid_h_negative_zero", dict(h=-0.0), PROBE, ""),
] + [c for c in SHARED if c[0] not in ("no_volumes", "empty_volume", "pointers_before_overlap", "null_labels")] + [
  ("no_volumes", dict(count=0, labels=None, image=None, out=None), 0, ""),
  ("empty_volume", dict(sz=0, labels=None, image=None, out=None, flags=0), 0, ""),
  ("pointers_before_overlap", dict(image=None, out=LAB), EINVAL, "null pointer"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
]


@pytest.mark.parametrize("case,overrides,rc,msg", CC_CASES, ids=[c[0] for c in CC_CASES])
def test_connected_components_argument_check(edt, case, overrides, rc, msg):
  check_case(edt, edt._lib().edtb200_connected_components, _cc_args, overrides, rc, msg)


@pytest.mark.parametrize("case,overrides,rc,msg", EM_CASES, ids=[c[0] for c in EM_CASES])
def test_extended_maxima_argument_check(edt, case, overrides, rc, msg):
  check_case(edt, edt._lib().edtb200_extended_maxima, _em_args, overrides, rc, msg)


def test_the_header_names_the_parameters():
  names = lambda fn: [re.sub(r"[*\s]", "", p.rsplit(" ", 1)[1]) for p in prototypes()[fn][1]]
  assert names("edtb200_connected_components") == ["labels", "label_bytes", "ndim", "sx", "sy", "sz", "count",
                                                   "connectivity", "flags", "out", "out_bytes", "device", "stream"]
  assert names("edtb200_extended_maxima") == ["labels", "label_bytes", "image", "ndim", "sx", "sy", "sz", "count",
                                              "h", "connectivity", "flags", "out", "out_bytes", "device", "stream"]
  assert "double h" in prototypes()["edtb200_extended_maxima"][1][8]


def test_the_header_documents_an_addition_at_the_same_version(edt):
  assert edt._lib().edtb200_version() == ABI_VERSION
  for fn in ("edtb200_connected_components", "edtb200_extended_maxima"):
    assert fn in HEADER[:HEADER.index("#define EDTB200_VERSION")]
  doc = header_doc("edtb200_connected_components")
  for text in ("neighbours under `connectivity` with the SAME label", "least voxel index in memory order",
               "scipy.ndimage.label's numbering", "NaN read as -inf and -0.0 as +0.0", "m = fl32(fl64(f) - h)",
               "R[v] = max(R[v], min(f[v], R[u]))", "R[u] == R[v]", "hanging the larger root under the smaller",
               "4 bytes per voxel of parents", "12 bytes per tile", "fewer than 2^32 voxels", "EDT_B200_VERBOSE"):
    assert text in doc, text


# ---- Python ---------------------------------------------------------------------------------------------

def test_signatures(edt):
  p = inspect.signature(edt.connected_components).parameters
  assert list(p) == ["labels", "connectivity", "stacked", "device"]
  p = inspect.signature(edt.extended_maxima).parameters
  assert list(p) == ["image", "h", "labels", "connectivity", "stacked", "device"]
  assert p["h"].default == 0.0 and p["labels"].default is None
  for name in ("connected_components", "extended_maxima"):
    assert name in edt.__all__


@pytest.mark.parametrize("bad", [1.0, True, "1", None, np.ones(3)])
def test_rejects_a_connectivity_that_is_not_an_int(no_device_use, bad):
  with pytest.raises(TypeError, match="connectivity must be an int"):
    no_device_use.connected_components(np.zeros((4, 5), np.uint8), connectivity=bad)
  with pytest.raises(TypeError, match="connectivity must be an int"):
    no_device_use.extended_maxima(np.zeros((4, 5), np.float32), connectivity=bad)


@pytest.mark.parametrize("shape,conn", [((4, 5), 0), ((4, 5), 3), ((6,), 2), ((3, 4, 5), 4), ((3, 4, 5), -1)])
def test_rejects_a_connectivity_outside_1_to_ndim(no_device_use, shape, conn):
  with pytest.raises(ValueError, match="connectivity must be 1 to %d" % len(shape)):
    no_device_use.connected_components(np.zeros(shape, np.uint8), connectivity=conn)
  with pytest.raises(ValueError, match="connectivity must be 1 to %d" % len(shape)):
    no_device_use.extended_maxima(np.zeros(shape, np.float32), connectivity=conn)
  with pytest.raises(ValueError, match="connectivity must be 1 to 2"):
    no_device_use.connected_components(np.zeros((2, 4, 5), np.uint8), connectivity=3, stacked=True)


@pytest.mark.parametrize("h", [-1.0, -1e-30, float("nan"), float("inf"), -float("inf")])
def test_rejects_an_h_that_is_negative_or_not_finite(no_device_use, h):
  with pytest.raises(ValueError, match="h must be finite and >= 0"):
    no_device_use.extended_maxima(np.zeros((4, 5), np.float32), h)


@pytest.mark.parametrize("h", ["1", None, True, np.ones(2), 1j])
def test_rejects_an_h_that_is_not_a_real_number(no_device_use, h):
  with pytest.raises(TypeError, match="h must be a real number"):
    no_device_use.extended_maxima(np.zeros((4, 5), np.float32), h)


@pytest.mark.parametrize("shape,stacked", [((), False), ((2, 2, 2, 2), False), ((4,), True), ((2,) * 5, True)])
def test_rejects_a_wrong_number_of_dimensions(no_device_use, shape, stacked):
  with pytest.raises(TypeError, match="-D to"):
    no_device_use.connected_components(np.zeros(shape, np.uint8), stacked=stacked)
  with pytest.raises(TypeError, match="-D to"):
    no_device_use.extended_maxima(np.zeros(shape, np.float32), stacked=stacked)


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.float16, np.complex64, object, "U3"])
def test_rejects_an_unsupported_label_dtype(no_device_use, dtype):
  with pytest.raises(TypeError, match="connected_components: unsupported label dtype"):
    no_device_use.connected_components(np.zeros((4, 5), dtype))
  with pytest.raises(TypeError, match="extended_maxima: unsupported label dtype"):
    no_device_use.extended_maxima(np.zeros((4, 5), np.float32), 0.0, np.zeros((4, 5), dtype))


@pytest.mark.parametrize("dtype", [np.complex64, np.complex128, object, "U3"])
def test_rejects_an_image_that_is_not_real(no_device_use, dtype):
  with pytest.raises(TypeError, match="unsupported image dtype"):
    no_device_use.extended_maxima(np.zeros((4, 5), dtype), 0.0, np.zeros((4, 5), np.uint8))


def test_rejects_an_image_of_another_shape(no_device_use):
  with pytest.raises(ValueError, match="image must have the volume's shape"):
    no_device_use.extended_maxima(np.zeros((5, 4), np.float32), 0.0, np.zeros((4, 5), np.uint8))


@pytest.mark.parametrize("order", ["C", "F"])
def test_empty_arrays_need_no_device(no_device_use, order):
  for shape, stacked in (((0, 3), False), ((3, 0, 2), False), ((0, 4, 4), True), ((0,), False)):
    out = no_device_use.connected_components(np.zeros(shape, np.uint16, order=order), stacked=stacked)
    assert isinstance(out, np.ndarray) and out.shape == shape and out.dtype == np.int32
    out = no_device_use.extended_maxima(np.zeros(shape, np.float64, order=order), 1.0, stacked=stacked)
    assert isinstance(out, np.ndarray) and out.shape == shape and out.dtype == np.int32


def test_docstrings_state_the_definitions(edt):
  cc_doc = " ".join(edt.connected_components.__doc__.split())
  em_doc = " ".join(edt.extended_maxima.__doc__.split())
  for text in ("at most `connectivity` of its components are non-zero", "least voxel index in memory order",
               "scipy.ndimage.label's numbering", "cc3d's default of 26 is connectivity=3", "np.stack of the per-volume",
               "float labels are a TypeError", "int32 when each volume has fewer than 2^31 voxels", "ENOMEM",
               "without a host synchronisation", "4 bytes per voxel of parents"):
    assert " ".join(text.split()) in cc_doc, text
  for text in ("NaN read as -inf and -0.0 as +0.0", "m = fl32(fl64(f) - fl64(h))",
               "R[v] = max(R[v], min(f[v], R[u]))", "R[u] == R[v]", "its R is not -inf", "exceeds h",
               "h_maxima keeps dynamics >= h", "top plateau", "extended_maxima(-f, h)", "watershed(-dist, markers, mask)",
               "converted to float32 once", "12 bytes per tile"):
    assert " ".join(text.split()) in em_doc, text
