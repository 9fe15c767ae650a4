"""CPU tests: the argument checks of edtb200_fill_holes and edtb200_dust in their documented order and the
header's parameter names, and the Python rejections of fill_holes and dust -- each before any device is
touched.  A fully valid call stops at the device probe (abi_checks.expect_probe)."""
import inspect
import re

import numpy as np
import pytest

from abi_checks import (ABI_VERSION, BIG, BOTH, EINVAL, ELIMIT, HEADER, LABELS_FLOAT, LABELS_ON_DEVICE, PROBE, SQRT,
                        check_case, header_doc, no_device_use, prototypes)

_LAB = np.zeros(128, np.uint32)          # 2 volumes of 4 x 4 x 4
_OUT = np.zeros(128, np.uint32)
_CNT = np.zeros(2, np.int64)
LAB, OUT, CNT = (a.ctypes.data for a in (_LAB, _OUT, _CNT))


def _fill_args(labels=LAB, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, count=2, connectivity=1, max_size=-1, flags=BOTH,
               out=OUT, fill_counts=CNT, device=63, stream=None):
  return (labels, label_bytes, ndim, sx, sy, sz, count, connectivity, max_size, flags, out, fill_counts, device, stream)


def _dust_args(labels=LAB, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, count=2, connectivity=1, threshold=3, invert=0,
               flags=BOTH, out=OUT, device=63, stream=None):
  return (labels, label_bytes, ndim, sx, sy, sz, count, connectivity, threshold, invert, flags, out, device, stream)


# the checks both entry points make in the same order around their own
SHARED = [
  ("label_bytes_0", dict(label_bytes=0), EINVAL, "label_bytes must be 1, 2, 4 or 8"),
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes must be 1, 2, 4 or 8"),
  ("label_width_before_ndim", dict(label_bytes=5, ndim=0), EINVAL, "label_bytes must be"),
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
  ("too_many_voxels", dict(count=1 << 60), ELIMIT, "too many voxels"),
  ("volume_of_2_to_the_32", dict(sx=1 << 12, sy=1 << 10, sz=1 << 10, count=1), ELIMIT,
   "volumes of fewer than 2^32 voxels"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_out", dict(out=None), EINVAL, "null pointer"),
  ("out_overlaps_labels", dict(out=LAB + 8), EINVAL, "out overlaps labels"),
  ("out_overlaps_labels_host", dict(out=LAB - 512 + 4, flags=0), EINVAL, "out overlaps labels"),
  ("size_before_count", dict(sx=BIG, count=-1), ELIMIT, "axis longer"),
  ("count_before_connectivity", dict(count=-1, connectivity=0), EINVAL, "negative count"),
  ("stack_before_volume", dict(sx=1 << 30, sy=1 << 30, sz=1, count=1 << 10), ELIMIT, "too many voxels"),
  ("volume_limit_before_empty", dict(sx=1 << 12, sy=1 << 10, sz=1 << 10, count=0, out=None), ELIMIT, "2^32"),
  ("no_volumes", dict(count=0, labels=None, out=None), 0, ""),
  ("empty_volume", dict(sz=0, labels=None, out=None, flags=0), 0, ""),
  ("pointers_before_overlap", dict(labels=None, out=LAB), EINVAL, "null pointer"),
  ("overlap_before_device", dict(out=LAB, device=64), EINVAL, "out overlaps labels"),
  ("valid", dict(), PROBE, ""),
  ("valid_host", dict(flags=0), PROBE, ""),
  ("valid_1_byte_labels", dict(label_bytes=1), PROBE, ""),
  ("valid_8_byte_labels", dict(label_bytes=8, count=1), PROBE, ""),
  ("valid_connectivity_3", dict(connectivity=3), PROBE, ""),
  ("valid_mixed_output_on_labels", dict(out=LAB, flags=LABELS_ON_DEVICE), PROBE, ""),
  ("valid_stack_past_2_to_the_32", dict(sx=1 << 10, sy=1 << 10, sz=1 << 10, count=8, flags=LABELS_ON_DEVICE),
   PROBE, ""),
  ("valid_1d", dict(ndim=1, sy=-1, sz=-1), PROBE, ""),
  ("valid_2d_connectivity_2", dict(ndim=2, sz=-1, connectivity=2), PROBE, ""),
]

FILL_CASES = [c for c in SHARED if c[0] != "valid_stack_past_2_to_the_32"] + [
  ("valid_stack_past_2_to_the_32", dict(sx=1 << 10, sy=1 << 10, sz=1 << 10, count=8, flags=LABELS_ON_DEVICE,
                                        fill_counts=None), PROBE, ""),
  ("max_size_minus_2", dict(max_size=-2), EINVAL, "max_size must be -1 (none) or >= 0"),
  ("connectivity_before_max_size", dict(connectivity=0, max_size=-2), EINVAL, "connectivity must be"),
  ("max_size_before_flags", dict(max_size=-2, flags=SQRT), EINVAL, "max_size must be"),
  ("counts_overlap_out", dict(fill_counts=OUT + 8), EINVAL, "fill_counts overlaps out"),
  ("counts_overlap_labels", dict(fill_counts=LAB + 8), EINVAL, "fill_counts overlaps labels"),
  ("valid_max_size_0", dict(max_size=0), PROBE, ""),
  ("valid_max_size_large", dict(max_size=(1 << 63) - 1), PROBE, ""),
  ("valid_no_counts", dict(fill_counts=None), PROBE, ""),
  ("valid_counts_on_labels_mixed", dict(fill_counts=LAB, flags=LABELS_ON_DEVICE), PROBE, ""),
]

DUST_CASES = SHARED + [
  ("threshold_negative", dict(threshold=-1), EINVAL, "threshold must be >= 0"),
  ("invert_2", dict(invert=2), EINVAL, "invert must be 0 or 1"),
  ("connectivity_before_threshold", dict(connectivity=0, threshold=-1), EINVAL, "connectivity must be"),
  ("threshold_before_invert", dict(threshold=-1, invert=2), EINVAL, "threshold must be"),
  ("invert_before_flags", dict(invert=-1, flags=SQRT), EINVAL, "invert must be"),
  ("valid_threshold_0", dict(threshold=0), PROBE, ""),
  ("valid_invert", dict(invert=1), PROBE, ""),
  ("valid_threshold_large", dict(threshold=(1 << 63) - 1), PROBE, ""),
]


@pytest.mark.parametrize("case,overrides,rc,msg", FILL_CASES, ids=[c[0] for c in FILL_CASES])
def test_fill_holes_argument_check(edt, case, overrides, rc, msg):
  check_case(edt, edt._lib().edtb200_fill_holes, _fill_args, overrides, rc, msg)


@pytest.mark.parametrize("case,overrides,rc,msg", DUST_CASES, ids=[c[0] for c in DUST_CASES])
def test_dust_argument_check(edt, case, overrides, rc, msg):
  check_case(edt, edt._lib().edtb200_dust, _dust_args, overrides, rc, msg)


def test_the_header_names_the_parameters():
  names = lambda fn: [re.sub(r"[*\s]", "", p.rsplit(" ", 1)[1]) for p in prototypes()[fn][1]]
  assert names("edtb200_fill_holes") == ["labels", "label_bytes", "ndim", "sx", "sy", "sz", "count", "connectivity",
                                         "max_size", "flags", "out", "fill_counts", "device", "stream"]
  assert names("edtb200_dust") == ["labels", "label_bytes", "ndim", "sx", "sy", "sz", "count", "connectivity",
                                   "threshold", "invert", "flags", "out", "device", "stream"]
  assert "int64_t *fill_counts" in prototypes()["edtb200_fill_holes"][1][11]


def test_the_header_documents_an_addition_at_the_same_version(edt):
  assert edt._lib().edtb200_version() == ABI_VERSION
  for fn in ("edtb200_fill_holes", "edtb200_dust"):
    assert fn in HEADER[:HEADER.index("#define EDTB200_VERSION")]
  doc = header_doc("edtb200_fill_holes")
  for text in ("at most `connectivity` of its components are non-zero", "Labels compare by their bits",
               "contains a voxel on a face of its volume", "whose only bordering label is L",
               "scipy.ndimage.binary_fill_holes", "stays 0", "atomicCAS(claim, 0, L)", "MIXED",
               "4 bytes per voxel of parents", "1 byte per voxel of state", "fewer than 2^32 voxels",
               "EDT_B200_VERBOSE", "fewer than `threshold` voxels"):
    assert text in doc, text


# ---- Python ---------------------------------------------------------------------------------------------

def test_signatures(edt):
  p = inspect.signature(edt.fill_holes).parameters
  assert list(p) == ["labels", "connectivity", "max_size", "return_fill_count", "stacked", "device"]
  assert p["max_size"].default is None and p["return_fill_count"].default is False
  p = inspect.signature(edt.dust).parameters
  assert list(p) == ["labels", "threshold", "connectivity", "invert", "stacked", "device"]
  assert p["connectivity"].default == 1 and p["invert"].default is False
  for name in ("fill_holes", "dust"):
    assert name in edt.__all__


@pytest.mark.parametrize("bad", [1.0, True, "3", np.float32(2), np.ones(2)])
def test_rejects_a_bound_that_is_not_an_int(no_device_use, bad):
  with pytest.raises(TypeError, match="max_size must be an int"):
    no_device_use.fill_holes(np.zeros((4, 5), np.uint8), max_size=bad)
  with pytest.raises(TypeError, match="threshold must be an int"):
    no_device_use.dust(np.zeros((4, 5), np.uint8), bad)


@pytest.mark.parametrize("bad", [-1, np.int64(-5)])
def test_rejects_a_negative_bound(no_device_use, bad):
  with pytest.raises(ValueError, match="max_size must be >= 0"):
    no_device_use.fill_holes(np.zeros((4, 5), np.uint8), max_size=bad)
  with pytest.raises(ValueError, match="threshold must be >= 0"):
    no_device_use.dust(np.zeros((4, 5), np.uint8), bad)


@pytest.mark.parametrize("bad", [1, None, "yes"])
def test_rejects_flags_that_are_not_bools(no_device_use, bad):
  with pytest.raises(TypeError, match="return_fill_count must be True or False"):
    no_device_use.fill_holes(np.zeros((4, 5), np.uint8), return_fill_count=bad)
  with pytest.raises(TypeError, match="invert must be True or False"):
    no_device_use.dust(np.zeros((4, 5), np.uint8), 2, invert=bad)


@pytest.mark.parametrize("shape,conn", [((4, 5), 0), ((4, 5), 3), ((6,), 2), ((3, 4, 5), 4), ((3, 4, 5), 1.0)])
def test_rejects_a_bad_connectivity(no_device_use, shape, conn):
  err = TypeError if isinstance(conn, float) else ValueError
  with pytest.raises(err, match="connectivity must be"):
    no_device_use.fill_holes(np.zeros(shape, np.uint8), connectivity=conn)
  with pytest.raises(err, match="connectivity must be"):
    no_device_use.dust(np.zeros(shape, np.uint8), 2, connectivity=conn)


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.float16, np.complex64, object])
def test_rejects_an_unsupported_label_dtype(no_device_use, dtype):
  with pytest.raises(TypeError, match="fill_holes: unsupported label dtype"):
    no_device_use.fill_holes(np.zeros((4, 5), dtype))
  with pytest.raises(TypeError, match="dust: unsupported label dtype"):
    no_device_use.dust(np.zeros((4, 5), dtype), 2)


@pytest.mark.parametrize("shape,stacked", [((), False), ((2, 2, 2, 2), False), ((4,), True)])
def test_rejects_a_wrong_number_of_dimensions(no_device_use, shape, stacked):
  with pytest.raises(TypeError, match="-D to"):
    no_device_use.fill_holes(np.zeros(shape, np.uint8), stacked=stacked)
  with pytest.raises(TypeError, match="-D to"):
    no_device_use.dust(np.zeros(shape, np.uint8), 2, stacked=stacked)


@pytest.mark.parametrize("order", ["C", "F"])
def test_empty_arrays_need_no_device(no_device_use, order):
  for shape, stacked in (((0, 3), False), ((3, 0, 2), False), ((0, 4, 4), True), ((0,), False)):
    out, n = no_device_use.fill_holes(np.zeros(shape, np.int16, order=order), return_fill_count=True, stacked=stacked)
    assert isinstance(out, np.ndarray) and out.shape == shape and out.dtype == np.int16
    assert (n.shape == (0,) and n.dtype == np.int64) if stacked else n == 0
    out = no_device_use.dust(np.zeros(shape, np.bool_, order=order), 3, stacked=stacked)
    assert out.shape == shape and out.dtype == np.bool_


def test_docstrings_state_the_definitions(edt):
  fill = " ".join(edt.fill_holes.__doc__.split())
  dust = " ".join(edt.dust.__doc__.split())
  for text in ("at most `connectivity` of its components are non-zero", "it has a voxel on a face of its volume",
               "whose only bordering label is L", "exactly scipy.ndimage.binary_fill_holes(mask",
               "fill_holes(labels == L)", "stays 0", "a nucleus (label 2)", "an int for one volume",
               "int64 array with one entry per volume", "without a host synchronisation", "ELIMIT",
               "1 byte per voxel of state", "compare by their bits"):
    assert " ".join(text.split()) in fill, text
  for text in ("FEWER than `threshold` voxels", "exactly `threshold` voxels is kept", "invert=True",
               "skimage versions disagree", "cc3d's default of 26 neighbours is connectivity=3",
               "4 bytes per voxel of sizes"):
    assert " ".join(text.split()) in dust, text
