"""CPU tests: the argument checks of edtb200_watershed in their documented order and the header's parameter
names, the Python rejections of watershed -- each before any device is touched -- and the statements of
its docstring and the header.  A fully valid call stops at the device probe (abi_checks.expect_probe)."""
import inspect
import re

import numpy as np
import pytest

from abi_checks import (ABI_VERSION, BIG, BOTH, EINVAL, ELIMIT, HEADER, LABELS_FLOAT, LABELS_ON_DEVICE, PROBE, SQRT,
                        check_case, header_doc, no_device_use, prototypes)

_LAB = np.zeros(128, np.uint32)          # 2 volumes of 4 x 4 x 4
_MARK = np.zeros(128, np.uint8)
_IMG = np.zeros(128, np.float32)
_OUT = np.zeros(128, np.uint8)
_LEVEL = np.zeros(128, np.float32)
LAB, MARK, IMG, OUT, LEVEL = (a.ctypes.data for a in (_LAB, _MARK, _IMG, _OUT, _LEVEL))


def _args(labels=LAB, label_bytes=4, markers=MARK, marker_bytes=1, image=IMG, ndim=3, sx=4, sy=4, sz=4, count=2,
          connectivity=1, flags=BOTH, out=OUT, level=None, device=63, stream=None):
  return (labels, label_bytes, markers, marker_bytes, image, ndim, sx, sy, sz, count, connectivity, flags, out, level,
          device, stream)


CASES = [
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes must be 0 (no labels), 1, 2, 4 or 8"),
  ("label_bytes_16", dict(label_bytes=16), EINVAL, "label_bytes must be"),
  ("marker_bytes_0", dict(marker_bytes=0), EINVAL, "marker_bytes must be"),
  ("marker_bytes_3", dict(marker_bytes=3), EINVAL, "marker_bytes must be"),
  ("ndim_0", dict(ndim=0), EINVAL, "ndim must be 1, 2 or 3"),
  ("ndim_4", dict(ndim=4), EINVAL, "ndim must be 1, 2 or 3"),
  ("negative_size", dict(sy=-1), EINVAL, "negative size"),
  ("axis_too_long", dict(sz=BIG), ELIMIT, "axis longer than 2^30"),
  ("negative_count", dict(count=-1), EINVAL, "negative count"),
  ("connectivity_0", dict(connectivity=0), EINVAL, "connectivity must be 1 to ndim (3)"),
  ("connectivity_4", dict(connectivity=4), EINVAL, "connectivity must be 1 to ndim (3)"),
  ("connectivity_3_in_2d", dict(ndim=2, connectivity=3), EINVAL, "connectivity must be 1 to ndim (2)"),
  ("connectivity_2_in_1d", dict(ndim=1, connectivity=2), EINVAL, "connectivity must be 1 to ndim (1)"),
  ("flag_sqrt", dict(flags=BOTH | SQRT), EINVAL, "only the residency flags"),
  ("flag_float", dict(flags=LABELS_FLOAT), EINVAL, "only the residency flags"),
  ("too_many_voxels", dict(count=1 << 60), ELIMIT, "too many voxels"),
  ("too_many_tiles", dict(ndim=1, sx=1, count=1 << 32, labels=None), ELIMIT, "fewer than 2^32 tiles"),
  ("tiles_just_below", dict(ndim=1, sx=1, count=(1 << 32) - 1, labels=None), EINVAL, "null pointer"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_markers", dict(markers=None), EINVAL, "null pointer"),
  ("null_image", dict(image=None), EINVAL, "null pointer"),
  ("null_out", dict(out=None), EINVAL, "null pointer"),
  ("out_overlaps_labels", dict(out=LAB + 8), EINVAL, "out overlaps labels"),
  ("out_overlaps_markers", dict(out=MARK + 4), EINVAL, "out overlaps markers"),
  ("out_overlaps_image", dict(out=IMG + 4), EINVAL, "out overlaps image"),
  ("out_overlaps_labels_host", dict(out=LAB - 128 + 4, flags=0), EINVAL, "out overlaps labels"),
  ("level_overlaps_image", dict(level=IMG + 8), EINVAL, "level_out overlaps image"),
  ("level_overlaps_out", dict(level=OUT + 4), EINVAL, "level_out overlaps out"),
  # order: label width, marker width, ndim, sizes, count, connectivity, flags, stack size, tiles, emptiness,
  # pointers, overlap, device
  ("label_width_before_marker_width", dict(label_bytes=5, marker_bytes=5), EINVAL, "label_bytes must be"),
  ("marker_width_before_ndim", dict(marker_bytes=5, ndim=0), EINVAL, "marker_bytes must be"),
  ("ndim_before_size", dict(ndim=5, sx=-1), EINVAL, "ndim"),
  ("size_before_count", dict(sx=BIG, count=-1), ELIMIT, "axis longer"),
  ("count_before_connectivity", dict(count=-1, connectivity=0), EINVAL, "negative count"),
  ("connectivity_before_flags", dict(connectivity=9, flags=SQRT), EINVAL, "connectivity must be"),
  ("flags_before_stack", dict(flags=SQRT, count=1 << 60), EINVAL, "only the residency flags"),
  ("stack_before_tiles", dict(ndim=1, sx=1 << 30, count=1 << 40), ELIMIT, "too many voxels"),
  ("tiles_before_empty", dict(ndim=1, sx=1, count=1 << 33, labels=None, out=None), ELIMIT, "tiles"),
  ("connectivity_before_empty", dict(connectivity=0, count=0), EINVAL, "connectivity must be"),
  ("flags_before_empty", dict(flags=SQRT, count=0), EINVAL, "only the residency flags"),
  ("no_volumes", dict(count=0, labels=None, markers=None, image=None, out=None), 0, ""),
  ("empty_volume", dict(sz=0, labels=None, markers=None, image=None, out=None, flags=0), 0, ""),
  ("pointers_before_overlap", dict(image=None, out=LAB), EINVAL, "null pointer"),
  ("overlap_before_device", dict(out=MARK, device=64), EINVAL, "out overlaps markers"),
  ("valid", dict(), PROBE, ""),
  ("valid_level", dict(level=LEVEL), PROBE, ""),
  ("valid_host", dict(flags=0, level=LEVEL), PROBE, ""),
  ("valid_no_labels", dict(label_bytes=0, labels=None), PROBE, ""),
  ("valid_no_labels_ignores_the_pointer", dict(label_bytes=0, labels=OUT + 1), PROBE, ""),
  ("valid_8_byte", dict(label_bytes=8, marker_bytes=8, count=1), PROBE, ""),
  ("valid_connectivity_3", dict(connectivity=3), PROBE, ""),
  ("valid_mixed_outputs_on_labels", dict(out=LAB, flags=LABELS_ON_DEVICE), PROBE, ""),
  ("valid_same_labels_and_markers", dict(markers=LAB, marker_bytes=4), PROBE, ""),
  ("valid_1d", dict(ndim=1, sy=-1, sz=-1), PROBE, ""),
  ("valid_2d_connectivity_2", dict(ndim=2, sz=-1, connectivity=2), PROBE, ""),
]


@pytest.mark.parametrize("case,overrides,rc,msg", CASES, ids=[c[0] for c in CASES])
def test_watershed_argument_check(edt, case, overrides, rc, msg):
  check_case(edt, edt._lib().edtb200_watershed, _args, overrides, rc, msg)


def test_the_header_names_the_parameters():
  params = prototypes()["edtb200_watershed"][1]
  names = [re.sub(r"[*\s]", "", p.rsplit(" ", 1)[1]) for p in params]
  assert names == ["labels", "label_bytes", "markers", "marker_bytes", "image", "ndim", "sx", "sy", "sz", "count",
                   "connectivity", "flags", "out", "level_out", "device", "stream"]
  assert "const float *image" in params[4] and "float *level_out" in params[13]


def test_the_header_documents_an_addition_at_the_same_version(edt):
  assert edt._lib().edtb200_version() == ABI_VERSION
  assert "edtb200_watershed" in HEADER[:HEADER.index("#define EDTB200_VERSION")]
  doc = header_doc("edtb200_watershed")
  for text in ("neighbours under `connectivity` with the SAME label", "NaN read as +inf and -0.0 as +0.0",
               "L[v] = min(L[v], max(f[v], L[u]))", "L[v] == max(f[v], L[u])", "least marker m with a tight path",
               "compared as unsigned integers of marker_bytes", "label_bytes 0: no labels",
               "ONE cooperative launch of watershed_relax_kernel", "never torn", "no round cap",
               "4 bytes per voxel for L, 4 for W (8 with 8-byte markers)", "12 bytes per tile",
               "Checks, in order: label width, marker width, ndim and sizes", "EDT_B200_VERBOSE",
               "rounds and tile visits"):
    assert text in doc, text


# ---- Python ---------------------------------------------------------------------------------------------

def _vol(shape=(4, 5), dtype=np.float32):
  return np.zeros(shape, dtype)


def test_signature(edt):
  p = inspect.signature(edt.watershed).parameters
  assert list(p) == ["image", "markers", "labels", "connectivity", "return_level", "stacked", "device"]
  assert p["labels"].default is None
  for name, default in (("connectivity", 1), ("return_level", False), ("stacked", False), ("device", 0)):
    assert p[name].kind is inspect.Parameter.KEYWORD_ONLY and p[name].default == default
  assert "watershed" in edt.__all__


@pytest.mark.parametrize("bad", [1, 0, "yes", None, np.array([True])])
def test_rejects_a_non_bool_return_level(no_device_use, bad):
  with pytest.raises(TypeError, match="return_level must be True or False"):
    no_device_use.watershed(_vol(), _vol(dtype=np.uint8), return_level=bad)


@pytest.mark.parametrize("bad", [1.0, True, "1", None, np.ones(3)])
def test_rejects_a_connectivity_that_is_not_an_int(no_device_use, bad):
  with pytest.raises(TypeError, match="connectivity must be an int"):
    no_device_use.watershed(_vol(), _vol(dtype=np.uint8), connectivity=bad)


@pytest.mark.parametrize("shape,conn", [((4, 5), 0), ((4, 5), 3), ((6,), 2), ((3, 4, 5), 4), ((3, 4, 5), -1)])
def test_rejects_a_connectivity_outside_1_to_ndim(no_device_use, shape, conn):
  with pytest.raises(ValueError, match="connectivity must be 1 to %d" % len(shape)):
    no_device_use.watershed(_vol(shape), _vol(shape, np.uint8), connectivity=conn)
  # a stack's volumes have one axis fewer
  with pytest.raises(ValueError, match="connectivity must be 1 to 2"):
    no_device_use.watershed(_vol((2, 4, 5)), _vol((2, 4, 5), np.uint8), connectivity=3, stacked=True)


@pytest.mark.parametrize("shape,stacked", [((), False), ((2, 2, 2, 2), False), ((4,), True), ((2,) * 5, True)])
def test_rejects_a_wrong_number_of_dimensions(no_device_use, shape, stacked):
  with pytest.raises(TypeError, match="-D to"):
    no_device_use.watershed(_vol(shape), _vol(shape, np.uint8), stacked=stacked)
  with pytest.raises(TypeError, match="-D to"):
    no_device_use.watershed(_vol(shape), _vol(shape, np.uint8), _vol(shape, np.uint8), stacked=stacked)


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.float16, np.complex64, object, "U3"])
def test_rejects_an_unsupported_label_dtype(no_device_use, dtype):
  with pytest.raises(TypeError, match="watershed: unsupported label dtype"):
    no_device_use.watershed(_vol(), _vol(dtype=np.uint8), np.zeros((4, 5), dtype))


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.complex64, object])
def test_rejects_an_unsupported_marker_dtype(no_device_use, dtype):
  with pytest.raises(TypeError, match="watershed: unsupported marker dtype"):
    no_device_use.watershed(_vol(), np.zeros((4, 5), dtype))


@pytest.mark.parametrize("dtype", [np.complex64, np.complex128, object, "U3"])
def test_rejects_an_image_that_is_not_real(no_device_use, dtype):
  with pytest.raises(TypeError, match="unsupported image dtype"):
    no_device_use.watershed(np.zeros((4, 5), dtype), _vol(dtype=np.uint8), _vol(dtype=np.uint8))


def test_rejects_arrays_of_another_shape(no_device_use):
  with pytest.raises(ValueError, match="markers must have the volume's shape"):
    no_device_use.watershed(_vol(), _vol((5, 4), np.uint8))
  with pytest.raises(ValueError, match="image must have the volume's shape"):
    no_device_use.watershed(_vol((4, 5, 1)), _vol(dtype=np.uint8), _vol(dtype=np.uint8))
  with pytest.raises(ValueError, match="markers must have the volume's shape"):
    no_device_use.watershed(_vol(), _vol((4, 6), np.uint8), _vol(dtype=np.uint8))


@pytest.mark.parametrize("order", ["C", "F"])
def test_empty_arrays_need_no_device(no_device_use, order):
  for shape, stacked in (((0, 3), False), ((3, 0, 2), False), ((0, 4, 4), True), ((0,), False)):
    img = np.zeros(shape, np.float64, order=order)
    for mdt, odt in ((np.int16, np.int16), (np.bool_, np.uint8), (np.uint64, np.uint64)):
      mk = np.zeros(shape, mdt, order=order)
      out = no_device_use.watershed(img, mk, stacked=stacked)
      assert isinstance(out, np.ndarray) and out.shape == shape and out.dtype == odt
      out, level = no_device_use.watershed(img, mk, np.zeros(shape, np.uint8), stacked=stacked, return_level=True)
      assert level.shape == shape and level.dtype == np.float32


def test_docstring_states_the_definition(edt):
  doc = " ".join(edt.watershed.__doc__.split())
  for text in ("watershed(-dist, markers, mask)", "mask=m is labels=m here", "at most `connectivity` of its "
               "components are non-zero", "NaN is read as +inf and -0.0 as +0.0",
               "L[v] = min(L[v], max(f[v], L[u]))", "L[v] == max(f[v], L[u])", "goes to the smaller marker value",
               "skimage breaks such ties by the order of its queue", "unsigned integers of the markers' width",
               "bool markers give uint8", "np.stack of the per-volume calls", "without a host synchronisation",
               "ENOMEM", "float labels are a TypeError", "float64 altitudes", "4 bytes per voxel for the level"):
    assert " ".join(text.split()) in doc, text
