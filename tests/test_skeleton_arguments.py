"""CPU tests: the argument checks of edtb200_skeletonize in their documented order, the header's parameter
names, the Python rejections of skeletonize -- each before any device is touched -- and the statements of its
docstring and the header.  A fully valid call stops at the device probe (abi_checks.expect_probe)."""
import inspect
import re

import numpy as np
import pytest

from abi_checks import (ABI_VERSION, BIG, BOTH, EINVAL, ELIMIT, HEADER, INF, LABELS_FLOAT, LABELS_ON_DEVICE, NAN,
                        PROBE, SQRT, check_case, header_doc, no_device_use, prototypes)

_LAB = np.zeros(128, np.uint32)          # 2 volumes of 4 x 4 x 4
_SKEL = np.zeros(128, np.uint8)
_DIST = np.zeros(128, np.float32)
LAB, SKEL, DIST = _LAB.ctypes.data, _SKEL.ctypes.data, _DIST.ctypes.data


def _args(labels=LAB, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, count=2, w=(1.0, 1.0, 1.0), black_border=0,
          flags=BOTH, skeleton=SKEL, dist=DIST, device=63, stream=None):
  return (labels, label_bytes, ndim, sx, sy, sz, count, w[0], w[1], w[2], black_border, flags, skeleton, dist, device,
          stream)


CASES = [
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes must be"),
  ("label_bytes_0", dict(label_bytes=0), EINVAL, "label_bytes must be"),
  ("ndim_0", dict(ndim=0), EINVAL, "ndim must be 1, 2 or 3"),
  ("ndim_4", dict(ndim=4), EINVAL, "ndim must be 1, 2 or 3"),
  ("negative_size", dict(sy=-1), EINVAL, "negative size"),
  ("axis_too_long", dict(sz=BIG), ELIMIT, "axis longer than 2^30"),
  ("ndim_1", dict(ndim=1), EINVAL, "takes 2-D and 3-D volumes"),
  ("negative_count", dict(count=-1), EINVAL, "negative count"),
  ("weight_zero", dict(w=(1.0, 0.0, 1.0)), EINVAL, "weight of axis 1"),
  ("weight_negative", dict(w=(-1.0, 1.0, 1.0)), EINVAL, "weight of axis 0"),
  ("weight_nan", dict(w=(1.0, 1.0, NAN)), EINVAL, "weight of axis 2"),
  ("weight_inf", dict(w=(INF, 1.0, 1.0)), EINVAL, "weight of axis 0"),
  ("flag_sqrt", dict(flags=BOTH | SQRT), EINVAL, "only the residency flags"),
  ("flag_float", dict(flags=LABELS_FLOAT), EINVAL, "only the residency flags"),
  ("flag_32", dict(flags=32), EINVAL, "only the residency flags"),
  ("too_many_voxels", dict(count=1 << 60), ELIMIT, "too many voxels"),
  ("subfield_too_big", dict(sx=1 << 20, sy=1 << 20, sz=1 << 6, count=1, labels=None), ELIMIT,
   "fewer than 2^32 voxels per subfield"),
  ("subfield_of_2_to_the_32", dict(sx=1 << 17, sy=1 << 17, sz=2, count=1, labels=None), ELIMIT, "per subfield"),
  ("subfield_just_below", dict(sx=(1 << 17) - 2, sy=1 << 17, sz=2, count=1, labels=None), EINVAL, "null pointer"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_skeleton", dict(skeleton=None), EINVAL, "null pointer"),
  ("skeleton_overlaps_labels", dict(skeleton=LAB + 4), EINVAL, "skeleton_out overlaps labels"),
  ("skeleton_overlaps_labels_end", dict(skeleton=LAB - 128 + 1), EINVAL, "skeleton_out overlaps labels"),
  ("skeleton_overlaps_labels_host", dict(skeleton=LAB + 511, flags=0), EINVAL, "skeleton_out overlaps labels"),
  ("dist_overlaps_labels", dict(dist=LAB + 8), EINVAL, "dist_out overlaps labels"),
  ("dist_overlaps_labels_host", dict(dist=LAB - 4 * 128 + 4, flags=0), EINVAL, "dist_out overlaps labels"),
  ("dist_overlaps_skeleton", dict(dist=SKEL + 4), EINVAL, "dist_out overlaps skeleton_out"),
  ("dist_overlaps_skeleton_mixed", dict(dist=SKEL - 4 * 128 + 1, flags=LABELS_ON_DEVICE), EINVAL,
   "dist_out overlaps skeleton_out"),
  # order: label width, ndim, sizes, ndim of 2 or 3, count, weights, flags, stack size, subfield size,
  # emptiness, pointers, overlap, device
  ("width_before_ndim", dict(label_bytes=5, ndim=0), EINVAL, "label_bytes must be"),
  ("ndim_before_size", dict(ndim=5, sx=-1), EINVAL, "ndim"),
  ("size_before_2d", dict(ndim=1, sx=BIG), ELIMIT, "axis longer"),
  ("2d_before_count", dict(ndim=1, count=-1), EINVAL, "takes 2-D and 3-D volumes"),
  ("count_before_weights", dict(count=-1, w=(0.0, 0.0, 0.0)), EINVAL, "negative count"),
  ("weights_before_flags", dict(w=(1.0, NAN, 1.0), flags=SQRT), EINVAL, "weight of axis 1"),
  ("flags_before_stack", dict(flags=SQRT, count=1 << 60), EINVAL, "only the residency flags"),
  ("stack_before_subfield", dict(sx=1 << 30, sy=1 << 30, count=1 << 10), ELIMIT, "too many voxels"),
  ("subfield_before_empty", dict(sx=1 << 20, sy=1 << 20, sz=1 << 6, count=1, labels=None, skeleton=None),
   ELIMIT, "per subfield"),
  ("weights_before_empty", dict(w=(0.0, 1.0, 1.0), count=0), EINVAL, "weight of axis 0"),
  ("flags_before_empty", dict(flags=SQRT, count=0), EINVAL, "only the residency flags"),
  ("no_volumes", dict(count=0, labels=None, skeleton=None, dist=None), 0, ""),
  ("empty_volume", dict(sz=0, labels=None, skeleton=None, flags=0), 0, ""),
  ("pointers_before_overlap", dict(labels=None, dist=SKEL), EINVAL, "null pointer"),
  ("labels_overlap_before_dist", dict(skeleton=LAB, dist=LAB), EINVAL, "skeleton_out overlaps labels"),
  ("overlap_before_device", dict(dist=SKEL, device=64), EINVAL, "dist_out overlaps skeleton_out"),
  ("valid", dict(), PROBE, ""),
  ("valid_no_dist", dict(dist=None), PROBE, ""),
  ("valid_host", dict(flags=0), PROBE, ""),
  ("valid_8_byte", dict(label_bytes=8, count=1), PROBE, ""),
  ("valid_border", dict(black_border=7), PROBE, ""),
  ("valid_mixed_outputs_on_labels", dict(skeleton=LAB, dist=LAB + 128, flags=LABELS_ON_DEVICE), PROBE, ""),
  ("valid_adjacent", dict(dist=SKEL + 128), PROBE, ""),
  ("valid_huge_weight", dict(w=(1e20, 3e38, 1.0)), PROBE, ""),
  ("valid_2d_ignores_sz_wz", dict(ndim=2, sz=-1, w=(1.0, 1.0, NAN)), PROBE, ""),
]


@pytest.mark.parametrize("case,overrides,rc,msg", CASES, ids=[c[0] for c in CASES])
def test_skeletonize_argument_check(edt, case, overrides, rc, msg):
  check_case(edt, edt._lib().edtb200_skeletonize, _args, overrides, rc, msg)


def test_the_header_names_the_parameters():
  params = prototypes()["edtb200_skeletonize"][1]
  names = [re.sub(r"[*\s]", "", p.rsplit(" ", 1)[1]) for p in params]
  assert names == ["labels", "label_bytes", "ndim", "sx", "sy", "sz", "count", "wx", "wy", "wz", "black_border",
                   "flags", "skeleton_out", "dist_out", "device", "stream"]
  assert "uint8_t *skeleton_out" in params[12] and "float *dist_out" in params[13]


def test_the_header_documents_an_addition_at_the_same_version(edt):
  assert edt._lib().edtb200_version() == ABI_VERSION
  assert "edtb200_skeletonize" in HEADER[:HEADER.index("#define EDTB200_VERSION")]
  doc = header_doc("edtb200_skeletonize")
  for text in ("26-connected (2-D: 8-)", "6-connected (2-D: 4-)", "exactly one 6-component",
               "theta_t = (t h)^2 in double", "R = +inf included", "start of the CYCLE",
               "k = (x & 1) | (y & 1) << 1 | (z & 1) << 2", "Euler characteristic", "thinness",
               "F-ordered array gives the C-ordered call on its transpose with the weights reversed",
               "3x3x3 cube in background gives exactly its centre", "x = 4 .. 10 at (z, y) = (3, 4)",
               "12 in 2-D and 3-D; 8 with dist_out", "skeleton_thin_kernel", "ONE cooperative launch",
               "EDT_B200_VERBOSE", "Checks, in order: label width, ndim, sizes", "below 2^32 voxels"):
    assert text in doc, text


# ---- Python ---------------------------------------------------------------------------------------------

def test_signature(edt):
  p = inspect.signature(edt.skeletonize).parameters
  assert list(p) == ["labels", "anisotropy", "black_border", "return_distance", "device", "stacked"]
  assert p["anisotropy"].default is None and p["black_border"].default is False
  for name, default in (("return_distance", False), ("device", 0), ("stacked", False)):
    assert p[name].kind is inspect.Parameter.KEYWORD_ONLY and p[name].default == default
  assert "skeletonize" in edt.__all__


@pytest.mark.parametrize("bad", [1, 0, "yes", None, np.array([True])])
def test_rejects_a_non_bool_return_distance(no_device_use, bad):
  with pytest.raises(TypeError, match="return_distance must be True or False"):
    no_device_use.skeletonize(np.ones((4, 5), np.uint8), return_distance=bad)


@pytest.mark.parametrize("shape,stacked", [((), False), ((4,), False), ((2, 2, 2, 2), False), ((4, 4), True),
                                           ((2,) * 5, True)])
def test_rejects_a_wrong_number_of_dimensions(no_device_use, shape, stacked):
  with pytest.raises(TypeError, match="-D to"):
    no_device_use.skeletonize(np.ones(shape, np.uint8), stacked=stacked)


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.float16, np.complex64, object, "U3", "V4"])
def test_rejects_an_unsupported_dtype(no_device_use, dtype):
  with pytest.raises(TypeError, match="unsupported label dtype"):
    no_device_use.skeletonize(np.zeros((3, 4), dtype))


def test_accepts_exactly_the_dtypes_of_nearest_labels(edt):
  for dtype in (np.bool_, np.int8, np.uint8, np.int16, np.uint16, np.int32, np.uint32, np.int64, np.uint64,
                np.float16, np.float32, np.float64, np.complex64):
    try:
      edt._nearest_label_bytes(np.dtype(dtype))
      nearest = True
    except TypeError:
      nearest = False
    try:
      edt.skeletonize(np.zeros((0, 3), dtype))
      ours = True
    except TypeError:
      ours = False
    assert ours == nearest, dtype


@pytest.mark.parametrize("anisotropy", [(1.0, 0.0), (1.0, -2.0), (np.nan, 1.0), (1.0, np.inf)])
def test_rejects_a_bad_weight(no_device_use, anisotropy):
  with pytest.raises(ValueError, match="finite and > 0"):
    no_device_use.skeletonize(np.ones((3, 4), np.uint8), anisotropy)


def test_rejects_a_weight_count_that_does_not_match(no_device_use):
  with pytest.raises(ValueError, match="one entry per volume axis"):
    no_device_use.skeletonize(np.ones((3, 4), np.uint8), (1.0, 2.0, 3.0))
  with pytest.raises(ValueError, match="one entry per volume axis"):
    no_device_use.skeletonize(np.ones((3, 4, 5), np.uint8), (1.0, 2.0, 3.0), stacked=True)


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("dtype", [np.bool_, np.int16, np.uint64])
def test_empty_arrays_need_no_device(no_device_use, order, dtype):
  for shape, stacked in (((0, 3), False), ((3, 0, 2), False), ((0, 4, 4), True), ((2, 3, 0, 1), True)):
    labels = np.zeros(shape, dtype, order=order)
    skel = no_device_use.skeletonize(labels, stacked=stacked)
    assert isinstance(skel, np.ndarray) and skel.shape == shape and skel.dtype == np.bool_
    skel, dist = no_device_use.skeletonize(labels, stacked=stacked, return_distance=True)
    assert skel.shape == shape and skel.dtype == np.bool_
    assert isinstance(dist, np.ndarray) and dist.shape == shape and dist.dtype == np.float32


def test_docstring_states_the_definition(edt):
  doc = " ".join(edt.skeletonize.__doc__.split())
  for text in ("26-connected (2-D: 8-)", "6-connected (2-D: 4-)", "R = edtsq(labels, anisotropy, black_border)",
               "theta_t = (t h)^2 in double", "R = +inf included", "was not an end point at the start of the cycle",
               "k = (x & 1) | (y & 1) << 1 | (z & 1) << 2", "Euler characteristic", "thin (no voxel of it is simple",
               "transpose with the weights reversed", "3x3x3 cube in background gives exactly its centre",
               "(skeleton, edt(labels, anisotropy, black_border))", "dist[skeleton]", "labels[skeleton]",
               "np.stack of the per-volume calls", "without a host synchronisation", "ENOMEM",
               "float labels are a TypeError", "12 bytes per voxel"):
    assert " ".join(text.split()) in doc, text
