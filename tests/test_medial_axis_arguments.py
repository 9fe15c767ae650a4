"""CPU tests: the argument checks of edtb200_medial_axis in their documented order, the header's parameter
names, the Python rejections of medial_axis -- each before any device is touched -- and the identities its
docstring and the header state.  A fully valid call stops at the device probe (abi_checks.expect_probe)."""
import inspect
import re

import numpy as np
import pytest

from abi_checks import (ABI_VERSION, BIG, BOTH, EINVAL, ELIMIT, HEADER, INF, LABELS_FLOAT, LABELS_ON_DEVICE, NAN,
                        PROBE, SQRT, check_case, header_doc, no_device_use, prototypes)

LINE = (1 << 26) + 1

_LAB = np.zeros(128, np.uint32)          # 2 volumes of 4 x 4 x 4
_MED = np.zeros(128, np.uint8)
_DIST = np.zeros(128, np.float32)
LAB, MED, DIST = _LAB.ctypes.data, _MED.ctypes.data, _DIST.ctypes.data


def _args(labels=LAB, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, count=2, w=(1.0, 1.0, 1.0), black_border=0,
          flags=BOTH, medial=MED, dist=DIST, device=63, stream=None):
  return (labels, label_bytes, ndim, sx, sy, sz, count, w[0], w[1], w[2], black_border, flags, medial, dist, device,
          stream)


CASES = [
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes must be"),
  ("label_bytes_0", dict(label_bytes=0), EINVAL, "label_bytes must be"),
  ("ndim_0", dict(ndim=0), EINVAL, "ndim"),
  ("ndim_4", dict(ndim=4), EINVAL, "ndim"),
  ("negative_size", dict(sy=-1), EINVAL, "negative size"),
  ("axis_too_long", dict(sz=BIG), ELIMIT, "axis longer than 2^30"),
  ("negative_count", dict(count=-1), EINVAL, "negative count"),
  ("weight_zero", dict(w=(1.0, 0.0, 1.0)), EINVAL, "weight of axis 1"),
  ("weight_negative", dict(w=(-1.0, 1.0, 1.0)), EINVAL, "weight of axis 0"),
  ("weight_nan", dict(w=(1.0, 1.0, NAN)), EINVAL, "weight of axis 2"),
  ("weight_inf", dict(w=(INF, 1.0, 1.0)), EINVAL, "weight of axis 0"),
  ("flag_sqrt", dict(flags=BOTH | SQRT), EINVAL, "residency flags and EDTB200_LABELS_FLOAT"),
  ("flag_32", dict(flags=32), EINVAL, "residency flags and EDTB200_LABELS_FLOAT"),
  ("float_width_2", dict(label_bytes=2, flags=LABELS_FLOAT), EINVAL, "EDTB200_LABELS_FLOAT needs 4- or 8-byte"),
  ("float_width_1", dict(label_bytes=1, flags=BOTH | LABELS_FLOAT), EINVAL, "EDTB200_LABELS_FLOAT needs"),
  ("too_many_voxels", dict(count=1 << 60), ELIMIT, "too many voxels"),
  ("line_x", dict(ndim=1, sx=LINE), ELIMIT, "lines of at most 2^26"),
  ("line_y", dict(sy=LINE, sx=0), ELIMIT, "lines of at most 2^26"),
  ("line_z_empty", dict(sz=LINE, count=0), ELIMIT, "lines of at most 2^26"),
  ("line_limit_is_inclusive", dict(ndim=1, sx=1 << 26, labels=None), EINVAL, "null pointer"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_medial", dict(medial=None), EINVAL, "null pointer"),
  ("medial_overlaps_labels", dict(medial=LAB + 4), EINVAL, "medial_out overlaps labels"),
  ("medial_overlaps_labels_end", dict(medial=LAB - 128 + 1), EINVAL, "medial_out overlaps labels"),
  ("medial_overlaps_labels_host", dict(medial=LAB + 511, flags=0), EINVAL, "medial_out overlaps labels"),
  ("dist_overlaps_labels", dict(dist=LAB + 8), EINVAL, "dist_out overlaps labels"),
  ("dist_overlaps_labels_host", dict(dist=LAB - 4 * 128 + 4, flags=0), EINVAL, "dist_out overlaps labels"),
  ("dist_overlaps_medial", dict(dist=MED + 4), EINVAL, "dist_out overlaps medial_out"),
  ("dist_overlaps_medial_mixed", dict(dist=MED - 4 * 128 + 1, flags=LABELS_ON_DEVICE), EINVAL,
   "dist_out overlaps medial_out"),
  # order: label width, ndim, sizes, count, weights, flags, float width, stack size, line, emptiness, pointers,
  # overlap, device
  ("width_before_ndim", dict(label_bytes=5, ndim=0), EINVAL, "label_bytes must be"),
  ("ndim_before_size", dict(ndim=5, sx=-1), EINVAL, "ndim"),
  ("size_before_count", dict(sx=BIG, count=-1), ELIMIT, "axis longer"),
  ("count_before_weights", dict(count=-1, w=(0.0, 0.0, 0.0)), EINVAL, "negative count"),
  ("weights_before_flags", dict(w=(1.0, NAN, 1.0), flags=SQRT), EINVAL, "weight of axis 1"),
  ("flags_before_float_width", dict(flags=SQRT | LABELS_FLOAT, label_bytes=2), EINVAL, "residency flags"),
  ("float_width_before_stack", dict(flags=LABELS_FLOAT, label_bytes=1, count=1 << 60), EINVAL, "needs 4- or 8-byte"),
  ("stack_before_line", dict(sx=LINE, count=1 << 40), ELIMIT, "too many voxels"),
  ("line_before_empty", dict(sx=LINE, sy=0), ELIMIT, "lines of at most 2^26"),
  ("weights_before_empty", dict(w=(0.0, 1.0, 1.0), count=0), EINVAL, "weight of axis 0"),
  ("flags_before_empty", dict(flags=SQRT, count=0), EINVAL, "residency flags"),
  ("no_volumes", dict(count=0, labels=None, medial=None, dist=None), 0, ""),
  ("empty_volume", dict(sz=0, labels=None, medial=None, flags=0), 0, ""),
  ("pointers_before_overlap", dict(labels=None, dist=MED), EINVAL, "null pointer"),
  ("labels_overlap_before_dist", dict(medial=LAB, dist=LAB), EINVAL, "medial_out overlaps labels"),
  ("overlap_before_device", dict(dist=MED, device=64), EINVAL, "dist_out overlaps medial_out"),
  ("valid", dict(), PROBE, ""),
  ("valid_no_dist", dict(dist=None), PROBE, ""),
  ("valid_host", dict(flags=0), PROBE, ""),
  ("valid_float", dict(flags=BOTH | LABELS_FLOAT), PROBE, ""),
  ("valid_float64", dict(label_bytes=8, count=1, flags=LABELS_FLOAT), PROBE, ""),
  ("valid_border", dict(black_border=7), PROBE, ""),
  ("valid_mixed_outputs_on_labels", dict(medial=LAB, dist=LAB + 128, flags=LABELS_ON_DEVICE), PROBE, ""),
  ("valid_adjacent", dict(dist=MED + 128), PROBE, ""),
  ("valid_huge_weight", dict(w=(1e20, 3e38, 1.0)), PROBE, ""),
  ("valid_2d_ignores_sz_wz", dict(ndim=2, sz=-1, w=(1.0, 1.0, NAN)), PROBE, ""),
  ("valid_1d_ignores_sy_sz", dict(ndim=1, sy=LINE, sz=BIG, w=(2.0, 0.0, -1.0)), PROBE, ""),
]


@pytest.mark.parametrize("case,overrides,rc,msg", CASES, ids=[c[0] for c in CASES])
def test_medial_axis_argument_check(edt, case, overrides, rc, msg):
  check_case(edt, edt._lib().edtb200_medial_axis, _args, overrides, rc, msg)


def test_the_header_names_the_parameters():
  params = prototypes()["edtb200_medial_axis"][1]
  names = [re.sub(r"[*\s]", "", p.rsplit(" ", 1)[1]) for p in params]
  assert names == ["labels", "label_bytes", "ndim", "sx", "sy", "sz", "count", "wx", "wy", "wz", "black_border",
                   "flags", "medial_out", "dist_out", "device", "stream"]
  assert "uint8_t *medial_out" in params[12] and "float *dist_out" in params[13]


def test_the_header_documents_an_addition_at_the_same_version(edt):
  assert edt._lib().edtb200_version() == ABI_VERSION
  assert "edtb200_medial_axis" in HEADER[:HEADER.index("#define EDTB200_VERSION")]
  doc = header_doc("edtb200_medial_axis")
  for text in ("least j", "REAL maximisers", "lexicographically least (z, y, x)", "not masked to",
               "-inf", "reduced discrete medial axis", "4 + 4 ndim", "16 in 3-D", "2^26", "EDTB200_ELIMIT",
               "D2 = 1 4 9 4 1", "medial {2}", "medial {1, 2}", "its first one", "not a topological skeleton",
               "EDT_B200_VERBOSE", "medial_mark_kernel", "Checks, in order: label width, ndim, sizes"):
    assert text in doc, text


# ---- Python ---------------------------------------------------------------------------------------------

def test_signature(edt):
  p = inspect.signature(edt.medial_axis).parameters
  assert list(p) == ["labels", "anisotropy", "black_border", "return_distance", "device", "stacked"]
  assert p["anisotropy"].default is None and p["black_border"].default is False
  for name, default in (("return_distance", False), ("device", 0), ("stacked", False)):
    assert p[name].kind is inspect.Parameter.KEYWORD_ONLY and p[name].default == default
  assert "medial_axis" in edt.__all__


@pytest.mark.parametrize("bad", [1, 0, "yes", None, np.array([True])])
def test_rejects_a_non_bool_return_distance(no_device_use, bad):
  with pytest.raises(TypeError, match="return_distance must be True or False"):
    no_device_use.medial_axis(np.ones((4, 5), np.uint8), return_distance=bad)


@pytest.mark.parametrize("shape,stacked", [((), False), ((2, 2, 2, 2), False), ((4,), True), ((2,) * 5, True)])
def test_rejects_a_wrong_number_of_dimensions(no_device_use, shape, stacked):
  with pytest.raises(TypeError, match="-D to"):
    no_device_use.medial_axis(np.ones(shape, np.uint8), stacked=stacked)


@pytest.mark.parametrize("dtype", [np.float16, np.complex64, object, "U3", "V4"])
def test_rejects_an_unsupported_dtype(no_device_use, dtype):
  with pytest.raises(TypeError, match="unsupported label dtype"):
    no_device_use.medial_axis(np.zeros((3, 4), dtype))


@pytest.mark.parametrize("anisotropy", [(1.0, 0.0), (1.0, -2.0), (np.nan, 1.0), (1.0, np.inf)])
def test_rejects_a_bad_weight(no_device_use, anisotropy):
  with pytest.raises(ValueError, match="finite and > 0"):
    no_device_use.medial_axis(np.ones((3, 4), np.uint8), anisotropy)


def test_rejects_a_weight_count_that_does_not_match(no_device_use):
  with pytest.raises(ValueError, match="one entry per volume axis"):
    no_device_use.medial_axis(np.ones((3, 4), np.uint8), (1.0, 2.0, 3.0))
  with pytest.raises(ValueError, match="one entry per volume axis"):
    no_device_use.medial_axis(np.ones((3, 4, 5), np.uint8), (1.0, 2.0, 3.0), stacked=True)


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("dtype", [np.bool_, np.int16, np.uint64, np.float32])
def test_empty_arrays_need_no_device(no_device_use, order, dtype):
  for shape, stacked in (((0,), False), ((3, 0, 2), False), ((0, 4, 4), True), ((2, 3, 0, 1), True)):
    labels = np.zeros(shape, dtype, order=order)
    medial = no_device_use.medial_axis(labels, stacked=stacked)
    assert isinstance(medial, np.ndarray) and medial.shape == shape and medial.dtype == np.bool_
    medial, dist = no_device_use.medial_axis(labels, stacked=stacked, return_distance=True)
    assert medial.shape == shape and medial.dtype == np.bool_
    assert isinstance(dist, np.ndarray) and dist.shape == shape and dist.dtype == np.float32


def test_docstring_states_the_definition_and_its_identities(edt):
  doc = edt.medial_axis.__doc__
  for text in ("D2 = edtsq(L, w, black_border)", "parabolic_dilate(D2, w, return_indices=True)",
               "0 on the background", "y = q(p) for some voxel p with L(p) != 0", "-0.0 is background",
               "least j among the REAL", "lexicographically least (z, y, x)", "reduced discrete medial axis",
               "Coeurjolly & Montanvert", "not thin and not connected", "topological skeleton",
               "parabolic_dilate(np.where(medial, D2, -np.inf), w) == V", "`... > 0` equals `labels != 0`",
               "every non-empty label has a medial voxel", "D2 = 1, 4, 9, 4, 1 and medial {2}",
               "D2 = 1, 4, 4, 1 and medial {1, 2}", "only medial voxel is its first voxel",
               "edt(labels, anisotropy, black_border), bit for bit", "np.stack of the per-volume calls",
               "ENOMEM", "16 in 3-D"):
    assert " ".join(text.split()) in " ".join(doc.split()), text


def test_the_docstring_examples_hold_on_the_restatement():
  import medial_axis_cases as mac
  for run, d2, medial in (([0, 1, 1, 1, 1, 1, 0], [0, 1, 4, 9, 4, 1, 0], [3]), ([0, 1, 1, 1, 1, 0], [0, 1, 4, 4, 1, 0],
                                                                                 [2, 3])):
    got, got_d2, values, _ = mac.restate(np.array(run, np.uint8))
    assert got_d2.tolist() == d2 and np.flatnonzero(got).tolist() == medial
    rec = mac.reconstruct(got, got_d2)
    fg = np.array(run) != 0
    assert np.array_equal(rec[fg], values[fg]) and np.array_equal(rec > 0, fg)
