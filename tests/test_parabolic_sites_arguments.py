"""CPU tests: the argument checks of edtb200_parabolic_sites in their documented order (those of
edtb200_parabolic, then the 2^26 line limit, then idx with the pointers and overlaps), the Python
rejections of return_indices, and the docstrings.  A fully valid call stops at the device probe
(abi_checks.expect_probe)."""
import re

import numpy as np
import pytest

from abi_checks import ABI_VERSION, BOTH, EINVAL, ELIMIT, HEADER, LABELS_ON_DEVICE, PROBE, check_case, no_device_use
from test_parabolic_arguments import CASES, IN, OUT

_IDX = np.zeros(3 * 512, np.int32)
IDX = _IDX.ctypes.data
LINE = (1 << 26) + 1


def _args(f=IN, ndim=3, sx=4, sy=4, sz=4, count=2, w=(1.0, 1.0, 1.0), op=0, flags=BOTH, out=OUT, idx=IDX, device=63,
          stream=None):
  return (f, ndim, sx, sy, sz, count, w[0], w[1], w[2], op, flags, out, idx, device, stream)


SITES_CASES = [(name.replace("parabolic", "parabolic_sites"), kw, rc, msg) for name, kw, rc, msg in CASES] + [
  ("line_x", dict(ndim=1, sx=LINE), ELIMIT, "lines of at most 2^26"),
  ("line_y", dict(sy=LINE, sx=0), ELIMIT, "lines of at most 2^26"),
  ("line_z_empty", dict(sz=LINE, count=0), ELIMIT, "lines of at most 2^26"),
  ("line_limit_is_inclusive", dict(ndim=1, sx=1 << 26, f=None), EINVAL, "null pointer"),
  ("line_2d_ignores_sz", dict(ndim=2, sz=LINE), PROBE, ""),
  ("stack_size_before_line", dict(sx=LINE, count=1 << 40), ELIMIT, "too many voxels"),
  ("flags_before_line", dict(sx=LINE, flags=1), EINVAL, "residency flags"),
  ("line_before_empty", dict(sx=LINE, sy=0), ELIMIT, "lines of at most 2^26"),
  ("null_idx", dict(idx=None), EINVAL, "null pointer"),
  ("null_idx_empty", dict(idx=None, count=0), 0, ""),
  ("idx_overlaps_out", dict(idx=OUT + 4), EINVAL, "idx overlaps out"),
  ("idx_overlaps_out_end", dict(idx=OUT - 4 * 3 * 128 + 4), EINVAL, "idx overlaps out"),
  ("idx_overlaps_out_host", dict(idx=OUT + 4, flags=0), EINVAL, "idx overlaps out"),
  ("idx_overlaps_f", dict(idx=IN), EINVAL, "idx overlaps f"),
  ("idx_overlaps_f_host", dict(idx=IN + 8, flags=0), EINVAL, "idx overlaps f"),
  ("idx_past_out", dict(idx=OUT + 4 * 128), PROBE, ""),
  ("idx_on_f_mixed", dict(idx=IN, flags=LABELS_ON_DEVICE), PROBE, ""),
  ("overlap_before_idx", dict(out=IN + 4, idx=IN), EINVAL, "out overlaps f"),
]


@pytest.mark.parametrize("case,overrides,rc,msg", SITES_CASES, ids=[c[0] for c in SITES_CASES])
def test_parabolic_sites_argument_check(edt, case, overrides, rc, msg):
  lib = edt._lib()
  check_case(edt, lib.edtb200_parabolic_sites, _args, overrides, rc, msg)
  if msg == "residency flags":
    assert b"edtb200_parabolic_sites" in lib.edtb200_last_error()


def test_the_header_documents_an_addition_at_the_same_version(edt):
  lib = edt._lib()
  assert lib.edtb200_version() == ABI_VERSION
  assert "edtb200_parabolic_sites" in HEADER[:HEADER.index("#define EDTB200_VERSION")]
  proto = re.search(r"int edtb200_parabolic_sites\(([^)]*)\);", HEADER)
  assert proto and "int32_t *idx" in proto.group(1)
  for text in ("least j among the REAL", "2^26", "EDTB200_ELIMIT", "-1 in every coordinate", "8 in 3-D"):
    assert text in HEADER, text


# ---- Python ---------------------------------------------------------------------------------------------

FNS = ["parabolic_erode", "parabolic_dilate"]


@pytest.mark.parametrize("name", FNS)
def test_return_indices_is_a_keyword_that_defaults_to_false(edt, name):
  import inspect
  p = inspect.signature(getattr(edt, name)).parameters["return_indices"]
  assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is False


@pytest.mark.parametrize("name", FNS)
@pytest.mark.parametrize("bad", [1, 0, "yes", None, np.array([True])])
def test_rejects_a_non_bool_return_indices(no_device_use, name, bad):
  with pytest.raises(TypeError, match="return_indices must be True or False"):
    getattr(no_device_use, name)(np.ones((4, 5), np.float32), return_indices=bad)


@pytest.mark.parametrize("name", FNS)
def test_the_other_checks_still_come_first(no_device_use, name):
  fn = getattr(no_device_use, name)
  with pytest.raises(ValueError, match="finite and > 0"):
    fn(np.ones((4, 5), np.float32), (1.0, 0.0), return_indices=True)
  with pytest.raises(TypeError, match="real or bool"):
    fn(np.zeros((3, 4), np.complex64), return_indices=True)
  with pytest.raises(TypeError, match="1-D to 3-D"):
    fn(np.ones((2, 2, 2, 2), np.float32), return_indices=True)
  with pytest.raises(ValueError, match="one entry per volume axis"):
    fn(np.ones((3, 4, 5), np.float32), (1.0, 2.0, 3.0), stacked=True, return_indices=True)


@pytest.mark.parametrize("name", FNS)
@pytest.mark.parametrize("order", ["C", "F"])
def test_empty_arrays_give_empty_indices_without_a_device(no_device_use, name, order):
  fn = getattr(no_device_use, name)
  for shape, stacked in (((0,), False), ((3, 0, 2), False), ((0, 4, 4), True), ((2, 3, 0, 1), True)):
    vals, idx = fn(np.zeros(shape, np.int16, order=order), stacked=stacked, return_indices=True)
    vnd = len(shape) - (1 if stacked else 0)
    assert isinstance(vals, np.ndarray) and vals.shape == shape and vals.dtype == np.float32
    assert isinstance(idx, np.ndarray) and idx.shape == (vnd,) + shape and idx.dtype == np.int32


@pytest.mark.parametrize("name", FNS)
def test_docstrings_define_the_sites_and_give_the_worked_uses(edt, name):
  doc = getattr(edt, name).__doc__
  for text in ("return_indices=True", "least j among the REAL minimisers", "float64 sum before its",
               "never sites", "least -inf position", "its own site", "least maximiser", "every coordinate is -1",
               "chain of rounded candidates", "cells = seed_labels[tuple(idx)]",
               "parabolic_dilate(score, w, return_indices=True)", "ball_ids[tuple(idx)]", "2^26"):
    assert text in doc, text
