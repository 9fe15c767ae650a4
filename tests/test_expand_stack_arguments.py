"""CPU tests: the argument checks of edtb200_expand_gather and the Python rejections of
expand_labels(stacked=True).

As in test_stack_arguments.py, every rejection comes with a return code and a message before any
device is touched, and a fully valid call stops at the device probe (abi_checks.expect_probe).  Nothing
here launches a kernel or copies a byte.
"""
import ctypes
import inspect

import numpy as np
import pytest

from abi_checks import (ABI_VERSION, BIG, BOTH, ECUDA, EINVAL, ELIMIT, LABELS_FLOAT, LABELS_ON_DEVICE, OUT_ON_DEVICE,
                        PROBE, SIGNED, SQRT, check_case)

# separate host blocks: the checks only test for NULL
_LABELS = np.zeros(512, np.uint64)
_DIST = np.zeros(512, np.float32)
_PLANE = np.zeros(512, np.int32)
L, D, P = _LABELS.ctypes.data, _DIST.ctypes.data, _PLANE.ctypes.data


def ptrs(*values):
  return (ctypes.c_void_p * len(values))(*values)


def _gather(labels=L, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, count=2, sqdist=D, idx=None, limit_sq=1.0,
            flags=BOTH, out=L, device=63, stream=None):
  idx = ptrs(P, P, P) if idx is None else idx
  return (labels, label_bytes, ndim, sx, sy, sz, count, sqdist, idx, limit_sq, flags, out, device, stream)


CASES = [
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes"),
  ("label_bytes_16", dict(label_bytes=16), EINVAL, "label_bytes"),
  ("ndim_0", dict(ndim=0), EINVAL, "ndim"),
  ("ndim_4", dict(ndim=4), EINVAL, "ndim"),
  ("negative_size", dict(sy=-1), EINVAL, "negative size"),
  ("axis_too_long", dict(sx=BIG), ELIMIT, "axis longer than 2^30"),
  ("negative_count", dict(count=-1), EINVAL, "negative count"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_sqdist", dict(sqdist=None), EINVAL, "null pointer"),
  ("null_planes", dict(idx=0), EINVAL, "null pointer"),
  ("null_plane_0", dict(idx=ptrs(None, P, P)), EINVAL, "null index plane 0"),
  ("null_plane_1", dict(idx=ptrs(P, None, P)), EINVAL, "null index plane 1"),
  ("null_plane_2", dict(idx=ptrs(P, P, None)), EINVAL, "null index plane 2"),
  ("null_out", dict(out=None), EINVAL, "null pointer"),
  ("host_buffers", dict(flags=0), EINVAL, "device buffers only"),
  ("labels_on_host", dict(flags=OUT_ON_DEVICE), EINVAL, "device buffers only"),
  ("out_on_host", dict(flags=LABELS_ON_DEVICE | LABELS_FLOAT), EINVAL, "device buffers only"),
  ("unknown_flag", dict(flags=BOTH | SQRT), EINVAL, "device buffers only"),
  ("signed_flag", dict(flags=BOTH | SIGNED), EINVAL, "device buffers only"),
  ("float_1_byte", dict(label_bytes=1, flags=BOTH | LABELS_FLOAT), EINVAL, "EDTB200_LABELS_FLOAT needs 4- or 8-byte"),
  ("float_2_bytes", dict(label_bytes=2, flags=BOTH | LABELS_FLOAT), EINVAL, "EDTB200_LABELS_FLOAT needs 4- or 8-byte"),
  # order: label width, ndim, sizes, count, emptiness, pointers, residency, float width
  ("label_bytes_before_ndim", dict(label_bytes=3, ndim=4), EINVAL, "label_bytes"),
  ("ndim_before_size", dict(ndim=5, sx=-1), EINVAL, "ndim"),
  ("size_before_count", dict(sx=BIG, count=-1), ELIMIT, "axis longer"),
  ("count_before_empty", dict(count=-1, sz=0), EINVAL, "negative count"),
  ("no_volumes", dict(count=0, labels=None, out=None, flags=0), 0, ""),
  ("empty_volume", dict(sy=0, labels=None, sqdist=None, idx=0, out=None, flags=0), 0, ""),
  ("labels_before_planes", dict(labels=None, idx=ptrs(None, P, P)), EINVAL, "null pointer"),
  ("planes_before_out", dict(idx=ptrs(P, None, P), out=None), EINVAL, "null index plane 1"),
  ("pointers_before_residency", dict(out=None, flags=0), EINVAL, "null pointer"),
  ("residency_before_float_width", dict(label_bytes=2, flags=LABELS_FLOAT), EINVAL, "device buffers only"),
  # 2-D ignores sz and plane 2, 1-D sy and sz and planes 1 and 2
  ("valid", dict(), PROBE, ""),
  ("valid_in_place", dict(out=L), PROBE, ""),
  ("valid_out_of_place", dict(out=P), PROBE, ""),
  ("valid_float_4", dict(flags=BOTH | LABELS_FLOAT), PROBE, ""),
  ("valid_float_8", dict(label_bytes=8, flags=BOTH | LABELS_FLOAT), PROBE, ""),
  ("valid_2d_ignores_plane_2", dict(ndim=2, sz=-1, idx=ptrs(P, P, None)), PROBE, ""),
  ("valid_1d_ignores_planes_1_2", dict(ndim=1, sy=-1, sz=BIG, idx=ptrs(P, None, None), count=300), PROBE, ""),
  ("valid_one_volume", dict(count=1), PROBE, ""),
  ("valid_nan_limit", dict(limit_sq=float("nan")), PROBE, ""),
  ("valid_inf_limit", dict(limit_sq=float("inf")), PROBE, ""),
]


@pytest.mark.parametrize("case,overrides,rc,msg", CASES, ids=[c[0] for c in CASES])
def test_expand_gather_argument_check(edt, case, overrides, rc, msg):
  check_case(edt, edt._lib().edtb200_expand_gather, _gather, overrides, rc, msg)


def test_expand_gather_is_an_addition_at_the_same_version(edt):
  lib = edt._lib()
  assert lib.edtb200_version() == ABI_VERSION
  assert hasattr(lib, "edtb200_expand_gather")
  assert lib.edtb200_expand_gather.argtypes[9] is ctypes.c_double


# ---- Python: expand_labels(stacked=True) ------------------------------------------------------------

def test_stacked_keyword(edt):
  p = inspect.signature(edt.expand_labels).parameters["stacked"]
  assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is False


def test_stacked_rejects_1d_and_5d(edt):
  with pytest.raises(ValueError, match="2-D to 4-D"):
    edt.expand_labels(np.ones(8, np.uint8), stacked=True)
  with pytest.raises(ValueError, match="2-D to 4-D"):
    edt.expand_labels(np.ones((2, 2, 2, 2, 2), np.uint8), stacked=True)


def test_stacked_rejects_anisotropy_of_the_wrong_length(edt):
  with pytest.raises(ValueError, match="one entry per volume axis"):
    edt.expand_labels(np.ones((3, 4, 4), np.uint8), 1.0, (1.0, 1.0, 1.0), stacked=True)
  with pytest.raises(ValueError, match="one entry per volume axis"):
    edt.expand_labels(np.ones((3, 4, 4, 4), np.uint8), 1.0, (1.0,), stacked=True)


def test_stacked_rejects_max_device_bytes(edt):
  for budget in (0, 1 << 20):
    with pytest.raises(ValueError, match="max_device_bytes"):
      edt.expand_labels(np.ones((3, 4, 4), np.uint8), max_device_bytes=budget, stacked=True)


def test_stacked_rejects_unsupported_dtype(edt):
  with pytest.raises(TypeError, match="unsupported label dtype"):
    edt.expand_labels(np.zeros((3, 4, 4), np.complex64), stacked=True)
  with pytest.raises(TypeError, match="unsupported label dtype"):
    edt.expand_labels(np.zeros((3, 4, 4), np.float16), stacked=True)


def test_stacked_empty_stack_touches_no_device(edt, monkeypatch):
  def no_device(*args):
    raise AssertionError("an empty stack reached the library")
  monkeypatch.setattr(edt, "device_count", no_device)
  monkeypatch.setattr(edt._lib(), "edtb200_expand_gather", no_device)
  monkeypatch.setattr(edt._lib(), "edtb200_feature_transform_stack", no_device)
  x = np.ones((0, 4, 4), np.uint8)
  out = edt.expand_labels(x, 2.0, stacked=True)
  assert out.shape == (0, 4, 4) and out.dtype == np.uint8 and out is not x
  y = np.ones((5, 0, 4), np.float32, order="F")
  out = edt.expand_labels(y, stacked=True)
  assert out.shape == (5, 0, 4) and out.dtype == np.float32


def test_stacked_reaches_the_library_without_a_device(edt):
  """Without a GPU a stacked call fails with ECUDA, as every transform does."""
  if edt.device_count() > 0:
    pytest.skip("a GPU is visible")
  for x in (np.ones((3, 4, 4), np.uint8), np.asfortranarray(np.zeros((3, 4, 5), np.float32))):
    with pytest.raises(edt.EDTError) as info:
      edt.expand_labels(x, stacked=True)
    assert info.value.code == ECUDA
