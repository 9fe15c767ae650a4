"""CPU tests: the argument checks of edtb200_transform_chunked and of the Python keyword
max_device_bytes.

As in test_capi_arguments.py, every rejection comes with a return code and a message before any
device is touched, and a fully valid call stops at the device probe (abi_checks.expect_probe).  Nothing
here launches a kernel or copies a byte.
"""
import ctypes

import numpy as np
import pytest

from abi_checks import (ABI_VERSION, BIG, ECUDA, EINVAL, ELIMIT, HEADER, LABELS_ON_DEVICE, OUT_ON_DEVICE, PROBE, SIGNED,
                        SQRT, check_case)

# two separate host blocks: the checks only test for NULL and for overlap
_LABELS = np.zeros(256, np.uint64)
_OUT = np.zeros(256, np.uint64)
L, O = _LABELS.ctypes.data, _OUT.ctypes.data


def _chunked(labels=L, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, w=(1.0, 1.0, 1.0), border=0, flags=0, out=O,
             device=63, device_bytes=0, chunks=None):
  return (labels, label_bytes, ndim, sx, sy, sz, *w, border, flags, out, device, device_bytes, chunks)


CASES = [
  ("labels_on_device", dict(flags=LABELS_ON_DEVICE), EINVAL, "HOST buffers"),
  ("out_on_device", dict(flags=OUT_ON_DEVICE), EINVAL, "HOST buffers"),
  ("both_on_device", dict(flags=LABELS_ON_DEVICE | OUT_ON_DEVICE | SQRT), EINVAL, "HOST buffers"),
  ("ndim_1", dict(ndim=1), EINVAL, "2-D or 3-D volume (got ndim 1)"),
  ("ndim_0", dict(ndim=0), EINVAL, "2-D or 3-D volume (got ndim 0)"),
  ("ndim_4", dict(ndim=4), EINVAL, "2-D or 3-D volume (got ndim 4)"),
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes"),
  ("label_bytes_16", dict(label_bytes=16), EINVAL, "label_bytes"),
  ("negative_size", dict(sy=-1), EINVAL, "negative size"),
  ("axis_too_long", dict(sx=BIG), ELIMIT, "axis longer than 2^30"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_out", dict(out=None), EINVAL, "null pointer"),
  # 64 voxels: 256 label bytes and 256 output bytes
  ("same_buffer", dict(out=L), EINVAL, "labels and out overlap"),
  ("out_inside_labels", dict(out=L + 128), EINVAL, "labels and out overlap"),
  ("labels_inside_out", dict(labels=O + 252), EINVAL, "labels and out overlap"),
  ("wide_labels_reach_out", dict(label_bytes=8, out=L + 511), EINVAL, "labels and out overlap"),
  # order: residency, dimensionality, label width, emptiness, pointers, overlap
  ("flags_before_ndim", dict(flags=OUT_ON_DEVICE, ndim=1), EINVAL, "HOST buffers"),
  ("ndim_before_label_bytes", dict(ndim=1, label_bytes=3), EINVAL, "2-D or 3-D"),
  ("label_bytes_before_null", dict(label_bytes=3, labels=None), EINVAL, "label_bytes"),
  ("empty_before_null", dict(sz=0, labels=None, out=None), 0, ""),
  ("null_before_overlap", dict(labels=None, out=0), EINVAL, "null pointer"),
  # adjacent buffers do not overlap; 2-D ignores sz
  ("valid_adjacent", dict(out=L + 256), PROBE, ""),
  ("valid_adjacent_below", dict(labels=O + 256), PROBE, ""),
  ("valid_2d_ignores_sz", dict(ndim=2, sz=-1), PROBE, ""),
  ("valid_budget", dict(device_bytes=1 << 20, flags=SQRT | SIGNED), PROBE, ""),
  ("valid", dict(), PROBE, ""),
]


@pytest.mark.parametrize("case,overrides,rc,msg", CASES, ids=[c[0] for c in CASES])
def test_chunked_argument_check(edt, case, overrides, rc, msg):
  chunks = []

  def build(**kw):
    chunks.append((ctypes.c_int64 * 2)(-7, -7))
    return _chunked(**kw, chunks=chunks[-1])
  check_case(edt, edt._lib().edtb200_transform_chunked, build, overrides, rc, msg)
  assert all(list(c) == [0, 0] for c in chunks)          # each call cleared its chunks before any check


def test_chunked_is_an_addition_at_the_same_version(edt):
  """edtb200_transform_chunked is exported next to the 202-level entry points, which keep the number."""
  lib = edt._lib()
  assert lib.edtb200_version() == ABI_VERSION
  assert hasattr(lib, "edtb200_transform_chunked") and hasattr(lib, "edtb200_feature_transform")


def test_chunk_reserve_is_declared():
  import re
  assert int(re.search(r"#define EDTB200_CHUNK_RESERVE (\d+)", HEADER).group(1)) == 512 << 20


# ---- Python: max_device_bytes ----------------------------------------------------------------

def test_max_device_bytes_rejects_1d(edt):
  with pytest.raises(ValueError, match="2-D or 3-D"):
    edt.edtsq(np.ones(8, np.uint8), max_device_bytes=1 << 20)
  with pytest.raises(ValueError, match="2-D or 3-D"):
    edt.sdf(np.ones(8, np.uint8), max_device_bytes=0)


def test_max_device_bytes_rejects_4d(edt):
  with pytest.raises(ValueError, match="2-D or 3-D"):
    edt.edt(np.ones((2, 2, 2, 2), np.uint8), max_device_bytes=0)


def test_max_device_bytes_rejects_voxel_graph(edt):
  a = np.ones((4, 4), np.uint8)
  with pytest.raises(ValueError, match="voxel_graph"):
    edt.edt(a, voxel_graph=np.full((4, 4), 63, np.uint8), max_device_bytes=1 << 20)
  with pytest.raises(ValueError, match="voxel_graph"):
    edt.edt2dsq(a, voxel_graph=np.full((4, 4), 63, np.uint8), max_device_bytes=1 << 20)


@pytest.mark.parametrize("devices", [[0, 1], [0]])
def test_max_device_bytes_rejects_devices(edt, devices):
  with pytest.raises(ValueError, match="devices"):
    edt.edtsq(np.ones((4, 4, 4), np.uint8), devices=devices, max_device_bytes=1 << 20)
  with pytest.raises(ValueError, match="devices"):
    edt.sdfsq(np.ones((4, 4, 4), np.uint8), devices=devices, max_device_bytes=0)


def test_max_device_bytes_rejects_negative(edt):
  with pytest.raises(ValueError, match="non-negative"):
    edt.edt3d(np.ones((4, 4, 4), np.uint8), max_device_bytes=-1)


def test_max_device_bytes_rejects_device_input(edt):
  class FakeDeviceArray:                     # what _device_array takes for device-resident input
    __module__ = "torch"
    is_cuda = True
    def dim(self):
      return 3
  with pytest.raises(ValueError, match="device-resident"):
    edt._front_door(FakeDeviceArray(), None, False, None, 0, 0, max_device_bytes=1 << 20)


def test_max_device_bytes_keyword_on_every_2d_3d_function(edt):
  import inspect
  for name in ("edt", "edtsq", "sdf", "sdfsq", "edt2d", "edt2dsq", "edt3d", "edt3dsq"):
    p = inspect.signature(getattr(edt, name)).parameters["max_device_bytes"]
    assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is None, name
  for name in ("edt1d", "edt1dsq"):
    assert "max_device_bytes" not in inspect.signature(getattr(edt, name)).parameters


def test_edt_error_carries_the_code(edt):
  lib = edt._lib()
  rc = lib.edtb200_transform_chunked(*_chunked(ndim=1))
  with pytest.raises(edt.EDTError) as info:
    edt._check(rc)
  assert info.value.code == EINVAL
  assert edt.EDTError("message").code is None


def test_budget_reaches_the_library_without_a_device(edt):
  """Without a GPU a chunked call fails at the device probe, as every transform does."""
  if edt.device_count() > 0:
    pytest.skip("a GPU is visible")
  with pytest.raises(edt.EDTError) as info:
    edt.edtsq(np.ones((4, 4, 4), np.uint8), max_device_bytes=1 << 20)
  assert info.value.code == ECUDA
