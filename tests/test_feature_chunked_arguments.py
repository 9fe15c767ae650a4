"""CPU tests: the argument checks of edtb200_feature_transform_chunked and of the Python keyword
max_device_bytes on feature_transform / expand_labels.

As in test_chunked_arguments.py, every rejection comes with a return code and a message before any
device is touched, and a fully valid call stops at the device probe (abi_checks.expect_probe).  Nothing
here launches a kernel or copies a byte.
"""
import ctypes
import itertools

import numpy as np
import pytest

from abi_checks import (ABI_VERSION, BIG, ECUDA, EINVAL, ELIMIT, LABELS_ON_DEVICE, OUT_ON_DEVICE, PROBE, SIGNED, SQRT,
                        check_case)

# separate host blocks: the checks only test for NULL and for overlap.  64 voxels: 256 label bytes
# (label_bytes 4), 256 bytes per distance volume and index plane.
_BLOCKS = [np.zeros(256, np.uint64) for _ in range(5)]
L, D, X, Y, Z = (b.ctypes.data for b in _BLOCKS)


def _planes(*ptrs):
  return (ctypes.c_void_p * 3)(*ptrs)


def _call(labels=L, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, w=(1.0, 1.0, 1.0), border=0, flags=0, dist=D,
          idx=(X, Y, Z), device=63, device_bytes=0, chunks=None):
  idx = None if idx is None else _planes(*idx)
  return (labels, label_bytes, ndim, sx, sy, sz, *w, border, flags, dist, idx, device, device_bytes, chunks)


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
  ("negative_sx", dict(sx=-4), EINVAL, "negative size"),
  ("axis_too_long", dict(sx=BIG), ELIMIT, "axis longer than 2^30"),
  ("z_too_long", dict(sz=BIG), ELIMIT, "axis longer than 2^30"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_planes", dict(idx=None), EINVAL, "null pointer"),
  ("null_plane_0", dict(idx=(None, Y, Z)), EINVAL, "null index plane 0"),
  ("null_plane_1", dict(idx=(X, None, Z)), EINVAL, "null index plane 1"),
  ("null_plane_2", dict(idx=(X, Y, None)), EINVAL, "null index plane 2"),
  ("null_plane_1_2d", dict(ndim=2, sz=1, idx=(X, None, None)), EINVAL, "null index plane 1"),
  # order: residency, dimensionality, label width, emptiness, pointers, overlap
  ("flags_before_ndim", dict(flags=OUT_ON_DEVICE, ndim=1), EINVAL, "HOST buffers"),
  ("ndim_before_label_bytes", dict(ndim=1, label_bytes=3), EINVAL, "2-D or 3-D"),
  ("label_bytes_before_null", dict(label_bytes=3, labels=None), EINVAL, "label_bytes"),
  ("empty_before_null", dict(sz=0, labels=None, idx=None), 0, ""),
  ("null_before_overlap", dict(labels=None, dist=X), EINVAL, "null pointer"),
  ("wide_labels_reach_dist", dict(label_bytes=8, dist=L + 511), EINVAL, "labels and dist_out overlap"),
  # adjacent buffers do not overlap; 2-D ignores sz and the third plane; dist_out may be NULL
  ("valid_adjacent", dict(dist=L + 256, idx=(L + 512, L + 768, L + 1024)), PROBE, ""),
  ("valid_adjacent_below", dict(labels=X + 256, dist=X + 512, idx=(X, X - 256, X - 512)), PROBE, ""),
  ("valid_2d_ignores_sz", dict(ndim=2, sz=-1, idx=(X, Y, L)), PROBE, ""),
  ("valid_no_dist", dict(dist=None), PROBE, ""),
  ("valid_budget", dict(device_bytes=1 << 20, flags=SQRT | SIGNED), PROBE, ""),
  ("valid", dict(), PROBE, ""),
]

# every pair of the five buffers, overlapping by one byte at either end or lying on each other
NAMES = ["labels", "dist_out", "index plane 0", "index plane 1", "index plane 2"]


def _overlap_cases():
  out = []
  for i, j in itertools.combinations(range(5), 2):
    for shift, how in ((0, "same"), (255, "end"), (-255, "start")):
      ptrs = [L, D, X, Y, Z]
      ptrs[j] = ptrs[i] + shift
      out.append(("%s-%s-%s" % (NAMES[i], NAMES[j], how), ptrs, "%s and %s overlap" % (NAMES[i], NAMES[j])))
  return out


@pytest.mark.parametrize("case,overrides,rc,msg", CASES, ids=[c[0] for c in CASES])
def test_feature_chunked_argument_check(edt, case, overrides, rc, msg):
  chunks = []

  def build(**kw):
    chunks.append((ctypes.c_int64 * 2)(-7, -7))
    return _call(**kw, chunks=chunks[-1])
  check_case(edt, edt._lib().edtb200_feature_transform_chunked, build, overrides, rc, msg)
  assert all(list(c) == [0, 0] for c in chunks)          # each call cleared its chunks before any check


@pytest.mark.parametrize("case,ptrs,msg", _overlap_cases(), ids=[c[0] for c in _overlap_cases()])
def test_feature_chunked_overlap(edt, case, ptrs, msg):
  lib = edt._lib()
  chunks = (ctypes.c_int64 * 2)(-7, -7)
  got = lib.edtb200_feature_transform_chunked(*_call(labels=ptrs[0], dist=ptrs[1], idx=ptrs[2:], chunks=chunks))
  err = lib.edtb200_last_error() or b""
  assert got == EINVAL and msg.encode() in err, (got, err)
  assert list(chunks) == [0, 0]


def test_feature_chunked_is_an_addition_at_the_same_version(edt):
  lib = edt._lib()
  assert lib.edtb200_version() == ABI_VERSION
  assert hasattr(lib, "edtb200_feature_transform_chunked") and hasattr(lib, "edtb200_transform_chunked")


# ---- Python: max_device_bytes ----------------------------------------------------------------

class FakeDeviceArray:                       # what _device_array takes for device-resident input
  __module__ = "torch"
  is_cuda = True

  def dim(self):
    return 3


def test_feature_transform_budget_rejections(edt):
  with pytest.raises(ValueError, match="2-D or 3-D"):
    edt.feature_transform(np.ones(8, np.uint8), max_device_bytes=1 << 20)
  with pytest.raises(ValueError, match="2-D or 3-D"):
    edt.feature_transform(np.ones((2, 2, 2, 2), np.uint8), max_device_bytes=0)
  with pytest.raises(ValueError, match="non-negative"):
    edt.feature_transform(np.ones((4, 4), np.uint8), max_device_bytes=-1)
  with pytest.raises(ValueError, match="device-resident"):
    edt.feature_transform(FakeDeviceArray(), max_device_bytes=1 << 20)


def test_expand_labels_budget_rejections(edt):
  pytest.importorskip("torch")
  with pytest.raises(ValueError, match="2-D or 3-D"):
    edt.expand_labels(np.ones(8, np.uint8), max_device_bytes=1 << 20)
  with pytest.raises(ValueError, match="non-negative"):
    edt.expand_labels(np.ones((4, 4, 4), np.uint16), max_device_bytes=-5)
  with pytest.raises(ValueError, match="device-resident"):
    edt.expand_labels(FakeDeviceArray(), max_device_bytes=0)


def test_max_device_bytes_keyword(edt):
  import inspect
  for fn in (edt.feature_transform, edt.expand_labels):
    p = inspect.signature(fn).parameters["max_device_bytes"]
    assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is None, fn.__name__


def test_budget_reaches_the_library_without_a_device(edt):
  """Without a GPU a chunked feature transform fails at the device probe, as every transform does."""
  if edt.device_count() > 0:
    pytest.skip("a GPU is visible")
  with pytest.raises(edt.EDTError) as info:
    edt.feature_transform(np.ones((4, 4, 4), np.uint8), max_device_bytes=1 << 20)
  assert info.value.code == ECUDA
