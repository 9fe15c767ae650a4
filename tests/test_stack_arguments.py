"""CPU tests: the argument checks of edtb200_transform_stack and edtb200_feature_transform_stack, and
the Python rejections of stacked=True.

As in test_chunked_arguments.py, every rejection comes with a return code and a message before any
device is touched, and a fully valid call stops at the device probe (abi_checks.expect_probe).  Nothing
here launches a kernel or copies a byte.
"""
import ctypes

import numpy as np
import pytest

from abi_checks import (ABI_VERSION, BIG, BOTH, ECUDA, EINVAL, ELIMIT, LABELS_ON_DEVICE, OUT_ON_DEVICE, PROBE, SIGNED,
                        SQRT, check_case)

# two separate host blocks: the checks only test for NULL and for overlap.  Each holds the largest extent a
# case passes (valid_1d: 300 volumes of 4 voxels, 4800 bytes), so that whether two valid extents overlap never
# depends on where the allocator placed the blocks
_LABELS = np.zeros(1024, np.uint64)
_OUT = np.zeros(1024, np.uint64)
L, O = _LABELS.ctypes.data, _OUT.ctypes.data


def ptrs(*values):
  return (ctypes.c_void_p * len(values))(*values)


def _stack(labels=L, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, count=2, w=(1.0, 1.0, 1.0), border=0, flags=0, out=O,
           device=63, device_bytes=0, groups=None, stream=None):
  return (labels, label_bytes, ndim, sx, sy, sz, count, *w, border, flags, out, device, device_bytes, groups, stream)


def _feature_stack(labels=L, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, count=2, w=(1.0, 1.0, 1.0), border=0, flags=0,
                   dist=None, idx=None, device=63, stream=None):
  idx = ptrs(O, O, O) if idx is None else idx
  return (labels, label_bytes, ndim, sx, sy, sz, count, *w, border, flags, dist, idx, device, stream)


STACK_CASES = [
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes"),
  ("label_bytes_16", dict(label_bytes=16), EINVAL, "label_bytes"),
  ("ndim_0", dict(ndim=0), EINVAL, "ndim"),
  ("ndim_4", dict(ndim=4), EINVAL, "ndim"),
  ("negative_size", dict(sy=-1), EINVAL, "negative size"),
  ("axis_too_long", dict(sx=BIG), ELIMIT, "axis longer than 2^30"),
  ("negative_count", dict(count=-1), EINVAL, "negative count"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_out", dict(out=None), EINVAL, "null pointer"),
  ("labels_on_device_only", dict(flags=LABELS_ON_DEVICE), EINVAL, "both on the device or both on the host"),
  ("out_on_device_only", dict(flags=OUT_ON_DEVICE | SQRT), EINVAL, "both on the device or both on the host"),
  # 2 volumes of 64 voxels: 512 label bytes and 512 output bytes
  ("same_buffer", dict(out=L), EINVAL, "labels and out overlap"),
  ("out_inside_labels", dict(out=L + 508), EINVAL, "labels and out overlap"),
  ("labels_inside_out", dict(labels=O + 508), EINVAL, "labels and out overlap"),
  # order: check_dims, count, emptiness, pointers, residency, overlap
  ("label_bytes_before_ndim", dict(label_bytes=3, ndim=4), EINVAL, "label_bytes"),
  ("size_before_count", dict(sx=BIG, count=-1), ELIMIT, "axis longer"),
  ("count_before_empty", dict(count=-1, sz=0), EINVAL, "negative count"),
  ("no_volumes", dict(count=0, labels=None, out=None, flags=LABELS_ON_DEVICE), 0, ""),
  ("empty_volume", dict(sy=0, labels=None, out=None), 0, ""),
  ("null_before_residency", dict(labels=None, flags=LABELS_ON_DEVICE), EINVAL, "null pointer"),
  ("residency_before_overlap", dict(out=L, flags=OUT_ON_DEVICE), EINVAL, "both on the device"),
  # on the device nothing is checked for overlap (in place is the caller's business); 2-D ignores sz
  ("valid_on_device_same_pointer", dict(out=L, flags=BOTH | SQRT), PROBE, ""),
  ("valid_adjacent", dict(out=L + 512), PROBE, ""),
  ("valid_2d_ignores_sz", dict(ndim=2, sz=-1), PROBE, ""),
  ("valid_1d", dict(ndim=1, sy=-1, sz=BIG, count=300), PROBE, ""),
  ("valid_budget", dict(device_bytes=1 << 20, flags=SQRT | SIGNED), PROBE, ""),
  ("valid_one_volume", dict(count=1), PROBE, ""),
  ("valid", dict(), PROBE, ""),
]

FEATURE_CASES = [
  ("label_bytes", dict(label_bytes=3), EINVAL, "label_bytes"),
  ("ndim", dict(ndim=4), EINVAL, "ndim"),
  ("negative_size", dict(sx=-4), EINVAL, "negative size"),
  ("axis_too_long", dict(ndim=1, sx=BIG), ELIMIT, "axis longer than 2^30"),
  ("negative_count", dict(count=-3), EINVAL, "negative count"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_planes", dict(idx=0), EINVAL, "null pointer"),
  ("null_plane_0", dict(idx=ptrs(None, O, O)), EINVAL, "null index plane 0"),
  ("null_plane_2", dict(idx=ptrs(O, O, None)), EINVAL, "null index plane 2"),
  ("count_before_empty", dict(count=-1, sz=0), EINVAL, "negative count"),
  ("no_volumes", dict(count=0, labels=None), 0, ""),
  ("empty_before_null", dict(sz=0, labels=None), 0, ""),
  ("label_bytes_before_count", dict(label_bytes=5, count=-1), EINVAL, "label_bytes"),
  ("ndim2_ignores_plane_2", dict(ndim=2, idx=ptrs(O, O, None)), PROBE, ""),
  ("ndim1_ignores_planes_1_2", dict(ndim=1, idx=ptrs(O, None, None)), PROBE, ""),
  ("valid", dict(), PROBE, ""),
  ("valid_with_distances", dict(dist=O), PROBE, ""),
  ("valid_on_device", dict(flags=BOTH, dist=O), PROBE, ""),
  ("valid_mixed", dict(flags=LABELS_ON_DEVICE), PROBE, ""),
]


@pytest.mark.parametrize("case,overrides,rc,msg", STACK_CASES, ids=[c[0] for c in STACK_CASES])
def test_transform_stack_argument_check(edt, case, overrides, rc, msg):
  groups = []

  def build(**kw):
    groups.append((ctypes.c_int64 * 1)(-7))
    return _stack(**kw, groups=groups[-1])
  check_case(edt, edt._lib().edtb200_transform_stack, build, overrides, rc, msg)
  assert all(g[0] == 0 for g in groups)                  # each call cleared its groups before any check


@pytest.mark.parametrize("case,overrides,rc,msg", FEATURE_CASES, ids=[c[0] for c in FEATURE_CASES])
def test_feature_transform_stack_argument_check(edt, case, overrides, rc, msg):
  check_case(edt, edt._lib().edtb200_feature_transform_stack, _feature_stack, overrides, rc, msg)


def test_stack_entry_points_are_additions_at_the_same_version(edt):
  lib = edt._lib()
  assert lib.edtb200_version() == ABI_VERSION
  assert hasattr(lib, "edtb200_transform_stack") and hasattr(lib, "edtb200_feature_transform_stack")


# ---- Python: stacked= ------------------------------------------------------------------------

FUNCTIONS = ("edt", "edtsq", "sdf", "sdfsq")


def test_stacked_keyword_on_every_function(edt):
  import inspect
  for name in FUNCTIONS + ("edt_cuda", "feature_transform"):
    p = inspect.signature(getattr(edt, name)).parameters["stacked"]
    assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is False, name


@pytest.mark.parametrize("name", FUNCTIONS)
def test_stacked_rejects_1d_and_5d(edt, name):
  fn = getattr(edt, name)
  with pytest.raises(ValueError, match="2-D to 4-D"):
    fn(np.ones(8, np.uint8), stacked=True)
  with pytest.raises(ValueError, match="2-D to 4-D"):
    fn(np.ones((2, 2, 2, 2, 2), np.uint8), stacked=True)
  with pytest.raises(ValueError, match="2-D to 4-D"):
    edt.feature_transform(np.ones(8, np.uint8), stacked=True)
  with pytest.raises(ValueError, match="2-D to 4-D"):
    edt.feature_transform(np.ones((2, 2, 2, 2, 2), np.uint8), stacked=True)


@pytest.mark.parametrize("name", FUNCTIONS)
def test_stacked_rejects_voxel_graph(edt, name):
  with pytest.raises(ValueError, match="voxel_graph"):
    getattr(edt, name)(np.ones((3, 4, 4), np.uint8), voxel_graph=np.full((3, 4, 4), 63, np.uint8), stacked=True)


@pytest.mark.parametrize("devices", [[0, 1], [0]])
def test_stacked_rejects_devices(edt, devices):
  for name in FUNCTIONS:
    with pytest.raises(ValueError, match="devices"):
      getattr(edt, name)(np.ones((3, 4, 4), np.uint8), devices=devices, stacked=True)


def test_stacked_rejects_anisotropy_of_the_wrong_length(edt):
  with pytest.raises(ValueError, match="one entry per volume axis"):
    edt.edtsq(np.ones((3, 4, 4), np.uint8), anisotropy=(1.0, 1.0, 1.0), stacked=True)
  with pytest.raises(ValueError, match="one entry per volume axis"):
    edt.feature_transform(np.ones((3, 4, 4), np.uint8), anisotropy=(1.0,), stacked=True)


def test_stacked_rejects_negative_budget(edt):
  with pytest.raises(ValueError, match="non-negative"):
    edt.edt(np.ones((3, 4, 4), np.uint8), max_device_bytes=-1, stacked=True)


def test_stacked_feature_transform_rejects_max_device_bytes(edt):
  with pytest.raises(ValueError, match="max_device_bytes"):
    edt.feature_transform(np.ones((3, 4, 4), np.uint8), max_device_bytes=1 << 20, stacked=True)


def test_stacked_rejects_budget_for_device_input(edt):
  class FakeDeviceArray:                     # what _device_array takes for device-resident input
    __module__ = "torch"
    is_cuda = True
    def dim(self):
      return 3
  with pytest.raises(ValueError, match="device-resident"):
    edt.edtsq(FakeDeviceArray(), max_device_bytes=1 << 20, stacked=True)


def test_stacked_empty_stack_touches_no_device(edt):
  out = edt.edtsq(np.ones((0, 4, 4), np.uint8), stacked=True)
  assert out.shape == (0, 4, 4) and out.dtype == np.float32
  out = edt.sdf(np.ones((5, 0, 4), np.uint32, order="F"), stacked=True)
  assert out.shape == (5, 0, 4)


def test_stacked_reaches_the_library_without_a_device(edt):
  """Without a GPU a stacked call fails at the device probe, as every transform does."""
  if edt.device_count() > 0:
    pytest.skip("a GPU is visible")
  with pytest.raises(edt.EDTError) as info:
    edt.edtsq(np.ones((3, 4, 4), np.uint8), stacked=True)
  assert info.value.code == ECUDA
  with pytest.raises(edt.EDTError) as info:
    edt.feature_transform(np.ones((3, 4, 4), np.uint8), stacked=True)
  assert info.value.code == ECUDA
