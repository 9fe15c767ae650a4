"""CPU tests: the argument checks of edtb200_surface_count and edtb200_surface_distances, and the Python
rejections of surface_distances, hausdorff_distance, average_surface_distance and surface_dice.

As in test_expand_stack_arguments.py, every rejection comes with a return code and a message before
any device is touched, and a fully valid call stops at the device probe (abi_checks.expect_probe).  Nothing
here launches a kernel or copies a byte.
"""
import ctypes
import functools
import inspect
import re

import numpy as np
import pytest

from abi_checks import (ABI_VERSION, BIG, BOTH, ECUDA, EINVAL, ELIMIT, HEADER, LABELS_ON_DEVICE, OUT_ON_DEVICE, PROBE,
                        SQRT, check_case)

# separate host blocks: the checks only test for NULL (the keys are read: they are host memory)
_A = np.zeros(512, np.uint64)
_B = np.zeros(512, np.uint64)
_OUT = np.zeros(512, np.int64)
A, B, OUT = _A.ctypes.data, _B.ctypes.data, _OUT.ctypes.data


def keys(values, label_bytes=4):
  arr = np.asarray(values, dtype="u%d" % label_bytes)
  keys.keep.append(arr)
  return arr.ctypes.data


keys.keep = []
K3 = keys([1, 2, 9])


def _count(a=A, b=B, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, count=2, keys=K3, nkeys=3, flags=BOTH, counts=OUT,
           device=63, stream=None):
  return (a, b, label_bytes, ndim, sx, sy, sz, count, keys, nkeys, flags, counts, device, stream)


def _dist(a=A, b=B, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, count=2, keys=K3, nkeys=3, flags=BOTH, offsets=OUT,
          values=OUT, device=63, device_bytes=0, groups=None, stream=None):
  return (a, b, label_bytes, ndim, sx, sy, sz, count, 1.0, 1.0, 1.0, keys, nkeys, flags, offsets, values, device,
          device_bytes, groups, stream)


# overrides shared by both calls (counts / offsets+values are "out")
CASES = [
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes"),
  ("ndim_0", dict(ndim=0), EINVAL, "ndim"),
  ("ndim_4", dict(ndim=4), EINVAL, "ndim"),
  ("negative_size", dict(sy=-1), EINVAL, "negative size"),
  ("axis_too_long", dict(sx=BIG), ELIMIT, "axis longer than 2^30"),
  ("negative_count", dict(count=-1), EINVAL, "negative count"),
  ("negative_nkeys", dict(nkeys=-1), EINVAL, "negative nkeys"),
  ("null_keys", dict(keys=None), EINVAL, "null pointer (keys)"),
  ("key_zero", dict(keys=keys([0, 2, 9])), EINVAL, "key 0 is 0"),
  ("key_zero_later", dict(keys=keys([1, 0, 9])), EINVAL, "key 1 is 0"),
  ("keys_descending", dict(keys=keys([1, 9, 2])), EINVAL, "strictly ascending (key 2)"),
  ("keys_repeated", dict(keys=keys([1, 2, 2])), EINVAL, "strictly ascending (key 2)"),
  ("keys_unsigned_order", dict(keys=keys([2, 0xFFFFFFFF, 1])), EINVAL, "strictly ascending (key 2)"),
  ("too_many_pairs", dict(count=1 << 60, nkeys=3), ELIMIT, "too many"),
  ("null_a", dict(a=None), EINVAL, "null pointer"),
  ("null_b", dict(b=None), EINVAL, "null pointer"),
  ("null_out", dict(out=None), EINVAL, "null pointer"),
  ("host_buffers", dict(flags=0), EINVAL, "device buffers only"),
  ("labels_on_host", dict(flags=OUT_ON_DEVICE), EINVAL, "device buffers only"),
  ("out_on_host", dict(flags=LABELS_ON_DEVICE), EINVAL, "device buffers only"),
  ("unknown_flag", dict(flags=BOTH | SQRT), EINVAL, "device buffers only"),
  # order: label width, ndim, sizes, count, nkeys and the keys, emptiness, pointers, residency, device
  ("label_bytes_before_ndim", dict(label_bytes=3, ndim=4), EINVAL, "label_bytes"),
  ("ndim_before_size", dict(ndim=5, sx=-1), EINVAL, "ndim"),
  ("size_before_count", dict(sx=BIG, count=-1), ELIMIT, "axis longer"),
  ("count_before_nkeys", dict(count=-1, nkeys=-1), EINVAL, "negative count"),
  ("nkeys_before_keys", dict(nkeys=-1, keys=None), EINVAL, "negative nkeys"),
  ("keys_before_empty", dict(keys=keys([3, 2, 1]), sy=0), EINVAL, "strictly ascending"),
  ("keys_before_pointers", dict(keys=keys([3, 2, 1]), a=None), EINVAL, "strictly ascending"),
  ("no_volumes", dict(count=0, a=None, b=None, out=None, flags=0), 0, ""),
  ("empty_volume", dict(sz=0, a=None, b=None, out=None, flags=0), 0, ""),
  ("no_keys", dict(nkeys=0, keys=None, a=None, out=None, flags=0), 0, ""),
  ("pointers_before_residency", dict(a=None, flags=0), EINVAL, "null pointer"),
  ("valid", dict(), PROBE, ""),
  ("valid_1_byte_keys", dict(label_bytes=1, keys=keys([1, 200, 255], 1)), PROBE, ""),
  ("valid_8_byte_keys", dict(label_bytes=8, keys=keys([1, 1 << 40, (1 << 64) - 1], 8)), PROBE, ""),
  ("valid_2d_ignores_sz", dict(ndim=2, sz=-1), PROBE, ""),
  ("valid_1d_ignores_sy_sz", dict(ndim=1, sy=-1, sz=BIG), PROBE, ""),
  ("valid_one_key", dict(nkeys=1), PROBE, ""),
]


def _args(fn, out=OUT, **o):
  if fn == "count":
    return _count(counts=out, **o)
  return _dist(offsets=out, values=out, **o)


@pytest.mark.parametrize("fn", ["count", "distances"])
@pytest.mark.parametrize("case,overrides,rc,msg", CASES, ids=[c[0] for c in CASES])
def test_surface_argument_check(edt, fn, case, overrides, rc, msg):
  lib = edt._lib()
  call = lib.edtb200_surface_count if fn == "count" else lib.edtb200_surface_distances
  check_case(edt, call, functools.partial(_args, fn), overrides, rc, msg)


def test_distances_null_offsets_and_values(edt):
  lib = edt._lib()
  for o in (dict(offsets=None), dict(values=None)):
    assert lib.edtb200_surface_distances(*_dist(**o)) == EINVAL
    assert b"null pointer" in lib.edtb200_last_error()


def test_distances_groups_zeroed_on_error_and_empty(edt):
  lib = edt._lib()
  g = (ctypes.c_int64 * 1)(7)
  assert lib.edtb200_surface_distances(*_dist(groups=g, nkeys=-1)) == EINVAL and g[0] == 0
  g[0] = 7
  assert lib.edtb200_surface_distances(*_dist(groups=g, count=0)) == 0 and g[0] == 0


def test_surface_entry_points_are_additions_at_the_same_version(edt):
  lib = edt._lib()
  assert lib.edtb200_version() == ABI_VERSION
  declared = set(re.findall(r"\b(edtb200_[a-z0-9_]+)\s*\(", HEADER))
  assert {"edtb200_surface_count", "edtb200_surface_distances"} <= declared
  raw = ctypes.CDLL(edt.library_path())
  assert hasattr(raw, "edtb200_surface_count") and hasattr(raw, "edtb200_surface_distances")
  assert lib.edtb200_surface_distances.argtypes[17] is ctypes.c_size_t


# ---- Python ---------------------------------------------------------------------------------------------

FNS = ["surface_distances", "hausdorff_distance", "average_surface_distance", "surface_dice"]


def _call(edt, name, a, b, *args, **kw):
  fn = getattr(edt, name)
  if name == "surface_dice":
    return fn(a, b, kw.pop("tolerance", 1.0), *args, **kw)
  return fn(a, b, *args, **kw)


def test_exported(edt):
  for name in FNS + ["SurfaceDistances"]:
    assert name in edt.__all__ and hasattr(edt, name)
  assert edt.SurfaceDistances._fields == ("labels", "offsets", "values")
  for name in FNS:
    params = inspect.signature(getattr(edt, name)).parameters
    for kw in ("labels", "stacked", "device", "max_device_bytes"):
      assert params[kw].kind is inspect.Parameter.KEYWORD_ONLY, (name, kw)
    assert params["stacked"].default is False and params["labels"].default is None


@pytest.mark.parametrize("name", FNS)
def test_rejects_mismatched_shapes(edt, name):
  with pytest.raises(ValueError, match="one shape"):
    _call(edt, name, np.ones((4, 5), np.uint8), np.ones((5, 4), np.uint8))


@pytest.mark.parametrize("name", FNS)
def test_rejects_mismatched_dtypes(edt, name):
  with pytest.raises(TypeError, match="one dtype"):
    _call(edt, name, np.ones((4, 5), np.uint8), np.ones((4, 5), np.int32))


@pytest.mark.parametrize("name", FNS)
def test_rejects_anisotropy_of_the_wrong_length(edt, name):
  with pytest.raises(ValueError, match="one entry per volume axis"):
    _call(edt, name, np.ones((4, 5), np.uint8), np.ones((4, 5), np.uint8), (1.0, 2.0, 3.0))
  with pytest.raises(ValueError, match="one entry per volume axis"):
    _call(edt, name, np.ones(6, np.uint8), np.ones(6, np.uint8), (1.0, 2.0))
  with pytest.raises(ValueError, match="one entry per volume axis"):
    _call(edt, name, np.ones((3, 4, 5), np.uint8), np.ones((3, 4, 5), np.uint8), (1.0, 2.0, 3.0), stacked=True)


@pytest.mark.parametrize("name", FNS)
def test_rejects_key_zero(edt, name):
  for labels in ([0], [1, 0], [2.0, -0.0]):
    dtype = np.float32 if isinstance(labels[-1], float) else np.uint8
    with pytest.raises(ValueError, match="must not contain 0"):
      _call(edt, name, np.ones((4, 5), dtype), np.ones((4, 5), dtype), labels=labels)


@pytest.mark.parametrize("name", FNS)
def test_rejects_repeated_keys(edt, name):
  with pytest.raises(ValueError, match="distinct"):
    _call(edt, name, np.ones((4, 5), np.int16), np.ones((4, 5), np.int16), labels=[3, -1, 3])


@pytest.mark.parametrize("name", FNS)
def test_rejects_unsupported_dtypes_and_ranks(edt, name):
  with pytest.raises(TypeError, match="unsupported label dtype"):
    _call(edt, name, np.ones(4, np.float16), np.ones(4, np.float16))
  with pytest.raises(TypeError, match="1-D to 3-D"):
    _call(edt, name, np.ones((2, 2, 2, 2), np.uint8), np.ones((2, 2, 2, 2), np.uint8))
  with pytest.raises(ValueError, match="2-D to 4-D"):
    _call(edt, name, np.ones(4, np.uint8), np.ones(4, np.uint8), stacked=True)


@pytest.mark.parametrize("name", FNS)
def test_rejects_negative_budget(edt, name):
  with pytest.raises(ValueError, match="max_device_bytes"):
    _call(edt, name, np.ones((4, 5), np.uint8), np.ones((4, 5), np.uint8), max_device_bytes=-1)


def test_rejects_percentile_outside_0_100(edt):
  x = np.ones((4, 5), np.uint8)
  for p in (-0.5, 100.5, float("nan"), float("inf")):
    with pytest.raises(ValueError, match="percentile"):
      edt.hausdorff_distance(x, x, percentile=p)


def test_rejects_negative_tolerance(edt):
  x = np.ones((4, 5), np.uint8)
  for t in (-1e-9, -3.0, float("nan")):
    with pytest.raises(ValueError, match="tolerance"):
      edt.surface_dice(x, x, t)


def test_empty_volumes_touch_no_device(edt, monkeypatch):
  def no_device(*args):
    raise AssertionError("an empty volume reached the library")
  monkeypatch.setattr(edt, "device_count", no_device)
  monkeypatch.setattr(edt, "_lib", no_device)
  x = np.zeros((0, 4), np.uint8)
  sd = edt.surface_distances(x, x)
  assert sd.labels.size == 0 and sd.offsets.tolist() == [0] and sd.values.size == 0
  sd = edt.surface_distances(x, x, labels=[1, 5])
  assert sd.labels.tolist() == [1, 5] and sd.offsets.tolist() == [0] * 5
  hd = edt.hausdorff_distance(x, x, labels=[1, 5])
  assert hd.shape == (2,) and np.isnan(hd).all()
  y = np.zeros((3, 0, 4), np.float32)
  assert edt.surface_dice(y, y, 1.0, labels=[2.5], stacked=True).shape == (3, 1)

def test_reaches_the_library_without_a_device(edt):
  """Without a GPU a valid call fails with ECUDA, as every transform does."""
  if edt.device_count() > 0:
    pytest.skip("a GPU is visible")
  x = np.ones((4, 5), np.uint8)
  for name in FNS:
    with pytest.raises(edt.EDTError) as info:
      _call(edt, name, x, x)
    assert info.value.code == ECUDA
