"""CPU tests (no GPU): host-side logic of the package and the C-ABI library itself.

No compute call is made here -- there is no GPU -- but the library must load, export every
symbol include/edt_b200.h declares, and refuse loudly to run without a device.
"""
import ctypes
import re

import numpy as np
import pytest

import abi_checks


def test_library_exports_every_declared_symbol(edt):
  header = abi_checks.HEADER
  declared = set(re.findall(r"\b(edtb200_[a-z0-9_]+)\s*\(", header))
  assert {"edtb200_transform", "edtb200_pass_first", "edtb200_pass_later", "edtb200_release",
          "edtb200_last_error", "edtb200_device_count", "edtb200_version"} <= declared
  lib = ctypes.CDLL(edt.library_path())
  for name in sorted(declared):
    assert hasattr(lib, name), name
  assert lib.edtb200_version() == int(re.search(r"#define EDTB200_VERSION (\d+)", header).group(1))


def test_header_flag_values_match_python(edt):
  vals = dict(re.findall(r"#define (EDTB200_[A-Z_]+)\s+(\d+)", abi_checks.HEADER))
  assert int(vals["EDTB200_SQRT"]) == edt.FLAG_SQRT
  assert int(vals["EDTB200_SIGNED"]) == edt.FLAG_SIGNED
  assert int(vals["EDTB200_LABELS_ON_DEVICE"]) == edt.FLAG_LABELS_ON_DEVICE
  assert int(vals["EDTB200_OUT_ON_DEVICE"]) == edt.FLAG_OUT_ON_DEVICE


_PARAM_TYPES = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "float": ctypes.c_float, "double": ctypes.c_double,
                "size_t": ctypes.c_size_t, "unsigned long long": ctypes.c_uint64, "uint64_t": ctypes.c_uint64}
_RESULT_TYPES = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "const char *": ctypes.c_char_p,
                 "void *": ctypes.c_void_p, "void": None}


def test_every_binding_matches_its_header_prototype(edt):
  """ctypes passes a value of the wrong width without complaint, so each binding must match the header."""
  lib = edt._lib()
  for name, (result, params) in abi_checks.prototypes().items():
    want = []
    for p in params:
      if name == "edtb200_slab_pack" and p.endswith("*y_start"):
        want.append(ctypes.POINTER(ctypes.c_int64))
      elif "*" in p or "[" in p:
        want.append(ctypes.c_void_p)
      else:
        want.append(_PARAM_TYPES[p.rsplit(" ", 1)[0]])
    fn = getattr(lib, name)
    assert list(fn.argtypes or []) == want, (name, fn.argtypes, want)
    assert fn.restype is _RESULT_TYPES[result], (name, fn.restype, result)


def test_no_silent_cpu_fallback(edt):
  """Without a device every transform must raise (the product has no CPU path)."""
  if edt.device_count() > 0:
    pytest.skip("a GPU is visible")
  with pytest.raises(edt.EDTError):
    edt.edtsq(np.ones((4, 4, 4), np.uint8))
  with pytest.raises(edt.EDTError):
    edt.sdf(np.ones((8,), np.uint8))


def test_argument_validation_in_c_abi(edt):
  lib = edt._lib()
  buf = np.zeros(8, np.float32)
  rc = lib.edtb200_transform(buf.ctypes.data, 3, 3, 2, 2, 2, 1.0, 1.0, 1.0, 0, 0, buf.ctypes.data, 0, None)
  assert rc == -1 and b"label_bytes" in lib.edtb200_last_error()
  rc = lib.edtb200_transform(buf.ctypes.data, 4, 4, 2, 2, 2, 1.0, 1.0, 1.0, 0, 0, buf.ctypes.data, 0, None)
  assert rc == -1 and b"ndim" in lib.edtb200_last_error()
  # empty volumes succeed without touching a device
  assert lib.edtb200_transform(buf.ctypes.data, 4, 3, 0, 2, 2, 1.0, 1.0, 1.0, 0, 0, buf.ctypes.data, 0, None) == 0


def test_front_door_mirrors_reference(edt):
  # empty input -> zeros of the same shape (src/edt.pyx:281-282), no device needed
  assert edt.edtsq(np.zeros((0, 3), np.uint8)).shape == (0, 3)
  assert edt.edt([]).shape == (0,)
  with pytest.raises(TypeError):
    edt.edtsq(np.zeros((2, 2, 2, 2), np.uint8))       # src/edt.pyx:310
  with pytest.raises(TypeError):
    edt.edtsq(np.zeros((4,), np.uint8), voxel_graph=np.zeros((4,), np.uint8))   # src/edt.pyx:291-292
  with pytest.raises(ValueError):
    edt.edtsq(np.zeros((4, 4), np.uint8), voxel_graph=np.zeros((4, 5), np.uint8))


def test_axis_mapping(edt):
  # src/edt.pyx:651-664: C order reverses axes and anisotropy, F order keeps them
  assert edt._x_fastest((2, 3, 4), (5, 6, 7), False) == ([4, 3, 2], [7.0, 6.0, 5.0])
  assert edt._x_fastest((2, 3, 4), (5, 6, 7), True) == ([2, 3, 4], [5.0, 6.0, 7.0])
  assert edt._x_fastest((9, 4), (2, 3), False) == ([4, 9, 1], [3.0, 2.0, 1.0])
  assert edt._x_fastest((9,), (2,), True) == ([9, 1, 1], [2.0, 1.0, 1.0])
  with pytest.raises(ValueError):
    edt._x_fastest((2, 3), (1, 2, 3), True)


def test_label_views(edt):
  # src/edt.pyx:670-732
  a = np.array([-1, 0, 5], dtype=np.int16)
  v = edt._label_view(a)
  assert v.dtype == np.uint16 and v[0] == 65535
  b = np.array([True, False])
  assert edt._label_view(b).dtype == np.uint8
  f = np.array([0.0, -0.0, 1.5], dtype=np.float32)
  v = edt._label_view(f)
  assert v.dtype == np.uint32 and v[0] == 0 and v[1] == 0 and v[2] != 0
  d = np.array([-0.0, 2.0], dtype=np.float64)
  assert edt._label_view(d)[0] == 0
  assert edt._label_view(np.zeros(3, np.float16)) is None


@pytest.mark.gpu
def test_each_mirrors_reference_contract(edt):
  """edt.each (src/edt.pyx:951-994, automated_test.py:831-856): per-label images from one
  multi-label transform; the images are drawn on the device (csrc/edt_each.cuh)."""
  rng = np.random.default_rng(8)
  labels = rng.integers(0, 6, (9, 8, 7)).astype(np.uint32)
  dt = rng.random((9, 8, 7)).astype(np.float32) * (labels != 0)
  for in_place in (False, True):
    it = edt.each(labels, dt, in_place=in_place)
    assert len(it) == len(set(np.unique(labels)) - {0})
    seen = []
    for label, img in it:
      assert np.array_equal(img, (labels == label) * dt)
      assert img.dtype == np.float32
      if in_place:
        assert not img.flags.writeable
      seen.append(int(label))
    assert seen == sorted(seen) and 0 not in seen
  f = np.asfortranarray(labels)
  _, img = next(iter(edt.each(f, np.asfortranarray(dt))))
  assert img.flags.f_contiguous
