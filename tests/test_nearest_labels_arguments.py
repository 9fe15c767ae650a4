"""CPU tests: the argument checks of edtb200_nearest_labels in their documented order, its plan against
edtb200_bounded_plan (radii, the staged or global variant, the 256-row limit), the Python rejections of
nearest_labels -- each before any device is touched -- and its docstring.  A fully valid call stops at the
device probe (abi_checks.expect_probe)."""
import ctypes
import inspect
import re

import numpy as np
import pytest

import nearest_labels_cases as nc
from abi_checks import (ABI_VERSION, BIG, BOTH, EINVAL, ELIMIT, HEADER, INF, LABELS_FLOAT, LABELS_ON_DEVICE, NAN,
                        PROBE, SQRT, check_case, no_device_use)

SQUARED = 32

_IN = np.zeros(512, np.uint32)
_DIST = np.zeros(2048, np.float32)
_LAB = np.zeros(2048, np.uint32)
IN, DIST, LAB = _IN.ctypes.data, _DIST.ctypes.data, _LAB.ctypes.data


def _args(labels=IN, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, count=2, w=(1.0, 1.0, 1.0), d=3.0, k=2, flags=BOTH,
          dist=DIST, lab=LAB, device=63, stream=None):
  return (labels, label_bytes, ndim, sx, sy, sz, count, w[0], w[1], w[2], d, k, flags, dist, lab, device, stream)


CASES = [
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes"),
  ("ndim_0", dict(ndim=0), EINVAL, "ndim"),
  ("ndim_4", dict(ndim=4), EINVAL, "ndim"),
  ("negative_size", dict(sy=-1), EINVAL, "negative size"),
  ("axis_too_long", dict(sx=BIG), ELIMIT, "axis longer than 2^30"),
  ("negative_count", dict(count=-1), EINVAL, "negative count"),
  ("weight_zero", dict(w=(1.0, 0.0, 1.0)), EINVAL, "weight of axis 1"),
  ("weight_nan", dict(w=(1.0, 1.0, NAN)), EINVAL, "weight of axis 2"),
  ("weight_inf", dict(w=(INF, 1.0, 1.0)), EINVAL, "weight of axis 0"),
  ("k_0", dict(k=0), EINVAL, "k must be"),
  ("k_5", dict(k=5), EINVAL, "k must be"),
  ("d_negative", dict(d=-1.0), EINVAL, "max_distance"),
  ("d_nan", dict(d=NAN), EINVAL, "max_distance"),
  ("d_inf", dict(d=INF), EINVAL, "unbounded"),
  ("radius_257", dict(d=257.0), ELIMIT, "limit is 256"),
  ("radius_257_y", dict(w=(1.0, 0.5, 1.0), d=128.6), ELIMIT, "axis 1"),
  ("flag_sqrt", dict(flags=BOTH | SQRT), EINVAL, "residency flags"),
  ("flag_float", dict(flags=LABELS_FLOAT), EINVAL, "residency flags"),
  ("too_many_voxels", dict(count=1 << 60), ELIMIT, "too many voxels"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_dist", dict(dist=None), EINVAL, "null pointer"),
  ("null_lab", dict(lab=None), EINVAL, "null pointer"),
  ("outputs_overlap", dict(lab=DIST + 4), EINVAL, "dist_out overlaps label_out"),
  ("dist_overlaps_labels", dict(dist=IN + 4), EINVAL, "overlaps labels"),
  ("lab_overlaps_labels_host", dict(lab=IN, flags=0), EINVAL, "overlaps labels"),
  # order: label width, ndim, sizes, count, weights, k, max_distance, radius, flags, stack size, emptiness,
  # pointers and overlap, device
  ("width_before_ndim", dict(label_bytes=0, ndim=0), EINVAL, "label_bytes"),
  ("size_before_count", dict(sx=BIG, count=-1), ELIMIT, "axis longer"),
  ("count_before_weights", dict(count=-1, w=(0.0, 1.0, 1.0)), EINVAL, "negative count"),
  ("weights_before_k", dict(w=(1.0, NAN, 1.0), k=9), EINVAL, "weight of axis 1"),
  ("k_before_distance", dict(k=9, d=-1.0), EINVAL, "k must be"),
  ("distance_before_radius", dict(d=INF, w=(1e-30, 1.0, 1.0)), EINVAL, "max_distance"),
  ("radius_before_flags", dict(d=300.0, flags=SQRT), ELIMIT, "limit is 256"),
  ("radius_before_empty", dict(d=300.0, count=0), ELIMIT, "limit is 256"),
  ("flags_before_empty", dict(flags=SQRT, count=0), EINVAL, "residency flags"),
  ("no_volumes", dict(count=0, labels=None, dist=None, lab=None), 0, ""),
  ("empty_volume", dict(sz=0, labels=None, flags=0), 0, ""),
  ("valid", dict(), PROBE, ""),
  ("valid_squared", dict(flags=BOTH | SQUARED), PROBE, ""),
  ("valid_host", dict(flags=0), PROBE, ""),
  ("valid_mixed_overlap", dict(flags=LABELS_ON_DEVICE, dist=IN + 4), PROBE, ""),
  ("valid_radius_256", dict(d=256.0), PROBE, ""),
  ("valid_zero_distance", dict(d=0.0), PROBE, ""),
  ("radius_of_a_later_axis", dict(w=(1e20, 1.0, 1.0), d=1e30), ELIMIT, "axis 1"),
  ("valid_k_1_and_4", dict(k=4, label_bytes=8), PROBE, ""),
  ("valid_2d_ignores_sz_wz", dict(ndim=2, sz=-1, w=(1.0, 1.0, NAN)), PROBE, ""),
  ("valid_1d", dict(ndim=1, sy=-1, w=(2.0, 0.0, -1.0)), PROBE, ""),
]


@pytest.mark.parametrize("case,overrides,rc,msg", CASES, ids=[c[0] for c in CASES])
def test_nearest_labels_argument_check(edt, case, overrides, rc, msg):
  check_case(edt, edt._lib().edtb200_nearest_labels, _args, overrides, rc, msg)


def test_an_addition_at_the_same_version(edt):
  lib = edt._lib()
  assert lib.edtb200_version() == ABI_VERSION
  names = set(re.findall(r"\b(edtb200_[a-z0-9_]+)\s*\(", HEADER))
  assert {"edtb200_nearest_labels", "edtb200_nearest_labels_plan"} <= names
  for name, value in (("NEAREST_SQUARED", 32), ("NEAREST_ROWS", 0), ("NEAREST_STAGED", 1), ("NEAREST_GLOBAL", 2)):
    assert re.search(r"#define EDTB200_%s\s+%d\b" % (name, value), HEADER), name


# ---- the plan ---------------------------------------------------------------------------------------------

def _plan(edt, ndim, w, d, k, label_bytes, sizes=(8, 8, 8)):
  radius = (ctypes.c_int64 * 3)()
  variant = (ctypes.c_int * 3)()
  rc = edt._lib().edtb200_nearest_labels_plan(ndim, *sizes, *w, d, k, label_bytes, radius, variant)
  return rc, list(radius), list(variant)


def _bounded_radius(edt, ndim, w, d):
  radius = (ctypes.c_int64 * 3)()
  windowed = (ctypes.c_int * 3)()
  assert edt._lib().edtb200_bounded_plan(ndim, 8, 8, 8, *w, d, radius, windowed) == 0
  return list(radius)


WEIGHTS = [(1.0, 1.0, 1.0), (2.0, 1.0, 3.0), (0.7, 1.3, 2.9), (0.1, 0.3, 0.7), (1e20, 1.0, 1.0), (1.0, 1.0, 0.25)]


@pytest.mark.parametrize("w", WEIGHTS, ids=str)
@pytest.mark.parametrize("d", [0.0, 1.0, 2.5, 8.0, 24.0, 43.9, 44.0, 64.0, 256.0, 256.5])
def test_plan_radii_and_variants(edt, w, d):
  for ndim in (1, 2, 3):
    for k in (1, 2, 3, 4):
      for lb in (1, 2, 4, 8):
        rc, radius, variant = _plan(edt, ndim, w, d, k, lb)
        assert rc == 0
        want = _bounded_radius(edt, ndim, w, d)
        assert radius == [want[a] if a < ndim else 0 for a in range(3)]
        for a in range(3):
          assert radius[a] == (nc.radius_of(w[a], nc.bound_of(d)) if a < ndim else 0)
          if a >= ndim or radius[a] > 256:
            assert variant[a] == -1, (a, radius, variant)
          elif a == 0:
            assert variant[a] == 0
          else:
            smem = (64 + 2 * radius[a]) * 32 * k * (4 + lb)
            assert variant[a] == (1 if smem <= 232448 else 2), (a, radius, k, lb, variant)


def test_plan_limit_and_examples(edt):
  assert _plan(edt, 3, (1.0,) * 3, 256.0, 2, 4)[2] == [0, 2, 2]
  assert _plan(edt, 3, (1.0,) * 3, 256.5, 2, 4)[2] == [0, 2, 2]
  assert _plan(edt, 3, (1.0,) * 3, 257.0, 2, 4)[2] == [-1, -1, -1]
  assert _plan(edt, 2, (1.0, 0.5, 9.0), 128.0, 1, 1)[1:] == ([128, 256, 0], [0, 1, -1])
  assert _plan(edt, 3, (1.0,) * 3, 43.9, 4, 8)[2] == [0, 1, 1]
  assert _plan(edt, 3, (1.0,) * 3, 44.0, 4, 8)[2] == [0, 2, 2]
  assert _plan(edt, 3, (1.0,) * 3, 256.0, 1, 1)[2] == [0, 1, 1]          # k = 1 bytes stage every radius


def test_plan_checks(edt):
  assert _plan(edt, 4, (1.0,) * 3, 2.0, 2, 4)[0] == EINVAL
  assert _plan(edt, 3, (1.0, NAN, 1.0), 2.0, 2, 4)[0] == EINVAL
  assert _plan(edt, 3, (1.0,) * 3, 2.0, 5, 4)[0] == EINVAL
  assert _plan(edt, 3, (1.0,) * 3, INF, 2, 4)[0] == EINVAL
  assert _plan(edt, 3, (1.0,) * 3, 2.0, 2, 3)[0] == EINVAL
  lib = edt._lib()
  assert lib.edtb200_nearest_labels_plan(3, 8, 8, 8, 1.0, 1.0, 1.0, 2.0, 2, 4, None, None) == EINVAL
  assert b"null pointer" in lib.edtb200_last_error()


# ---- Python ---------------------------------------------------------------------------------------------

def test_exported(edt):
  assert "nearest_labels" in edt.__all__
  params = inspect.signature(edt.nearest_labels).parameters
  assert list(params)[:3] == ["labels", "max_distance", "anisotropy"]
  for kw, default in (("k", 2), ("squared", False), ("stacked", False), ("device", 0)):
    assert params[kw].kind is inspect.Parameter.KEYWORD_ONLY and params[kw].default == default, kw


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.float16, np.complex64])
def test_rejects_float_labels(no_device_use, dtype):
  with pytest.raises(TypeError, match="integer or bool"):
    no_device_use.nearest_labels(np.ones((4, 5), dtype), 2.0)


@pytest.mark.parametrize("k", [0, 5, -1, 2.0, True, "2"])
def test_rejects_bad_k(no_device_use, k):
  with pytest.raises(ValueError, match="k must be"):
    no_device_use.nearest_labels(np.ones((4, 5), np.uint8), 2.0, k=k)


@pytest.mark.parametrize("d", [-1.0, NAN, INF])
def test_rejects_bad_distance(no_device_use, d):
  with pytest.raises(ValueError, match="max_distance must be finite"):
    no_device_use.nearest_labels(np.ones((4, 5), np.uint8), d)


@pytest.mark.parametrize("w", [0.0, -1.0, NAN, INF])
def test_rejects_bad_weights(no_device_use, w):
  with pytest.raises(ValueError, match="finite and > 0"):
    no_device_use.nearest_labels(np.ones((4, 5), np.uint8), 2.0, (1.0, w))


def test_rejects_dimensions(no_device_use):
  fn = no_device_use.nearest_labels
  with pytest.raises(TypeError, match="1-D to 3-D"):
    fn(np.ones((2, 2, 2, 2), np.uint8), 2.0)
  with pytest.raises(TypeError, match="2-D to 4-D"):
    fn(np.ones(4, np.uint8), 2.0, stacked=True)
  with pytest.raises(ValueError, match="one entry per volume axis"):
    fn(np.ones((4, 5), np.uint8), 2.0, (1.0, 2.0, 3.0))


def test_radius_limit_from_python(edt):
  with pytest.raises(edt.EDTError) as err:
    edt.nearest_labels(np.ones((4, 5), np.uint8), 300.0)
  assert err.value.code == ELIMIT


def test_docstring_states_the_definition_and_the_worked_use(edt):
  doc = edt.nearest_labels.__doc__
  for phrase in ("parabolic_erode(np.where(labels == M, 0, np.inf), anisotropy)", "fl32(fl64(w2 * (i-j)^2) + fl64(g(j)))",
                 "float64(B) <= max_distance^2", "k smallest D_M(p)", "ties go to the", "U-Net weight map",
                 "w0 * np.exp(-(d[0] + d[1]) ** 2 / (2 * sigma ** 2))", "float labels raise TypeError", "ENOMEM",
                 "+inf and label 0", "k * (4 + itemsize)"):
    assert phrase in " ".join(doc.split()), phrase
