"""CPU tests: the argument checks of edtb200_geodesic in their documented order, the header's parameter
names and version comment, the Python rejections of geodesic_distance -- each before any device is touched
-- and the statements of its docstring and the header, with the docstring's examples checked on the CPU
restatement.  A fully valid call stops at the device probe (abi_checks.expect_probe)."""
import ctypes
import inspect
import re

import numpy as np
import pytest

import geodesic_cases as gc
from abi_checks import (ABI_VERSION, BIG, BOTH, EINVAL, ELIMIT, HEADER, INF, LABELS_FLOAT, LABELS_ON_DEVICE, NAN,
                        PROBE, SQRT, check_case, header_doc, no_device_use, prototypes)

_LAB = np.zeros(128, np.uint32)          # 2 volumes of 4 x 4 x 4
_SEED = np.zeros(128, np.uint8)
_DIST = np.zeros(128, np.float32)
_PL = np.zeros((3, 128), np.int32)
LAB, SEED, DIST = _LAB.ctypes.data, _SEED.ctypes.data, _DIST.ctypes.data
P0, P1, P2 = (_PL[k].ctypes.data for k in range(3))


def _planes(*ptrs):
  return (ctypes.c_void_p * len(ptrs))(*ptrs)


def _args(labels=LAB, label_bytes=4, seeds=SEED, seed_bytes=1, ndim=3, sx=4, sy=4, sz=4, count=2,
          w=(1.0, 1.0, 1.0), flags=BOTH, dist=DIST, idx=None, device=63, stream=None):
  return (labels, label_bytes, seeds, seed_bytes, ndim, sx, sy, sz, count, w[0], w[1], w[2], flags, dist, idx, device,
          stream)


CASES = [
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes must be"),
  ("label_bytes_0", dict(label_bytes=0), EINVAL, "label_bytes must be"),
  ("seed_bytes_3", dict(seed_bytes=3), EINVAL, "seed_bytes must be"),
  ("seed_bytes_16", dict(seed_bytes=16), EINVAL, "seed_bytes must be"),
  ("ndim_0", dict(ndim=0), EINVAL, "ndim must be 1, 2 or 3"),
  ("ndim_4", dict(ndim=4), EINVAL, "ndim must be 1, 2 or 3"),
  ("negative_size", dict(sy=-1), EINVAL, "negative size"),
  ("axis_too_long", dict(sz=BIG), ELIMIT, "axis longer than 2^30"),
  ("negative_count", dict(count=-1), EINVAL, "negative count"),
  ("weight_zero", dict(w=(1.0, 0.0, 1.0)), EINVAL, "weight of axis 1"),
  ("weight_negative", dict(w=(-1.0, 1.0, 1.0)), EINVAL, "weight of axis 0"),
  ("weight_nan", dict(w=(1.0, 1.0, NAN)), EINVAL, "weight of axis 2"),
  ("weight_inf", dict(w=(INF, 1.0, 1.0)), EINVAL, "weight of axis 0"),
  ("flag_sqrt", dict(flags=BOTH | SQRT), EINVAL, "only the residency flags"),
  ("flag_float", dict(flags=LABELS_FLOAT), EINVAL, "only the residency flags"),
  ("too_many_voxels", dict(count=1 << 60), ELIMIT, "too many voxels"),
  ("too_many_tiles", dict(ndim=1, sx=1, count=1 << 32, labels=None), ELIMIT, "fewer than 2^32 tiles"),
  ("tiles_just_below", dict(ndim=1, sx=1, count=(1 << 32) - 1, labels=None), EINVAL, "null pointer"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_seeds", dict(seeds=None), EINVAL, "null pointer"),
  ("null_dist", dict(dist=None), EINVAL, "null pointer"),
  ("null_plane", dict(idx=_planes(P0, None, P2)), EINVAL, "null index plane 1"),
  ("dist_overlaps_labels", dict(dist=LAB + 8), EINVAL, "dist_out overlaps labels"),
  ("dist_overlaps_seeds", dict(dist=SEED + 4), EINVAL, "dist_out overlaps seeds"),
  ("dist_overlaps_labels_host", dict(dist=LAB - 4 * 128 + 4, flags=0), EINVAL, "dist_out overlaps labels"),
  ("plane_overlaps_labels", dict(idx=_planes(P0, LAB, P2)), EINVAL, "index plane 1 overlaps labels"),
  ("plane_overlaps_dist", dict(idx=_planes(P0, P1, DIST + 4)), EINVAL, "index plane 2 overlaps dist_out"),
  ("planes_overlap", dict(idx=_planes(P0, P0 + 4, P2)), EINVAL, "index plane 1 overlaps index plane 0"),
  # order: label width, seed width, ndim, sizes, count, weights, flags, stack size, tiles, emptiness, pointers,
  # overlap, device
  ("label_width_before_seed_width", dict(label_bytes=5, seed_bytes=5), EINVAL, "label_bytes must be"),
  ("seed_width_before_ndim", dict(seed_bytes=5, ndim=0), EINVAL, "seed_bytes must be"),
  ("ndim_before_size", dict(ndim=5, sx=-1), EINVAL, "ndim"),
  ("size_before_count", dict(sx=BIG, count=-1), ELIMIT, "axis longer"),
  ("count_before_weights", dict(count=-1, w=(0.0, 0.0, 0.0)), EINVAL, "negative count"),
  ("weights_before_flags", dict(w=(1.0, NAN, 1.0), flags=SQRT), EINVAL, "weight of axis 1"),
  ("flags_before_stack", dict(flags=SQRT, count=1 << 60), EINVAL, "only the residency flags"),
  ("stack_before_tiles", dict(ndim=1, sx=1 << 30, count=1 << 40), ELIMIT, "too many voxels"),
  ("tiles_before_empty", dict(ndim=1, sx=1, count=1 << 33, labels=None, dist=None), ELIMIT, "tiles"),
  ("weights_before_empty", dict(w=(0.0, 1.0, 1.0), count=0), EINVAL, "weight of axis 0"),
  ("flags_before_empty", dict(flags=SQRT, count=0), EINVAL, "only the residency flags"),
  ("no_volumes", dict(count=0, labels=None, seeds=None, dist=None), 0, ""),
  ("empty_volume", dict(sz=0, labels=None, seeds=None, dist=None, flags=0), 0, ""),
  ("pointers_before_overlap", dict(seeds=None, dist=LAB), EINVAL, "null pointer"),
  ("overlap_before_device", dict(dist=SEED, device=64), EINVAL, "dist_out overlaps seeds"),
  ("valid", dict(), PROBE, ""),
  ("valid_indices", dict(idx=_planes(P0, P1, P2)), PROBE, ""),
  ("valid_host", dict(flags=0, idx=_planes(P0, P1, P2)), PROBE, ""),
  ("valid_8_byte", dict(label_bytes=8, seed_bytes=8, count=1), PROBE, ""),
  ("valid_mixed_outputs_on_labels", dict(dist=LAB, flags=LABELS_ON_DEVICE), PROBE, ""),
  ("valid_same_labels_and_seeds", dict(seeds=LAB, seed_bytes=4), PROBE, ""),
  ("valid_1d_one_plane", dict(ndim=1, sy=-1, sz=-1, w=(1.0, NAN, NAN), idx=_planes(P0)), PROBE, ""),
  ("valid_2d_ignores_sz_wz", dict(ndim=2, sz=-1, w=(1.0, 1.0, NAN)), PROBE, ""),
]


@pytest.mark.parametrize("case,overrides,rc,msg", CASES, ids=[c[0] for c in CASES])
def test_geodesic_argument_check(edt, case, overrides, rc, msg):
  check_case(edt, edt._lib().edtb200_geodesic, _args, overrides, rc, msg)


def test_the_header_names_the_parameters():
  params = prototypes()["edtb200_geodesic"][1]
  names = [re.sub(r"[*\s]", "", p.rsplit(" ", 1)[1]) for p in params]
  assert names == ["labels", "label_bytes", "seeds", "seed_bytes", "ndim", "sx", "sy", "sz", "count", "wx", "wy", "wz",
                   "flags", "dist_out", "idx_out", "device", "stream"]
  assert "float *dist_out" in params[13] and "int32_t *const *idx_out" in params[14]


def test_the_header_documents_an_addition_at_the_same_version(edt):
  assert edt._lib().edtb200_version() == ABI_VERSION
  assert "edtb200_geodesic" in HEADER[:HEADER.index("#define EDTB200_VERSION")]
  doc = header_doc("edtb200_geodesic")
  for text in ("26-neighbours (2-D: 8, 1-D: 2) with the SAME label", "in the order x, y, z",
               "D[v] = min(D[v], fl64(D[u] + w(u, v)))", "float32(D), rounded once to nearest",
               "least linear seed index c (x-fastest within the volume)", "D[u_{i+1}] == fl64(D[u_i] + w)",
               "-1 in every plane where D is +inf", "ONE cooperative launch of geodesic_relax_kernel",
               "8x8x8 voxels (2-D 16x16, 1-D 256)", "up to 26", "never torn", "no round cap",
               "8 bytes per voxel for D, 8 more for S with idx_out", "12 bytes per tile",
               "Checks, in order: label width, seed width, ndim and sizes", "EDT_B200_VERBOSE",
               "rounds and tile visits"):
    assert text in doc, text


# ---- Python ---------------------------------------------------------------------------------------------

def test_signature(edt):
  p = inspect.signature(edt.geodesic_distance).parameters
  assert list(p) == ["labels", "seeds", "anisotropy", "return_indices", "stacked", "device"]
  assert p["anisotropy"].default is None
  for name, default in (("return_indices", False), ("stacked", False), ("device", 0)):
    assert p[name].kind is inspect.Parameter.KEYWORD_ONLY and p[name].default == default
  assert "geodesic_distance" in edt.__all__


@pytest.mark.parametrize("bad", [1, 0, "yes", None, np.array([True])])
def test_rejects_a_non_bool_return_indices(no_device_use, bad):
  with pytest.raises(TypeError, match="return_indices must be True or False"):
    no_device_use.geodesic_distance(np.ones((4, 5), np.uint8), np.ones((4, 5), bool), return_indices=bad)


@pytest.mark.parametrize("shape,stacked", [((), False), ((2, 2, 2, 2), False), ((4,), True), ((2,) * 5, True)])
def test_rejects_a_wrong_number_of_dimensions(no_device_use, shape, stacked):
  with pytest.raises(TypeError, match="-D to"):
    no_device_use.geodesic_distance(np.ones(shape, np.uint8), np.ones(shape, bool), stacked=stacked)


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.float16, np.complex64, object, "U3"])
def test_rejects_an_unsupported_label_dtype(no_device_use, dtype):
  with pytest.raises(TypeError, match="unsupported label dtype"):
    no_device_use.geodesic_distance(np.zeros((3, 4), dtype), np.zeros((3, 4), bool))


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.complex64, object])
def test_rejects_an_unsupported_seed_dtype(no_device_use, dtype):
  with pytest.raises(TypeError, match="unsupported seed dtype"):
    no_device_use.geodesic_distance(np.zeros((3, 4), np.uint8), np.zeros((3, 4), dtype))


def test_rejects_seeds_of_another_shape(no_device_use):
  with pytest.raises(ValueError, match="seeds must have the labels' shape"):
    no_device_use.geodesic_distance(np.zeros((3, 4), np.uint8), np.zeros((4, 3), bool))
  with pytest.raises(ValueError, match="seeds must have the labels' shape"):
    no_device_use.geodesic_distance(np.zeros((3, 4), np.uint8), np.zeros((3, 4, 1), bool))


@pytest.mark.parametrize("anisotropy", [(1.0, 0.0), (1.0, -2.0), (np.nan, 1.0), (1.0, np.inf)])
def test_rejects_a_bad_weight(no_device_use, anisotropy):
  with pytest.raises(ValueError, match="finite and > 0"):
    no_device_use.geodesic_distance(np.ones((3, 4), np.uint8), np.ones((3, 4), bool), anisotropy)


def test_rejects_a_weight_count_that_does_not_match(no_device_use):
  with pytest.raises(ValueError, match="one entry per volume axis"):
    no_device_use.geodesic_distance(np.ones((3, 4), np.uint8), np.ones((3, 4), bool), (1.0, 2.0, 3.0))


@pytest.mark.parametrize("order", ["C", "F"])
def test_empty_arrays_need_no_device(no_device_use, order):
  for shape, stacked in (((0, 3), False), ((3, 0, 2), False), ((0, 4, 4), True), ((0,), False)):
    labels = np.zeros(shape, np.uint16, order=order)
    seeds = np.zeros(shape, bool, order=order)
    dist = no_device_use.geodesic_distance(labels, seeds, stacked=stacked)
    assert isinstance(dist, np.ndarray) and dist.shape == shape and dist.dtype == np.float32
    dist, idx = no_device_use.geodesic_distance(labels, seeds, stacked=stacked, return_indices=True)
    assert idx.shape == (len(shape) - stacked,) + shape and idx.dtype == np.int32


def test_docstring_states_the_definition(edt):
  doc = " ".join(edt.geodesic_distance.__doc__.split())
  for text in ("26-neighbours (2-D: 8, 1-D: 2) with the same label", "squares summed in double in the order x, y, z",
               "D[v] = min(D[v], fl64(D[u] + w(u, v)))", "scipy.sparse.csgraph.dijkstra(G, indices=seeds, min_only=True)",
               "float32(D), rounded once to nearest", "least linear seed index c (x-fastest within the volume)",
               "D[u_{i+1}] == fl64(D[u_i] + w)", "markers[tuple(idx)]", "np.where(idx[0] >= 0",
               "np.stack of the per-volume calls", "without a host synchronisation", "ENOMEM",
               "float labels are a TypeError", "8 bytes per voxel for D, 8 more with return_indices",
               "-1 in every plane where dist is +inf"):
    assert " ".join(text.split()) in doc, text


def test_the_docstring_examples_hold_on_the_restatement(edt):
  doc = edt.geodesic_distance.__doc__
  assert "[0, 0.5, 1, 1.5, 2, 2.5, 3]" in doc and "np.float32(6 + np.sqrt(2)) = 7.4142137" in doc
  assert "sqrt(32) = 5.656854" in doc
  labels = np.zeros((3, 9), np.uint8)
  labels[1, 1:8] = 1
  seeds = np.zeros((3, 9), bool)
  seeds[1, 1] = True
  dist, _ = gc.restate(labels, seeds, (1.0, 0.5))
  assert dist[1, 1:8].tolist() == [0, 0.5, 1, 1.5, 2, 2.5, 3]
  assert np.isinf(dist[labels == 0]).all()
  labels = np.zeros((5, 5), np.uint8)
  labels[0, :] = 1
  labels[:, 4] = 1
  seeds = np.zeros((5, 5), bool)
  seeds[0, 0] = True
  dist, _ = gc.restate(labels, seeds)
  assert dist[4, 4] == np.float32(6 + np.sqrt(2)) and repr(float(dist[4, 4]))[:9] == "7.4142136"
  assert "%.7f" % dist[4, 4] == "7.4142137" and "%.6f" % np.sqrt(32) == "5.656854"
