"""CPU tests: the argument checks of edtb200_transform_voxel_graph_chunked.

As in test_chunked_arguments.py, every rejection comes with a return code and a message before any
device is touched, and a fully valid call stops at the device probe (abi_checks.expect_probe).  Nothing
here launches a kernel or copies a byte.
"""
import ctypes
import os

import numpy as np
import pytest

from abi_checks import (ABI_VERSION, BIG, ECUDA, EINVAL, ELIMIT, HEADER, LABELS_FLOAT, LABELS_ON_DEVICE, OUT_ON_DEVICE,
                        PROBE, ROOT, SIGNED, SQRT, check_case)

HALF = (1 << 29) + 1                    # fits one axis, but its doubled axis is longer than 2^30

# separate host blocks: the checks only test for NULL and for overlap.  64 voxels: 256 label bytes
# (label_bytes 4), 64 graph bytes, 256 output bytes.
_BLOCKS = [np.zeros(256, np.uint64) for _ in range(3)]
L, G, O = (b.ctypes.data for b in _BLOCKS)


def _call(labels=L, label_bytes=4, graph=G, ndim=3, sx=4, sy=4, sz=4, w=(1.0, 1.0, 1.0), border=0, flags=0, out=O,
          device=63, device_bytes=0, chunks=None):
  return (labels, label_bytes, graph, ndim, sx, sy, sz, *w, border, flags, out, device, device_bytes, chunks)


CASES = [
  ("labels_on_device", dict(flags=LABELS_ON_DEVICE), EINVAL, "HOST buffers"),
  ("out_on_device", dict(flags=OUT_ON_DEVICE), EINVAL, "HOST buffers"),
  ("both_on_device", dict(flags=LABELS_ON_DEVICE | OUT_ON_DEVICE | SQRT), EINVAL, "HOST buffers"),
  ("ndim_1", dict(ndim=1), EINVAL, "2-D or 3-D volume (got ndim 1)"),
  ("ndim_0", dict(ndim=0), EINVAL, "2-D or 3-D volume (got ndim 0)"),
  ("ndim_4", dict(ndim=4), EINVAL, "2-D or 3-D volume (got ndim 4)"),
  ("signed", dict(flags=SIGNED), EINVAL, "EDTB200_SIGNED is not defined with a voxel graph"),
  ("signed_sqrt", dict(flags=SIGNED | SQRT), EINVAL, "EDTB200_SIGNED"),
  ("float_1_byte", dict(flags=LABELS_FLOAT, label_bytes=1), EINVAL, "EDTB200_LABELS_FLOAT needs 4- or 8-byte"),
  ("float_2_bytes", dict(flags=LABELS_FLOAT, label_bytes=2), EINVAL, "EDTB200_LABELS_FLOAT needs 4- or 8-byte"),
  ("label_bytes_3", dict(label_bytes=3), EINVAL, "label_bytes"),
  ("label_bytes_16", dict(label_bytes=16), EINVAL, "label_bytes"),
  ("negative_size", dict(sy=-1), EINVAL, "negative size"),
  ("negative_sx", dict(sx=-4), EINVAL, "negative size"),
  ("axis_too_long", dict(sx=BIG), ELIMIT, "axis longer than 2^30"),
  ("z_too_long", dict(sz=BIG), ELIMIT, "axis longer than 2^30"),
  ("doubled_x_too_long", dict(sx=HALF), ELIMIT, "axis longer than 2^30"),
  ("doubled_y_too_long_2d", dict(ndim=2, sy=HALF), ELIMIT, "axis longer than 2^30"),
  ("doubled_z_too_long", dict(sz=HALF), ELIMIT, "axis longer than 2^30"),
  ("null_labels", dict(labels=None), EINVAL, "null pointer"),
  ("null_graph", dict(graph=None), EINVAL, "null pointer"),
  ("null_out", dict(out=None), EINVAL, "null pointer"),
  ("same_buffer", dict(out=L), EINVAL, "labels and out overlap"),
  ("out_inside_labels", dict(out=L + 128), EINVAL, "labels and out overlap"),
  ("labels_inside_out", dict(labels=O + 252), EINVAL, "labels and out overlap"),
  ("wide_labels_reach_out", dict(label_bytes=8, out=L + 511), EINVAL, "labels and out overlap"),
  ("graph_is_out", dict(graph=O), EINVAL, "graph and out overlap"),
  ("graph_reaches_out", dict(graph=O - 63), EINVAL, "graph and out overlap"),
  ("out_reaches_graph", dict(out=G - 255), EINVAL, "graph and out overlap"),
  # order: residency, dimensionality, sign, float labels, label width and sizes, emptiness, pointers,
  # doubled axes, overlap
  ("flags_before_ndim", dict(flags=OUT_ON_DEVICE, ndim=1), EINVAL, "HOST buffers"),
  ("ndim_before_signed", dict(ndim=1, flags=SIGNED), EINVAL, "2-D or 3-D"),
  ("signed_before_float", dict(flags=SIGNED | LABELS_FLOAT, label_bytes=1), EINVAL, "EDTB200_SIGNED"),
  ("float_before_label_bytes", dict(flags=LABELS_FLOAT, label_bytes=3), EINVAL, "EDTB200_LABELS_FLOAT"),
  ("label_bytes_before_size", dict(label_bytes=3, sy=-1), EINVAL, "label_bytes"),
  ("size_before_null", dict(sx=BIG, labels=None), ELIMIT, "axis longer than 2^30"),
  ("empty_before_null", dict(sz=0, labels=None, graph=None, out=None), 0, ""),
  ("empty_2d", dict(ndim=2, sx=0, sz=-1), 0, ""),
  ("null_before_doubled", dict(sx=HALF, graph=None), EINVAL, "null pointer"),
  ("doubled_before_overlap", dict(sx=HALF, out=L), ELIMIT, "axis longer than 2^30"),
  ("labels_before_graph_overlap", dict(out=L, graph=L), EINVAL, "labels and out overlap"),
  # adjacent buffers do not overlap; the two inputs may overlap; 2-D ignores sz
  ("valid_adjacent", dict(out=L + 256, graph=L + 512), PROBE, ""),
  ("valid_adjacent_below", dict(labels=O + 256, graph=O - 64), PROBE, ""),
  ("valid_inputs_overlap", dict(graph=L), PROBE, ""),
  ("valid_2d_ignores_sz", dict(ndim=2, sz=-1), PROBE, ""),
  ("valid_float", dict(flags=LABELS_FLOAT | SQRT, label_bytes=8), PROBE, ""),
  ("valid_budget", dict(device_bytes=1 << 20, flags=SQRT, border=1), PROBE, ""),
  ("valid", dict(), PROBE, ""),
]


@pytest.mark.parametrize("case,overrides,rc,msg", CASES, ids=[c[0] for c in CASES])
def test_voxel_graph_chunked_argument_check(edt, case, overrides, rc, msg):
  chunks = []

  def build(**kw):
    chunks.append((ctypes.c_int64 * 2)(-7, -7))
    return _call(**kw, chunks=chunks[-1])
  check_case(edt, edt._lib().edtb200_transform_voxel_graph_chunked, build, overrides, rc, msg)
  assert all(list(c) == [0, 0] for c in chunks)          # each call cleared its chunks before any check


def test_voxel_graph_chunked_is_an_addition_at_the_same_version(edt):
  lib = edt._lib()
  assert lib.edtb200_version() == ABI_VERSION
  assert hasattr(lib, "edtb200_transform_voxel_graph_chunked") and hasattr(lib, "edtb200_transform_voxel_graph")


def test_voxel_graph_chunked_is_declared():
  assert "int edtb200_transform_voxel_graph_chunked(" in HEADER
  shim = open(os.path.join(ROOT, "include", "edt_voxel_graph.hpp")).read()
  assert "edtb200_transform_voxel_graph_chunked(" in shim


def test_python_keeps_rejecting_a_budget_with_a_graph(edt):
  with pytest.raises(ValueError, match="voxel_graph"):
    edt.edtsq(np.ones((4, 4, 4), np.uint8), voxel_graph=np.full((4, 4, 4), 63, np.uint8), max_device_bytes=0)


def test_graph_call_reaches_the_library_without_a_device(edt):
  """Without a GPU the one-shot graph call fails at the device probe with ECUDA, which is not retried."""
  if edt.device_count() > 0:
    pytest.skip("a GPU is visible")
  with pytest.raises(edt.EDTError) as info:
    edt.edt(np.ones((4, 4, 4), np.uint8), voxel_graph=np.full((4, 4, 4), 63, np.uint8))
  assert info.value.code == ECUDA
