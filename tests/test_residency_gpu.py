"""GPU tests: the residency contract of the three C-ABI transforms that accept host buffers.

edtb200_transform, edtb200_feature_transform and edtb200_transform_voxel_graph take their inputs
and outputs in host or device memory (EDTB200_LABELS_ON_DEVICE / EDTB200_OUT_ON_DEVICE), on the
NULL stream or a caller's stream.  Every combination must compute what the device-resident call
computes, bit for bit, and a call that touches host memory must be complete on return: its host
outputs are read here without any synchronise.  Two sizes: one copied directly (under 4 MiB), one
staged from pageable memory through the pinned chunk buffers in more than one 32 MiB chunk; the
larger size also runs once from pinned host memory.
"""
import ctypes

import numpy as np
import pytest

LABELS_ON_DEVICE, OUT_ON_DEVICE, SQRT = 4, 8, 1

SMALL = (40, 36, 28)               # 161 KB of float32: direct copies
LARGE = (256, 256, 160)            # 40 MiB of uint32 labels and of float32 distances: two chunks
RESIDENCY = [(False, False), (True, False), (False, True), (True, True)]
RES_IDS = ["host-host", "device-host", "host-device", "device-device"]


def _labels(shape, seed, high=4):
  """x-fastest uint32 labels in runs of 8 along x, so that the distances are not all tiny."""
  n = int(np.prod(shape))
  rng = np.random.default_rng(seed)
  return np.ascontiguousarray(np.repeat(rng.integers(0, high, n // 8 + 1, dtype=np.uint32), 8)[:n])


def _dims(shape):
  return tuple(shape) + (1,) * (3 - len(shape))


class Call:
  """Buffers of one C-ABI call, placed on the host (pageable or pinned) or on the device."""

  def __init__(self, torch, stream):
    self.torch = torch
    self.stream = stream
    self.keep = []

  def put(self, array, on_device, pinned=False):
    torch = self.torch
    if array.dtype == np.uint32:
      array = array.view(np.int32)                                 # the same bytes, a type torch copies
    if on_device:
      t = torch.from_numpy(array).cuda()
      self.keep.append(t)
      return t.data_ptr()
    if pinned:
      t = torch.from_numpy(array).pin_memory()
      self.keep.append(t)
      return t.data_ptr()
    self.keep.append(array)
    return array.ctypes.data

  def empty(self, n, dtype, on_device, pinned=False):
    """An output buffer with every bit set (no distance, and no index with black_border), and its reader."""
    torch = self.torch
    host = np.full(n, -1, np.int32).view(dtype)
    if on_device:
      t = torch.from_numpy(host).cuda()
      self.keep.append(t)
      return t.data_ptr(), lambda: t.cpu().numpy()
    if pinned:
      t = torch.from_numpy(host).pin_memory()
      self.keep.append(t)
      return t.data_ptr(), lambda: t.numpy()
    self.keep.append(host)
    return host.ctypes.data, lambda: host

  def run(self, fn, *args):
    """Calls fn on device 0 and this call's stream, which first waits for the work that made the
    device inputs."""
    torch = self.torch
    if self.stream is not None:
      self.stream.wait_stream(torch.cuda.current_stream())        # the device inputs are ready
      handle = ctypes.c_void_p(self.stream.cuda_stream)
    else:
      handle = None
    return fn(*args, 0, handle)


def _finish(torch, call, lab_dev, out_dev):
  if lab_dev and out_dev:
    (call.stream or torch.cuda.current_stream()).synchronize()


def _same_bits(a, b):
  return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.fixture(scope="module")
def torch_cuda():
  torch = pytest.importorskip("torch")
  if not torch.cuda.is_available():
    pytest.skip("no CUDA device")
  return torch


def _stream(torch, kind):
  return torch.cuda.Stream() if kind == "side" else None


# ---- edtb200_transform -----------------------------------------------------------------------

def _transform(edt, torch, shape, lab_dev, out_dev, stream_kind, pinned=False):
  lib = edt._lib()
  sx, sy, sz = _dims(shape)
  labels = _labels(shape, 1)
  call = Call(torch, _stream(torch, stream_kind))
  lab = call.put(labels, lab_dev, pinned)
  out, read = call.empty(labels.size, np.float32, out_dev, pinned)
  flags = (LABELS_ON_DEVICE if lab_dev else 0) | (OUT_ON_DEVICE if out_dev else 0)
  rc = call.run(lib.edtb200_transform, lab, 4, len(shape), sx, sy, sz, 1.0, 1.5, 2.0, 0, flags, out)
  assert rc == 0, lib.edtb200_last_error()
  _finish(torch, call, lab_dev, out_dev)
  return read().copy()


_REF = {}


def _reference(key, compute):
  if key not in _REF:
    _REF[key] = compute()
  return _REF[key]


@pytest.mark.gpu
@pytest.mark.parametrize("stream_kind", ["null", "side"])
@pytest.mark.parametrize("lab_dev,out_dev", RESIDENCY, ids=RES_IDS)
@pytest.mark.parametrize("shape", [SMALL, LARGE], ids=["small", "large"])
def test_transform_residency(edt, torch_cuda, shape, lab_dev, out_dev, stream_kind):
  want = _reference(("transform", shape), lambda: _transform(edt, torch_cuda, shape, True, True, "null"))
  got = _transform(edt, torch_cuda, shape, lab_dev, out_dev, stream_kind)
  assert _same_bits(got, want)


# ---- edtb200_feature_transform ---------------------------------------------------------------

FEATURE_SHAPES = {"1d": (5000,), "2d": (120, 90), "3d": SMALL, "3d-large": LARGE}


def _feature(edt, torch, shape, lab_dev, out_dev, stream_kind, with_dist, pinned=False):
  lib = edt._lib()
  sx, sy, sz = _dims(shape)
  nd = len(shape)
  labels = _labels(shape, 2)
  call = Call(torch, _stream(torch, stream_kind))
  lab = call.put(labels, lab_dev, pinned)
  dist, read_dist = call.empty(labels.size, np.float32, out_dev, pinned) if with_dist else (None, None)
  planes = [call.empty(labels.size, np.int32, out_dev, pinned) for _ in range(nd)]
  idx = (ctypes.c_void_p * 3)(*([p for p, _ in planes] + [None] * (3 - nd)))
  flags = (LABELS_ON_DEVICE if lab_dev else 0) | (OUT_ON_DEVICE if out_dev else 0)
  rc = call.run(lib.edtb200_feature_transform, lab, 4, nd, sx, sy, sz, 1.0, 2.0, 1.5, 1, flags, dist, idx)
  assert rc == 0, lib.edtb200_last_error()
  _finish(torch, call, lab_dev, out_dev)
  got = [read().copy() for _, read in planes]
  return (read_dist().copy() if with_dist else None), got


@pytest.mark.gpu
@pytest.mark.parametrize("with_dist", [False, True], ids=["no-dist", "dist"])
@pytest.mark.parametrize("stream_kind", ["null", "side"])
@pytest.mark.parametrize("lab_dev,out_dev", RESIDENCY, ids=RES_IDS)
@pytest.mark.parametrize("shape_id", sorted(FEATURE_SHAPES))
def test_feature_transform_residency(edt, torch_cuda, shape_id, lab_dev, out_dev, stream_kind, with_dist):
  shape = FEATURE_SHAPES[shape_id]
  want_dist, want_idx = _reference(("feature", shape),
                                   lambda: _feature(edt, torch_cuda, shape, True, True, "null", True))
  dist, idx = _feature(edt, torch_cuda, shape, lab_dev, out_dev, stream_kind, with_dist)
  assert len(idx) == len(want_idx) and all(_same_bits(a, b) for a, b in zip(idx, want_idx))
  if with_dist:
    assert _same_bits(dist, want_dist)


# ---- edtb200_transform_voxel_graph -----------------------------------------------------------

def _voxel_graph(edt, torch, shape, lab_dev, out_dev, stream_kind, pinned=False):
  lib = edt._lib()
  sx, sy, sz = _dims(shape)
  labels = _labels(shape, 3, high=3)
  graph = np.random.default_rng(4).integers(0, 64, labels.size, dtype=np.uint8)
  call = Call(torch, _stream(torch, stream_kind))
  lab = call.put(labels, lab_dev, pinned)
  gr = call.put(graph, lab_dev, pinned)
  out, read = call.empty(labels.size, np.float32, out_dev, pinned)
  flags = SQRT | (LABELS_ON_DEVICE if lab_dev else 0) | (OUT_ON_DEVICE if out_dev else 0)
  rc = call.run(lib.edtb200_transform_voxel_graph, lab, 4, gr, len(shape), sx, sy, sz, 1.0, 1.0, 2.0, 1, flags, out)
  assert rc == 0, lib.edtb200_last_error()
  _finish(torch, call, lab_dev, out_dev)
  return read().copy()


@pytest.mark.gpu
@pytest.mark.parametrize("stream_kind", ["null", "side"])
@pytest.mark.parametrize("lab_dev,out_dev", RESIDENCY, ids=RES_IDS)
@pytest.mark.parametrize("shape", [SMALL, LARGE], ids=["small", "large"])
def test_voxel_graph_residency(edt, torch_cuda, shape, lab_dev, out_dev, stream_kind):
  want = _reference(("voxel_graph", shape), lambda: _voxel_graph(edt, torch_cuda, shape, True, True, "null"))
  got = _voxel_graph(edt, torch_cuda, shape, lab_dev, out_dev, stream_kind)
  assert _same_bits(got, want)


# ---- pinned host memory, copied directly whatever its size ------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["transform", "feature", "voxel_graph"])
def test_pinned_host_buffers(edt, torch_cuda, kind):
  if kind == "transform":
    want = _reference(("transform", LARGE), lambda: _transform(edt, torch_cuda, LARGE, True, True, "null"))
    assert _same_bits(_transform(edt, torch_cuda, LARGE, False, False, "null", pinned=True), want)
  elif kind == "feature":
    want_dist, want_idx = _reference(("feature", LARGE),
                                     lambda: _feature(edt, torch_cuda, LARGE, True, True, "null", True))
    dist, idx = _feature(edt, torch_cuda, LARGE, False, False, "null", True, pinned=True)
    assert _same_bits(dist, want_dist) and all(_same_bits(a, b) for a, b in zip(idx, want_idx))
  else:
    want = _reference(("voxel_graph", LARGE), lambda: _voxel_graph(edt, torch_cuda, LARGE, True, True, "null"))
    assert _same_bits(_voxel_graph(edt, torch_cuda, LARGE, False, False, "null", pinned=True), want)
