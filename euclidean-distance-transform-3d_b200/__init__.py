"""H100-native multi-label anisotropic Euclidean distance transform.

Host-side mirror of the reference's Python API (seung-lab/euclidean-distance-transform-3d,
``src/edt.pyx``): same function names, positional/keyword arguments, dtype handling, C/F
order handling and error behaviour, so that ``import edt_b200 as edt`` is a drop-in for
``import edt`` on the distance-transform path.  All arithmetic happens in hand-written
sm_90a CUDA kernels reached through the C ABI of ``include/edt_b200.h`` (ctypes); there is
no CPU implementation in this package -- if ``libedt_b200.so`` is missing or no CUDA device
is usable the calls raise.

Reference entry points mirrored here (file:line in the reference):
  edt      src/edt.pyx:205-242      edtsq    src/edt.pyx:245-310
  sdf      src/edt.pyx:121-158      sdfsq    src/edt.pyx:161-202
  edt1d/edt1dsq  src/edt.pyx:312-399   edt2d/edt2dsq  src/edt.pyx:401-512
  edt3d/edt3dsq  src/edt.pyx:622-734

Differences, all additive: ``parallel`` is accepted and ignored (the CUDA grid replaces the
thread pool); keyword-only ``device=`` selects the GPU; ``sdf``/``sdfsq`` run ONE fused
transform (background treated as a label, sign applied in the last store) instead of two;
``voxel_graph=`` (2-D / 3-D, src/edt.pyx:514-620, 736-844) draws the doubled grid and runs
the transform on the device.
``edt_cuda`` transforms a torch CUDA tensor without touching host memory, and every function
above accepts device-resident input directly (a torch CUDA tensor or any object exposing
``__cuda_array_interface__``) and then returns a torch CUDA tensor.
"""
import collections
import ctypes
import math
import os

import numpy as np

__version__ = "0.1.0"
__all__ = [
  "edt", "edtsq", "sdf", "sdfsq",
  "edt1d", "edt1dsq", "edt2d", "edt2dsq", "edt3d", "edt3dsq",
  "edt_cuda", "transform_batch", "each", "each_cuda", "label_stats_cuda", "device_count", "library_path", "EDTError",
  "feature_transform", "expand_labels",
  "surface_distances", "SurfaceDistances", "hausdorff_distance", "average_surface_distance", "surface_dice",
  "spherical_erode", "spherical_dilate", "spherical_open", "spherical_close",
  "parabolic_erode", "parabolic_dilate", "nearest_labels", "medial_axis",
  "skeletonize", "local_thickness", "geodesic_distance", "watershed",
  "connected_components", "extended_maxima", "fill_holes", "dust",
]

FLAG_SQRT = 1
FLAG_SIGNED = 2
FLAG_LABELS_ON_DEVICE = 4
FLAG_OUT_ON_DEVICE = 8
FLAG_LABELS_FLOAT = 16

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


_TOO_MANY_DIMS = "Multi-Label EDT library only supports up to 3 dimensions got {}."
_GRAPH_DIMS = "Voxel connectivity graph is only supported for 2D and 3D. Got {}."

ECUDA = -2                # EDTB200_ECUDA
ENOMEM = -3               # EDTB200_ENOMEM


class EDTError(RuntimeError):
  """A C-ABI call failed (CUDA error, no device, unsupported size...).  `code` is the call's
  EDTB200_E* return code (None where the error did not come from one)."""

  def __init__(self, message, code=None):
    super().__init__(message)
    self.code = code


def library_path():
  """The CUDA library built in-tree by __graft_entry__.build().  EDTB200_LIBRARY overrides the
  path (A/B measurements of two builds on the same box); it is still this library, never a
  CPU substitute."""
  return os.environ.get("EDTB200_LIBRARY") or os.path.join(_HERE, "libedt_b200.so")


def _lib():
  """Load libedt_b200.so (built in-tree by __graft_entry__.build()); fail loudly if absent."""
  global _LIB
  if _LIB is not None:
    return _LIB
  path = library_path()
  if not os.path.exists(path):
    raise ImportError(
      "edt_b200: %s is missing -- build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
      "There is no CPU fallback." % path)
  lib = ctypes.CDLL(path)
  i64, f32, vp, ci = ctypes.c_int64, ctypes.c_float, ctypes.c_void_p, ctypes.c_int
  lib.edtb200_version.restype = ci
  lib.edtb200_last_error.restype = ctypes.c_char_p
  lib.edtb200_device_count.restype = ci
  lib.edtb200_transform.argtypes = [vp, ci, ci, i64, i64, i64, f32, f32, f32, ci, ci, vp, ci, vp]
  lib.edtb200_transform.restype = ci
  lib.edtb200_transform_chunked.argtypes = [vp, ci, ci, i64, i64, i64, f32, f32, f32, ci, ci, vp, ci,
                                            ctypes.c_size_t, vp]
  lib.edtb200_transform_chunked.restype = ci
  lib.edtb200_feature_transform.argtypes = [vp, ci, ci, i64, i64, i64, f32, f32, f32, ci, ci, vp, vp, ci, vp]
  lib.edtb200_feature_transform.restype = ci
  lib.edtb200_feature_transform_chunked.argtypes = [vp, ci, ci, i64, i64, i64, f32, f32, f32, ci, ci, vp, vp, ci,
                                                    ctypes.c_size_t, vp]
  lib.edtb200_feature_transform_chunked.restype = ci
  lib.edtb200_transform_stack.argtypes = [vp, ci, ci, i64, i64, i64, i64, f32, f32, f32, ci, ci, vp, ci,
                                          ctypes.c_size_t, vp, vp]
  lib.edtb200_transform_stack.restype = ci
  lib.edtb200_feature_transform_stack.argtypes = [vp, ci, ci, i64, i64, i64, i64, f32, f32, f32, ci, ci, vp, vp, ci,
                                                  vp]
  lib.edtb200_feature_transform_stack.restype = ci
  lib.edtb200_transform_bounded.argtypes = [vp, ci, ci, i64, i64, i64, f32, f32, f32, ci, ci, vp, ci, vp,
                                            ctypes.c_double]
  lib.edtb200_transform_bounded.restype = ci
  lib.edtb200_feature_transform_bounded.argtypes = [vp, ci, ci, i64, i64, i64, f32, f32, f32, ci, ci, vp, vp, ci, vp,
                                                    ctypes.c_double]
  lib.edtb200_feature_transform_bounded.restype = ci
  lib.edtb200_bounded_plan.argtypes = [ci, i64, i64, i64, f32, f32, f32, ctypes.c_double, vp, vp]
  lib.edtb200_bounded_plan.restype = ci
  lib.edtb200_morphology.argtypes = [vp, ci, ci, i64, i64, i64, i64, f32, f32, f32, ci, ctypes.c_double, ci, ci, vp,
                                     ci, vp]
  lib.edtb200_morphology.restype = ci
  lib.edtb200_local_thickness.argtypes = [vp, ci, ci, i64, i64, i64, i64, f32, f32, f32, ci, ci, vp, ci, vp, vp, ci,
                                          vp]
  lib.edtb200_local_thickness.restype = ci
  lib.edtb200_parabolic.argtypes = [vp, ci, i64, i64, i64, i64, f32, f32, f32, ci, ci, vp, ci, vp]
  lib.edtb200_parabolic.restype = ci
  lib.edtb200_parabolic_sites.argtypes = [vp, ci, i64, i64, i64, i64, f32, f32, f32, ci, ci, vp, vp, ci, vp]
  lib.edtb200_parabolic_sites.restype = ci
  lib.edtb200_nearest_labels.argtypes = [vp, ci, ci, i64, i64, i64, i64, f32, f32, f32, ctypes.c_double, ci, ci, vp,
                                         vp, ci, vp]
  lib.edtb200_nearest_labels.restype = ci
  lib.edtb200_nearest_labels_plan.argtypes = [ci, i64, i64, i64, f32, f32, f32, ctypes.c_double, ci, ci, vp, vp]
  lib.edtb200_nearest_labels_plan.restype = ci
  lib.edtb200_medial_axis.argtypes = [vp, ci, ci, i64, i64, i64, i64, f32, f32, f32, ci, ci, vp, vp, ci, vp]
  lib.edtb200_medial_axis.restype = ci
  lib.edtb200_skeletonize.argtypes = [vp, ci, ci, i64, i64, i64, i64, f32, f32, f32, ci, ci, vp, vp, ci, vp]
  lib.edtb200_skeletonize.restype = ci
  lib.edtb200_geodesic.argtypes = [vp, ci, vp, ci, ci, i64, i64, i64, i64, f32, f32, f32, ci, vp, vp, ci, vp]
  lib.edtb200_geodesic.restype = ci
  lib.edtb200_watershed.argtypes = [vp, ci, vp, ci, vp, ci, i64, i64, i64, i64, ci, ci, vp, vp, ci, vp]
  lib.edtb200_watershed.restype = ci
  lib.edtb200_connected_components.argtypes = [vp, ci, ci, i64, i64, i64, i64, ci, ci, vp, ci, ci, vp]
  lib.edtb200_connected_components.restype = ci
  lib.edtb200_extended_maxima.argtypes = [vp, ci, vp, ci, i64, i64, i64, i64, ctypes.c_double, ci, ci, vp, ci, ci, vp]
  lib.edtb200_extended_maxima.restype = ci
  lib.edtb200_fill_holes.argtypes = [vp, ci, ci, i64, i64, i64, i64, ci, i64, ci, vp, vp, ci, vp]
  lib.edtb200_fill_holes.restype = ci
  lib.edtb200_dust.argtypes = [vp, ci, ci, i64, i64, i64, i64, ci, i64, ci, ci, vp, ci, vp]
  lib.edtb200_dust.restype = ci
  lib.edtb200_expand_gather.argtypes = [vp, ci, ci, i64, i64, i64, i64, vp, vp, ctypes.c_double, ci, vp, ci, vp]
  lib.edtb200_expand_gather.restype = ci
  lib.edtb200_surface_count.argtypes = [vp, vp, ci, ci, i64, i64, i64, i64, vp, i64, ci, vp, ci, vp]
  lib.edtb200_surface_count.restype = ci
  lib.edtb200_surface_distances.argtypes = [vp, vp, ci, ci, i64, i64, i64, i64, f32, f32, f32, vp, i64, ci, vp, vp,
                                            ci, ctypes.c_size_t, vp, vp]
  lib.edtb200_surface_distances.restype = ci
  lib.edtb200_transform_multi.argtypes = [vp, ci, ci, i64, i64, i64, f32, f32, f32, ci, ci, vp, vp, ci]
  lib.edtb200_transform_multi.restype = ci
  lib.edtb200_transform_batch.argtypes = [vp, vp, ci, ci, ci, i64, i64, i64, f32, f32, f32, ci, ci, ci]
  lib.edtb200_transform_batch.restype = ci
  lib.edtb200_transform_voxel_graph.argtypes = [vp, ci, vp, ci, i64, i64, i64, f32, f32, f32, ci, ci, vp, ci, vp]
  lib.edtb200_transform_voxel_graph.restype = ci
  lib.edtb200_transform_voxel_graph_chunked.argtypes = [vp, ci, vp, ci, i64, i64, i64, f32, f32, f32, ci, ci, vp, ci,
                                                        ctypes.c_size_t, vp]
  lib.edtb200_transform_voxel_graph_chunked.restype = ci
  lib.edtb200_pass_first.argtypes = [vp, ci, i64, i64, i64, f32, ci, ci, vp, ci, vp]
  lib.edtb200_pass_first.restype = ci
  lib.edtb200_pass_later.argtypes = [vp, ci, ci, i64, i64, i64, f32, ci, ci, ci, vp, ci, vp]
  lib.edtb200_pass_later.restype = ci
  lib.edtb200_pass_window.argtypes = [vp, ci, ci, i64, i64, i64, f32, ci, ci, ci, ctypes.c_double, vp, vp, vp, ci,
                                      vp]
  lib.edtb200_pass_window.restype = ci
  lib.edtb200_noise_planes.argtypes = [vp, ci, ci, i64, i64, i64, i64, f32, f32, f32, ci, ci, ci, ci, ci, vp, vp, vp,
                                       ci, vp]
  lib.edtb200_noise_planes.restype = ci
  lib.edtb200_slab_pack.argtypes = [vp, vp, i64, i64, i64, ci, ctypes.POINTER(ctypes.c_int64), ci, ci, vp]
  lib.edtb200_slab_pack.restype = ci
  lib.edtb200_slab_face_runs.argtypes = [vp, ci, i64, i64, i64, ci, ci, ci, vp, vp, ci, vp]
  lib.edtb200_slab_face_runs.restype = ci
  lib.edtb200_slab_face_fixup.argtypes = [vp, ci, i64, i64, i64, ci, ci, f32, ci, vp, vp, vp, vp, vp, ci, vp]
  lib.edtb200_slab_face_fixup.restype = ci
  lib.edtb200_profile_passes.argtypes = [ci]
  lib.edtb200_profile_passes.restype = ci
  lib.edtb200_pass_ms.argtypes = [ci, vp]
  lib.edtb200_pass_ms.restype = ci
  lib.edtb200_last_later_launch.argtypes = [vp]
  lib.edtb200_last_later_launch.restype = ci
  lib.edtb200_slab_stage_bytes.argtypes = [i64, i64, ci, ci]
  lib.edtb200_slab_stage_bytes.restype = i64
  lib.edtb200_slab_step.argtypes = [vp, ci, i64, i64, i64, f32, f32, f32, ci, ci, ci, ci, vp, ci, vp, vp, vp,
                                    ctypes.c_uint64, vp, ci, vp]
  lib.edtb200_slab_step.restype = ci
  lib.edtb200_label_stats.argtypes = [vp, ci, vp, i64, i64, i64, ci, vp, vp, vp, vp, vp, vp, ci, vp]
  lib.edtb200_label_stats.restype = ci
  lib.edtb200_label_extract.argtypes = [vp, ci, vp, i64, i64, i64, ctypes.c_uint64, vp, ci, vp, ci, vp]
  lib.edtb200_label_extract.restype = ci
  lib.edtb200_host_alloc.argtypes = [ctypes.c_size_t]
  lib.edtb200_host_alloc.restype = vp
  lib.edtb200_host_free.argtypes = [vp]
  lib.edtb200_host_free.restype = None
  lib.edtb200_release.restype = ci
  _LIB = lib
  return lib


def _check(rc):
  if rc != 0:
    msg = _lib().edtb200_last_error()
    raise EDTError("edt_b200 error %d: %s" % (rc, msg.decode("utf-8", "replace") if msg else "?"), rc)


def device_count():
  return int(_lib().edtb200_device_count())


LATER_LAUNCH_FIELDS = ("kernel", "tx", "tma", "wide", "ctas", "int_hull", "epilogue", "all_double")


def last_later_launch():
  """Kernel variant of the last Y / Z pass this thread launched (edtb200_last_later_launch), as a
  dict: kernel "tile", "long" or "window" (a bounded transform's window kernel, whose radius is in
  tx), tile width tx, tma, wide, ctas (per SM), int_hull, epilogue, all_double (every candidate
  formed in double), settled (tiles the X pass left settled were skipped)."""
  # the plan fields (LATER_LAUNCH_FIELDS), then whether settled tiles were skipped
  info = (ctypes.c_int * (len(LATER_LAUNCH_FIELDS) + 1))()
  _check(_lib().edtb200_last_later_launch(info))
  out = dict(zip(LATER_LAUNCH_FIELDS + ("settled",), (int(v) for v in info)))
  out["kernel"] = {0: "tile", 1: "long", 2: "window"}[out["kernel"]]
  return out


def _bound(max_distance, voxel_graph=None, devices=None, stacked=False, max_device_bytes=None):
  """max_distance as a float (None: unbounded), after rejecting a bad value and what the bounded
  transforms do not cover."""
  if max_distance is None:
    return None
  d = float(max_distance)
  if not d >= 0.0:
    raise ValueError("max_distance must be zero or more, got %r" % (max_distance,))
  for given, name in ((voxel_graph is not None, "voxel_graph"), (devices is not None, "devices=[...]"),
                      (stacked, "stacked=True"), (max_device_bytes is not None, "max_device_bytes")):
    if given:
      raise ValueError("max_distance cannot be combined with %s" % name)
  return None if d == float("inf") else d


def nvl(val, default_val):
  return default_val if val is None else val


# ---------------------------------------------------------------------------------------
# host-side logic mirrored from the reference's Cython layer
# ---------------------------------------------------------------------------------------

def _label_view(data):
  """Labels as raw unsigned integers (src/edt.pyx:670-732): signed ints are reinterpreted,
  bool is one byte, floats are compared by value (so -0.0 is folded onto +0.0 first).
  Returns None for dtypes the reference does not dispatch on (it then returns zeros)."""
  dt = data.dtype
  if dt == np.bool_:
    return data.view(np.uint8)
  if dt.kind in "iu" and dt.itemsize in (1, 2, 4, 8):
    return data.view(np.dtype("u%d" % dt.itemsize))
  if dt == np.float32:
    return (data + np.float32(0)).view(np.uint32)
  if dt == np.float64:
    return (data + np.float64(0)).view(np.uint64)
  return None


def _x_fastest(shape, anisotropy, f_contiguous):
  """(sx, sy, sz), (wx, wy, wz) for an array of `shape`: Fortran order keeps the axes,
  C order reverses them (src/edt.pyx:429-440, 651-664)."""
  dims = [int(s) for s in shape]
  weights = [float(a) for a in anisotropy]
  if len(weights) != len(dims):
    raise ValueError("anisotropy must have one entry per dimension")
  if not f_contiguous:
    dims.reverse()
    weights.reverse()
  while len(dims) < 3:
    dims.append(1)
    weights.append(1.0)
  return dims, weights


# ---------------------------------------------------------------------------------------
# result arrays backed by recycled page-locked memory
# ---------------------------------------------------------------------------------------
# A fresh 512 MiB numpy array costs ~130 000 page faults while the result is copied into it, and
# pageable memory has to be staged through pinned buffers on the way back from the GPU.  Large
# results are therefore placed in page-locked blocks (edtb200_host_alloc) that return to a small
# pool when the array that wraps them is garbage collected: from the second call of a loop on, the
# download is ONE direct DMA into memory that is already mapped.  The pool holds at most
# EDTB200_PINNED_POOL_MB (default 2048) of idle blocks and hands out at most twice that in total;
# beyond it, and for arrays below 4 MiB, plain numpy memory is used.  EDTB200_PINNED_POOL_MB=0
# turns the pool off.

import threading as _threading
import weakref as _weakref

_POOL_LOCK = _threading.Lock()
_POOL_FREE = {}            # nbytes -> [ptr, ...]
_POOL_IDLE = 0             # bytes sitting in _POOL_FREE
_POOL_OUT = 0              # bytes currently behind live arrays
_POOL_MIN = 4 << 20


def _pool_cap():
  try:
    return int(os.environ.get("EDTB200_PINNED_POOL_MB", "2048")) << 20
  except ValueError:
    return 2048 << 20


def _pool_release(ptr, nbytes):
  global _POOL_IDLE, _POOL_OUT
  with _POOL_LOCK:
    _POOL_OUT -= nbytes
    if _POOL_IDLE + nbytes <= _pool_cap():
      _POOL_FREE.setdefault(nbytes, []).append(ptr)
      _POOL_IDLE += nbytes
      return
  try:
    _lib().edtb200_host_free(ctypes.c_void_p(ptr))
  except Exception:        # interpreter shutdown
    pass


def _result_buffer(count):
  """float32[count] for a result: page-locked and recycled when the pool allows, else np.empty."""
  global _POOL_IDLE, _POOL_OUT
  nbytes = int(count) * 4
  cap = _pool_cap()
  if nbytes < _POOL_MIN or cap <= 0:
    return np.empty(count, dtype=np.float32)
  ptr = None
  with _POOL_LOCK:
    free = _POOL_FREE.get(nbytes)
    if free:
      ptr = free.pop()
      _POOL_IDLE -= nbytes
      _POOL_OUT += nbytes
    elif _POOL_OUT + nbytes > 2 * cap:
      return np.empty(count, dtype=np.float32)
  if ptr is None:
    lib = _lib()
    if _POOL_IDLE:                              # make room: drop idle blocks of other sizes
      with _POOL_LOCK:
        for size in list(_POOL_FREE):
          while _POOL_FREE[size] and _POOL_IDLE + nbytes > cap:
            lib.edtb200_host_free(ctypes.c_void_p(_POOL_FREE[size].pop()))
            _POOL_IDLE -= size
    ptr = lib.edtb200_host_alloc(ctypes.c_size_t(nbytes))
    if not ptr:
      return np.empty(count, dtype=np.float32)
    with _POOL_LOCK:
      _POOL_OUT += nbytes
  block = (ctypes.c_char * nbytes).from_address(ptr)
  _weakref.finalize(block, _pool_release, ptr, nbytes)
  return np.frombuffer(block, dtype=np.float32, count=count)


def _graph_bytes(voxel_graph, order):
  """The graph as uint8 in the data's memory order (src/edt.pyx:294-298, 527-530)."""
  g = np.asarray(voxel_graph)
  g = np.ascontiguousarray(g) if order == "C" else np.asfortranarray(g)
  return g.view(np.uint8) if g.dtype in (np.uint8, np.int8) else g.astype(np.uint8)


def _device_array(data):
  """torch CUDA tensor view of `data` if it already lives on a GPU (a torch CUDA tensor, or any
  object exposing `__cuda_array_interface__`: CuPy, Numba, ...), else None.  Zero-copy."""
  if isinstance(data, (np.ndarray, list, tuple)) or np.isscalar(data):
    return None
  mod = type(data).__module__
  if mod.startswith("torch"):
    return data if getattr(data, "is_cuda", False) else None
  if hasattr(data, "__cuda_array_interface__"):
    import torch
    t = torch.as_tensor(data, device="cuda")
    # interface v3: "stream" names the stream the producer's work was queued on (1 = legacy
    # default, 2 = per-thread default, else a cudaStream_t); order torch's current stream after it
    stream = data.__cuda_array_interface__.get("stream")
    if stream is not None and stream != 0:
      cur = torch.cuda.current_stream(t.device)
      if stream in (1, 2):
        torch.cuda.synchronize(t.device)
      elif int(stream) != cur.cuda_stream:
        ev = torch.cuda.Event()
        ev.record(torch.cuda.ExternalStream(int(stream), device=t.device))
        cur.wait_event(ev)
    return t
  return None


def _weights(n, anisotropy, rule="volume"):
  """One float weight for each of `n` axes; None gives 1.0 each.  How a scalar and a sequence count is the
  caller's `rule`:
    "volume"  stacks and the whole-volume operations: a scalar for one axis, else the entries of any shape;
    "first"   a single host volume, and feature_transform, as src/edt.pyx takes them: a 1-D volume takes a
              scalar or the first entry, more axes iterate the entries (a scalar is a TypeError);
    "wrap"    a single device volume of the edt family: a scalar is one entry;
    "cuda"    edt_cuda and transform_batch: a scalar for one axis, more axes iterate the entries."""
  if anisotropy is None:
    return (1.0,) * n
  if rule == "volume":
    if np.ndim(anisotropy) == 0 and n == 1:
      return (float(anisotropy),)
    weights = tuple(float(a) for a in np.asarray(anisotropy).reshape(-1))
    if len(weights) != n:
      raise ValueError("anisotropy must have one entry per volume axis (%d), got %d" % (n, len(weights)))
    return weights
  if np.ndim(anisotropy) == 0 and (n == 1 or rule == "wrap"):
    anisotropy = (anisotropy,)
  elif n == 1 and rule == "first":
    anisotropy = (np.asarray(anisotropy).reshape(-1)[0],)
  weights = tuple(float(a) for a in anisotropy)
  if len(weights) != n:
    raise ValueError("anisotropy must have one entry per dimension")
  return weights


class _Volume:
  """The input of one transform or whole-volume operation, resolved for its C ABI call.  A numpy array (or a
  list) gives numpy results; a device array (a torch CUDA tensor or any __cuda_array_interface__ object)
  gives torch CUDA results computed on its current stream.  With `stacked` the slowest axis in memory
  indexes same-shaped volumes.  Given `dims`, the (least, most) dimensions of one volume, the number of
  dimensions is checked as the whole-volume operations check it and the memory order is fixed at once;
  the transforms check the dimensions with their own messages and then call order()."""

  def __init__(self, name, data, stacked=False, dims=None, device=0):
    t = _device_array(data)
    self.on_device = t is not None
    self.arr = t if self.on_device else np.asarray(data)
    self.nd = self.arr.dim() if self.on_device else self.arr.ndim
    self.stacked = 1 if stacked else 0
    self.vnd = self.nd - self.stacked
    self.name, self._device = name, device
    if dims is not None:
      lo, hi = dims[0] + self.stacked, dims[1] + self.stacked
      if not lo <= self.nd <= hi:
        raise TypeError("%s: %s takes %d-D to %d-D arrays, got %d-D"
                        % (name, "stacked=True" if stacked else "it", lo, hi, self.nd))
      self.order()

  def order(self, f_first=False, c_only=False):
    """Make `arr` C- or F-contiguous: C where both apply (F with `f_first`, as a single host volume of the
    transforms is read), a strided array copied to C order (any non-C tensor, with `c_only`).  The C ABI
    reads an F-ordered one as its C-ordered transpose, with the weights reversed."""
    arr, self.shape = self.arr, tuple(self.arr.shape)
    if self.on_device:
      contiguous = arr.is_contiguous()
      self.fortran = (not (contiguous or c_only) and self.nd > 1
                      and arr.permute(*reversed(range(self.nd))).is_contiguous())
      if not contiguous and not self.fortran:
        arr = arr.contiguous()
      self.size, self.flags = math.prod(self.shape), FLAG_LABELS_ON_DEVICE | FLAG_OUT_ON_DEVICE
    else:
      flags = arr.flags
      if not (flags.c_contiguous or flags.f_contiguous):
        arr = np.ascontiguousarray(arr)
        flags = arr.flags
      self.fortran = flags.f_contiguous and (f_first or not flags.c_contiguous)
      self.size, self.flags = arr.size, 0
    self.arr, self.dtype = arr, arr.dtype
    return self

  def set_weights(self, anisotropy, positive=True, rule="volume"):
    """One weight per volume axis by `rule` (see _weights; None: `anisotropy` is that tuple already), and with
    `positive` each finite and > 0; sets `geometry`, the vnd, sx, sy, sz, count, wx, wy, wz of the C ABI call."""
    weights = anisotropy if rule is None else _weights(self.vnd, anisotropy, rule)
    if positive:
      for w in weights:
        if not (np.isfinite(w) and w > 0.0):
          raise ValueError("%s: every anisotropy weight must be finite and > 0, got %r" % (self.name, anisotropy))
    dims, count = self.shape, 1
    if not self.fortran:                    # x-fastest: the last axis of a C-ordered array first
      dims, weights = dims[::-1], weights[::-1]
    if self.stacked:                        # the slowest axis in memory indexes the volumes
      dims, count = dims[:-1], dims[-1]
    pad = 3 - self.vnd
    (sx, sy, sz), (wx, wy, wz) = dims + (1,) * pad, tuple(weights) + (1.0,) * pad
    self.geometry = (self.vnd, sx, sy, sz, count, wx, wy, wz)
    self.volume_geometry = (self.vnd, sx, sy, sz, wx, wy, wz)       # of a C ABI call on one volume

  def labels(self):
    """(raw, nbytes): the label bits the C ABI compares -- floats by value (-0.0 folded onto +0.0),
    unsigned and bool labels as the integers of their width -- or None for a dtype it does not take."""
    if not self.on_device:
      raw = _label_view(self.arr)
      return None if raw is None else (raw, raw.dtype.itemsize)
    import torch
    t = self.arr
    raw = _torch_raw_labels(torch).get(t.dtype)
    if raw is None:
      return None
    if t.dtype in (torch.float32, torch.float64):
      t = t + 0
    return (t if raw is t.dtype else t.view(raw)), t.element_size()

  @property
  def floating(self):
    return self.dtype.is_floating_point if self.on_device else self.dtype.kind == "f"

  @property
  def ptr(self):
    return self.ptr_of(self.arr)

  def ptr_of(self, x):
    """The address of `x`, an array on the input's side (None: None)."""
    if x is None:
      return None
    return x.data_ptr() if self.on_device else x.ctypes.data

  @property
  def where(self):
    """The device and stream of the C ABI call."""
    if not self.on_device:
      return int(self._device), None
    import torch
    device = self.arr.device
    return device.index, ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)

  def empty(self, dtype=None, planes=None):
    """An output in the input's shape and memory order, or with `planes=k` k of them as one array of
    shape (k,) + shape.  `dtype`: a name numpy and torch share ("bool", "int32", "float32"), None for the
    input's."""
    lead = () if planes is None else (planes,)
    shape = lead + (self.shape[::-1] if self.fortran else self.shape)     # as the C ABI reads the input
    if not self.on_device:
      dtype = self.dtype if dtype is None else dtype
      if not lead:
        return np.empty(self.shape, dtype, order="F" if self.fortran else "C")
      out = np.empty(shape, dtype)
    else:
      import torch
      out = torch.empty(shape, dtype=self.dtype if dtype is None else getattr(torch, dtype), device=self.arr.device)
    if not self.fortran:
      return out
    back = tuple(range(len(lead))) + tuple(range(out.ndim - 1, len(lead) - 1, -1))
    return out.permute(*back) if self.on_device else out.transpose(back)

  def upload(self, device):
    """The ordered host array as a torch tensor on `device`, in its memory order: float labels as they are,
    others as the integers of their width that torch takes (uint8 for one byte, else signed)."""
    import torch
    arr = self.arr
    raw = arr if self.floating else arr.view(np.uint8 if arr.itemsize == 1 else np.dtype("i%d" % arr.itemsize))
    return torch.from_numpy(raw).to(device)

  def shaped(self, flat):
    """A flat host buffer of `size` elements viewed in the input's shape and memory order."""
    return flat.reshape(self.shape, order="F" if self.fortran else "C")

  def plane_ptrs(self, planes):
    """The C ABI's x-fastest index planes of `planes` (made by empty(planes=vnd)): plane j is the caller's
    axis j of an F-ordered input and axis vnd - 1 - j of a C-ordered one (within a volume, for a stack)."""
    axes = range(self.vnd) if self.fortran else range(self.vnd - 1, -1, -1)
    ptrs = [planes[k].data_ptr() for k in axes] if self.on_device else [planes[k].ctypes.data for k in axes]
    return (ctypes.c_void_p * self.vnd)(*ptrs)


def _chunk_budget(max_device_bytes, on_device=False, voxel_graph=None, dims=None, staged=False):
  """max_device_bytes as an int, after rejecting what the chunked and stacked transforms do not cover: a
  budget for a device-resident array or with a voxel graph, for a single volume (`dims`) not of 2 or 3
  dimensions, and any budget for a stack that is `staged` on the GPU whole."""
  if staged:
    raise ValueError("stacked=True stages the whole stack on the GPU at once; it cannot be combined with "
                     "max_device_bytes")
  if on_device:
    raise ValueError("max_device_bytes streams a host array through the GPU; a device-resident array already fits")
  if voxel_graph is not None:
    raise ValueError("max_device_bytes cannot be combined with voxel_graph")
  if dims is not None and dims not in (2, 3):
    raise ValueError("max_device_bytes needs a 2-D or 3-D array, got %d-D" % dims)
  budget = int(max_device_bytes)
  if budget < 0:
    raise ValueError("max_device_bytes must be non-negative (0: what the device has free)")
  return budget


def _stack_dims(dims, voxel_graph=None):
  """The volume ndim of a stacked array of `dims` dimensions, after rejecting what stacks do not cover."""
  if voxel_graph is not None:
    raise ValueError("stacked=True cannot be combined with voxel_graph")
  if dims < 2 or dims > 4:
    raise ValueError("stacked=True needs a 2-D to 4-D array: volumes of 1 to 3 dimensions along its slowest axis, "
                     "got %d-D" % dims)
  return dims - 1


def _transform(v, labels, nbytes, black_border, flags, out, budget=None, bound=None, graph=None):
  """The distance transform of the resolved volume `v` from the raw label bits `labels` into `out`,
  through the entry point the arguments ask for: edtb200_transform_multi for a single host volume
  on several GPUs, _stack for a stack (budget: its groups' device memory), _voxel_graph with a
  graph, _bounded with a bound, _chunked with a budget, else edtb200_transform.  A one-shot host
  transform that runs out of device memory (of a 2-D / 3-D volume, or any voxel graph) is
  streamed through one GPU in chunks instead."""
  lib = _lib()
  bb, flags, device = int(bool(black_border)), int(flags) | v.flags, v._device
  if not (v.on_device or v.stacked or graph is not None) and (
      isinstance(device, (list, tuple, range)) or (isinstance(device, np.ndarray) and device.ndim == 1)):
    # several GPUs of this process share ONE host volume (edtb200_transform_multi): Z slabs for the
    # X / Y passes, Y slabs for the Z pass, re-partitioned over NVLink; exact for any input
    devs = [int(d) for d in device]
    _check(lib.edtb200_transform_multi(v.ptr_of(labels), nbytes, *v.volume_geometry, bb, flags, v.ptr_of(out),
                                       (ctypes.c_int * len(devs))(*devs), len(devs)))
    return
  device, stream = v.where
  if v.stacked:
    _check(lib.edtb200_transform_stack(v.ptr_of(labels), nbytes, *v.geometry, bb, flags, v.ptr_of(out), device,
                                       budget, None, stream))
    return
  if graph is not None:
    one_shot, chunked = lib.edtb200_transform_voxel_graph, lib.edtb200_transform_voxel_graph_chunked
    args = (v.ptr_of(labels), nbytes, v.ptr_of(graph)) + v.volume_geometry + (bb, flags, v.ptr_of(out), device)
  else:
    one_shot, chunked = lib.edtb200_transform, lib.edtb200_transform_chunked
    args = (v.ptr_of(labels), nbytes) + v.volume_geometry + (bb, flags, v.ptr_of(out), device)
  if bound is not None:
    _check(lib.edtb200_transform_bounded(*args, stream, bound))
    return
  if budget is None:
    try:
      _check(one_shot(*args, stream))
      return
    except EDTError as e:
      if e.code != ENOMEM or v.on_device or (graph is None and v.nd not in (2, 3)):
        raise
    budget = 0                              # too large for the device: stream it through in chunks
  _check(chunked(*args, budget, stream))


def _voxel_graph(v, voxel_graph, anisotropy, rule, black_border, flags):
  """__edt2dsq_voxel_graph / __edt3dsq_voxel_graph, src/edt.pyx:514-620, 736-844, of a resolved volume; with
  FLAG_SIGNED f(data) - f(data == 0), both under the graph (src/edt.pyx:147-158).  The labels only say
  foreground / background, and for floats the reference tests `labels[loc] > 0`
  (src/edt_voxel_graph.hpp:76, 151): negative values and NaN are background, on the host through
  EDTB200_LABELS_FLOAT and on the device as a uint8 mask."""
  signed = bool(flags & FLAG_SIGNED)
  flags &= ~FLAG_SIGNED
  if v.on_device:
    import torch
    labels = ((v.arr > 0).to(torch.uint8), 1) if v.dtype in (torch.float32, torch.float64) else v.labels()
    if labels is None:
      raise TypeError("edt_cuda: unsupported label dtype %s" % v.dtype)
    graph = _device_array(voxel_graph)
    if graph is None:
      graph = torch.as_tensor(np.ascontiguousarray(voxel_graph), device=v.arr.device)
    if graph.dtype not in (torch.uint8, torch.int8):
      graph = graph.to(torch.uint8)
    if not (graph.device == v.arr.device and tuple(graph.shape) == v.shape):
      raise ValueError("edt_cuda: voxel_graph must be a uint8/int8 CUDA tensor shaped like labels")
    graph = (graph.permute(*reversed(range(v.nd))) if v.fortran else graph).contiguous()
    new = lambda: v.empty("float32")
    background = lambda: (labels[0] == 0).view(torch.uint8)
  else:
    graph = _graph_bytes(voxel_graph, "F" if v.fortran else "C")
    if graph.shape != v.shape:
      raise ValueError("voxel_graph must have the shape of data")
    if v.dtype in (np.float32, np.float64):
      labels, flags = (v.arr, v.arr.itemsize), flags | FLAG_LABELS_FLOAT
    else:
      labels = v.labels()
    new = lambda: v.shaped(np.empty(v.size, dtype=np.float32))
    background = lambda: (v.arr == 0).view(np.uint8)
  if labels is None:                        # no branch in the reference: f(data) is zeros
    out = np.zeros(v.shape, dtype=np.float32, order="F" if v.fortran else "C")
    if not signed:
      return out
  v.set_weights(anisotropy, positive=False, rule=rule)
  if labels is not None:
    out = new()
    _transform(v, *labels, black_border, flags, out, graph=graph)
  if signed:
    other = new()
    _transform(v, background(), 1, black_border, flags & ~FLAG_LABELS_FLOAT, other, graph=graph)
    out -= other
  return out


def _front_door(data, anisotropy, black_border, voxel_graph, flags, device, fixed_dims=None, max_device_bytes=None,
                stacked=False, bound=None):
  """Argument handling of edtsq(), src/edt.pyx:276-310, for host and device arrays and stacks.  bound:
  max_distance after _bound.  `max_device_bytes` streams a 2-D / 3-D host volume through one GPU in chunks
  within that budget, and with None a one-shot transform that runs out of device memory is retried once
  that way; for a host stack it is the budget of the groups of whole volumes that go through the GPU."""
  v = _Volume("edt", data, stacked, device=device[0] if voxel_graph is not None and isinstance(device, (list, tuple))
              else device)
  nd, rule = v.nd, "first"                 # a single host volume takes its weights as src/edt.pyx does
  if stacked:
    _stack_dims(nd, voxel_graph)
    anisotropy, rule = _weights(v.vnd, anisotropy), None
    max_device_bytes = 0 if max_device_bytes is None else _chunk_budget(max_device_bytes, v.on_device)
  else:
    if v.on_device and max_device_bytes is not None:
      _chunk_budget(max_device_bytes, True)
    if fixed_dims is not None and nd != fixed_dims:
      raise ValueError("expected a %d-D array, got %d-D" % (fixed_dims, nd))
    if max_device_bytes is not None:
      max_device_bytes = _chunk_budget(max_device_bytes, False, voxel_graph, nd)
  if v.on_device:
    import torch
    if not stacked:
      if nd > 3:
        raise TypeError(_TOO_MANY_DIMS.format(nd))
      if voxel_graph is not None and nd not in (2, 3):
        raise TypeError(_GRAPH_DIMS.format(nd))
    if v.arr.numel() == 0:
      return torch.zeros(v.arr.shape, dtype=torch.float32, device=v.arr.device)
    if not stacked:
      anisotropy, rule = _weights(nd, anisotropy, "wrap"), None
      if nd < 1:
        raise TypeError(_TOO_MANY_DIMS.format(nd))
  elif not stacked:
    if v.arr.size == 0:
      return np.zeros(shape=v.arr.shape, dtype=np.float32)
    if voxel_graph is not None and nd not in (2, 3):
      raise TypeError(_GRAPH_DIMS.format(nd))
    if voxel_graph is None and not 1 <= nd <= 3:
      raise TypeError(_TOO_MANY_DIMS.format(nd))
  v.order(f_first=not (stacked or v.on_device))
  if voxel_graph is not None:
    return _voxel_graph(v, voxel_graph, anisotropy, rule, black_border, flags)
  labels = v.labels() if v.size else None
  if labels is None:
    if v.on_device:
      raise TypeError("edt_cuda: unsupported label dtype %s" % v.dtype)
    return np.zeros(v.shape, dtype=np.float32, order="F" if v.fortran else "C")
  v.set_weights(anisotropy, positive=False, rule=rule)
  out = v.empty("float32") if v.on_device else v.shaped(_result_buffer(v.size))
  _transform(v, *labels, black_border, flags, out, max_device_bytes, bound)
  return out


# ---------------------------------------------------------------------------------------
# public API (signatures follow src/edt.pyx; `device` is keyword-only and additive)
# ---------------------------------------------------------------------------------------

def _pick(device, devices, max_device_bytes=None, stacked=False):
  """`devices` (a sequence of GPU ordinals: one host volume spread over them) wins over `device`."""
  if devices is None:
    return device
  if stacked:
    raise ValueError("stacked=True runs on one GPU; it cannot be combined with devices=[...]")
  if max_device_bytes is not None:
    raise ValueError("max_device_bytes streams through one GPU; it cannot be combined with devices=[...]")
  devs = [int(d) for d in devices]
  if not devs:
    raise ValueError("devices must name at least one GPU")
  return devs if len(devs) > 1 else devs[0]


# `max_device_bytes=N` (every function below but the 1-D ones) streams a 2-D / 3-D host array
# through one GPU in chunks that fit N bytes of device memory (0: what the GPU has free), with the
# result of the one-shot transform bit for bit; with None a one-shot transform that runs out of
# device memory falls back to that once (see _transform).
#
# `stacked=True` (edt, edtsq, sdf, sdfsq, edt_cuda, feature_transform, expand_labels) takes a 2-D to
# 4-D array whose slowest axis in memory (axis 0 of a C-ordered array, the last of an F-ordered one) indexes
# independent volumes of 1 to 3 dimensions: each is transformed on its own, with one launch per pass
# for the whole stack.  `anisotropy` has one entry per volume axis, black_border applies to every
# volume's own faces, and the result has the input's shape and memory order, equal to np.stack of
# the per-volume calls.  For host arrays max_device_bytes is the budget of the groups of whole volumes
# that go through the GPU at once.
#
# `max_distance=d` (every function below, edt_cuda and feature_transform) computes only the distances
# up to d: where the unbounded squared distance S (|S| for sdf / sdfsq) has (double)S <= d * d the
# result is the unbounded one bit for bit, elsewhere +inf (-inf on signed background); unsigned
# background stays 0.  Later passes then only look d / w rows either way (include/edt_b200.h,
# DESIGN.md section 5).  None or +inf is the unbounded transform; d = 0 is allowed, a negative or NaN
# d is a ValueError, and so is max_distance with voxel_graph, devices=[...], stacked=True or
# max_device_bytes.

def edtsq(data, anisotropy=None, black_border=False, parallel=1, voxel_graph=None, order=None,
          *, device=0, devices=None, max_device_bytes=None, stacked=False, max_distance=None):
  """Squared anisotropic multi-label EDT of a 1-D, 2-D or 3-D array (src/edt.pyx:245-310).
  `devices=[0, 1, ...]` spreads one host volume over several GPUs (see _transform)."""
  bound = _bound(max_distance, voxel_graph, devices, stacked, max_device_bytes)
  return _front_door(data, anisotropy, black_border, voxel_graph, 0, _pick(device, devices, max_device_bytes, stacked),
                     max_device_bytes=max_device_bytes, stacked=stacked, bound=bound)


def edt(data, anisotropy=None, black_border=False, parallel=1, voxel_graph=None, order=None,
        *, device=0, devices=None, max_device_bytes=None, stacked=False, max_distance=None):
  """Anisotropic multi-label EDT (src/edt.pyx:205-242); the sqrt is fused into the last pass."""
  bound = _bound(max_distance, voxel_graph, devices, stacked, max_device_bytes)
  return _front_door(data, anisotropy, black_border, voxel_graph, FLAG_SQRT,
                     _pick(device, devices, max_device_bytes, stacked), max_device_bytes=max_device_bytes,
                     stacked=stacked, bound=bound)


def sdf(data, anisotropy=None, black_border=False, parallel=1, voxel_graph=None, order=None,
        *, device=0, devices=None, max_device_bytes=None, stacked=False, max_distance=None):
  """Signed distance function, edt(data) - edt(data == 0) (src/edt.pyx:121-158), computed as
  one transform with background as a label and the sign applied in the last store."""
  bound = _bound(max_distance, voxel_graph, devices, stacked, max_device_bytes)
  return _front_door(data, anisotropy, black_border, voxel_graph, FLAG_SQRT | FLAG_SIGNED,
                     _pick(device, devices, max_device_bytes, stacked), max_device_bytes=max_device_bytes,
                     stacked=stacked, bound=bound)


def sdfsq(data, anisotropy=None, black_border=False, parallel=1, voxel_graph=None, *, device=0, devices=None,
          max_device_bytes=None, stacked=False, max_distance=None):
  """Squared signed distance function (src/edt.pyx:161-202)."""
  bound = _bound(max_distance, voxel_graph, devices, stacked, max_device_bytes)
  return _front_door(data, anisotropy, black_border, voxel_graph, FLAG_SIGNED,
                     _pick(device, devices, max_device_bytes, stacked), max_device_bytes=max_device_bytes,
                     stacked=stacked, bound=bound)


def edt1dsq(data, anisotropy=1.0, black_border=False, *, device=0, max_distance=None):
  return _front_door(data, anisotropy, black_border, None, 0, device, fixed_dims=1, bound=_bound(max_distance))


def edt1d(data, anisotropy=1.0, black_border=False, *, device=0, max_distance=None):
  return _front_door(data, anisotropy, black_border, None, FLAG_SQRT, device, fixed_dims=1,
                     bound=_bound(max_distance))


def edt2dsq(data, anisotropy=(1.0, 1.0), black_border=False, parallel=1, voxel_graph=None,
            *, device=0, max_device_bytes=None, max_distance=None):
  bound = _bound(max_distance, voxel_graph, max_device_bytes=max_device_bytes)
  return _front_door(data, anisotropy, black_border, voxel_graph, 0, device, fixed_dims=2,
                     max_device_bytes=max_device_bytes, bound=bound)


def edt2d(data, anisotropy=(1.0, 1.0), black_border=False, parallel=1, voxel_graph=None,
          *, device=0, max_device_bytes=None, max_distance=None):
  bound = _bound(max_distance, voxel_graph, max_device_bytes=max_device_bytes)
  return _front_door(data, anisotropy, black_border, voxel_graph, FLAG_SQRT, device, fixed_dims=2,
                     max_device_bytes=max_device_bytes, bound=bound)


def edt3dsq(data, anisotropy=(1.0, 1.0, 1.0), black_border=False, parallel=1, voxel_graph=None,
            *, device=0, max_device_bytes=None, max_distance=None):
  bound = _bound(max_distance, voxel_graph, max_device_bytes=max_device_bytes)
  return _front_door(data, anisotropy, black_border, voxel_graph, 0, device, fixed_dims=3,
                     max_device_bytes=max_device_bytes, bound=bound)


def edt3d(data, anisotropy=(1.0, 1.0, 1.0), black_border=False, parallel=1, voxel_graph=None,
          *, device=0, max_device_bytes=None, max_distance=None):
  bound = _bound(max_distance, voxel_graph, max_device_bytes=max_device_bytes)
  return _front_door(data, anisotropy, black_border, voxel_graph, FLAG_SQRT, device, fixed_dims=3,
                     max_device_bytes=max_device_bytes, bound=bound)


# ---------------------------------------------------------------------------------------
# device-resident entry (zero-copy): torch CUDA tensor in, torch CUDA tensor out
# ---------------------------------------------------------------------------------------

_TORCH_LABEL_BYTES = None
_TORCH_RAW_LABELS = None


def _torch_label_bytes(torch):
  global _TORCH_LABEL_BYTES
  if _TORCH_LABEL_BYTES is None:
    table = {torch.bool: 1, torch.uint8: 1, torch.int8: 1, torch.int16: 2, torch.int32: 4,
             torch.int64: 8}
    for name, size in (("uint16", 2), ("uint32", 4), ("uint64", 8)):
      if hasattr(torch, name):
        table[getattr(torch, name)] = size
    _TORCH_LABEL_BYTES = table
  return _TORCH_LABEL_BYTES


def _torch_raw_labels(torch):
  """The dtype whose bits the C ABI compares, for each torch label dtype: floats by value (folded first),
  unsigned and bool labels as the integers of their width."""
  global _TORCH_RAW_LABELS
  if _TORCH_RAW_LABELS is None:
    signed = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}
    table = {d: (d if d == torch.int8 else signed[n]) for d, n in _torch_label_bytes(torch).items()}
    table.update({torch.float32: torch.int32, torch.float64: torch.int64})
    _TORCH_RAW_LABELS = table
  return _TORCH_RAW_LABELS


def edt_cuda(labels, anisotropy=None, black_border=False, *, sqrt=False, signed=False, out=None,
             voxel_graph=None, stacked=False, max_distance=None):
  """Transform a C-contiguous integer/bool torch CUDA tensor of 1-3 dims on its own device
  and current stream, asynchronously; returns a float32 CUDA tensor of the same shape
  (`out` may be passed to reuse a buffer).  Same semantics as edtsq/edt/sdfsq/sdf.
  `voxel_graph` (a uint8/int8 CUDA tensor of the same shape, 2-D / 3-D only, not with `signed`)
  selects the connectivity-graph transform.  `stacked=True` takes a (B, ...) tensor of 2-4 dims:
  B volumes of 1-3 dims, each transformed on its own, one launch per pass for all of them
  (`anisotropy`: one entry per volume axis).  `max_distance`: the bounded transform, as for edtsq."""
  import torch
  if not (isinstance(labels, torch.Tensor) and labels.is_cuda):
    raise TypeError("edt_cuda expects a torch CUDA tensor")
  bound = _bound(max_distance, voxel_graph, stacked=stacked)
  v = _Volume("edt_cuda", labels, stacked)
  nd = v.nd
  if stacked:
    _stack_dims(nd, voxel_graph)
  elif nd < 1 or nd > 3:
    raise TypeError(_TOO_MANY_DIMS.format(nd))
  labels = v.order(c_only=True).arr
  nbytes = _torch_label_bytes(torch).get(v.dtype)
  if nbytes is None:
    raise TypeError("edt_cuda: unsupported label dtype %s" % v.dtype)
  if out is None:
    out = torch.empty(v.shape, dtype=torch.float32, device=labels.device)
  elif not (out.is_cuda and out.dtype == torch.float32 and out.is_contiguous()
            and out.shape == labels.shape and out.device == labels.device):
    raise ValueError("edt_cuda: `out` must be a contiguous float32 CUDA tensor of the same shape/device")
  if v.size == 0:
    return out
  v.set_weights(anisotropy, positive=False, rule="cuda")
  if voxel_graph is not None:
    if nd not in (2, 3):
      raise TypeError(_GRAPH_DIMS.format(nd))
    if signed:
      raise ValueError("edt_cuda: with voxel_graph, form f(labels) - f(labels == 0) from two calls")
    if not (isinstance(voxel_graph, torch.Tensor) and voxel_graph.device == labels.device
            and voxel_graph.dtype in (torch.uint8, torch.int8) and voxel_graph.shape == labels.shape):
      raise ValueError("edt_cuda: voxel_graph must be a uint8/int8 CUDA tensor shaped like labels")
    voxel_graph = voxel_graph.contiguous()
  flags = (FLAG_SQRT if sqrt else 0) | (FLAG_SIGNED if signed else 0)
  _transform(v, labels, nbytes, black_border, flags, out, budget=0 if stacked else None, bound=bound,
             graph=voxel_graph)
  return out


def transform_batch(volumes, anisotropy=None, black_border=False, *, sqrt=False, signed=False, outs=None,
                    device=0):
  """edtsq (or edt / sdfsq / sdf via `sqrt` / `signed`) of many arrays of ONE shape, dtype and
  memory order -- e.g. the chunks of a dataset -- pipelined through the GPU: the upload of chunk
  k+1 and the download of chunk k-1 overlap the transform of chunk k (`edtb200_transform_batch`).
  Returns a list of float32 arrays (the arrays of `outs`, if given: same shape and order as the
  inputs, float32; pass pinned buffers, e.g. `torch.empty(..., pin_memory=True).numpy()`, to let
  the copies run at the PCIe rate).  Each result equals the single-call function's."""
  vols = [np.asarray(v) for v in volumes]
  if not vols:
    return []
  first = vols[0]
  if first.ndim < 1 or first.ndim > 3:
    raise TypeError(_TOO_MANY_DIMS.format(first.ndim))
  order = "F" if first.flags.f_contiguous else "C"
  fixed = []
  for v in vols:
    if v.shape != first.shape or v.dtype != first.dtype:
      raise ValueError("transform_batch: all volumes must share one shape and dtype")
    if order == "F" and not v.flags.f_contiguous:
      v = np.asfortranarray(v)
    elif order == "C" and not v.flags.c_contiguous:
      v = np.ascontiguousarray(v)
    fixed.append(v)
  if outs is None:
    outs = [np.empty(first.shape, dtype=np.float32, order=order) for _ in fixed]
  else:
    outs = list(outs)
    if len(outs) != len(fixed):
      raise ValueError("transform_batch: one output array per volume")
    for o in outs:
      ok = isinstance(o, np.ndarray) and o.dtype == np.float32 and o.shape == first.shape and \
          (o.flags.f_contiguous if order == "F" else o.flags.c_contiguous) and o.flags.writeable
      if not ok:
        raise ValueError("transform_batch: outs must be writable float32 arrays shaped and ordered like the volumes")
  if first.size == 0:
    for o in outs:
      o[...] = 0
    return outs
  views = [_label_view(v) for v in fixed]
  if views[0] is None:                      # dtype the reference does not dispatch on: zeros
    for o in outs:
      o[...] = 0
    return outs
  nd = first.ndim
  (sx, sy, sz), (wx, wy, wz) = _x_fastest(first.shape, _weights(nd, anisotropy, "cuda"), order == "F")
  n = len(views)
  lab_ptrs = (ctypes.c_void_p * n)(*[v.ctypes.data for v in views])
  out_ptrs = (ctypes.c_void_p * n)(*[o.ctypes.data for o in outs])
  flags = (FLAG_SQRT if sqrt else 0) | (FLAG_SIGNED if signed else 0)
  _check(_lib().edtb200_transform_batch(lab_ptrs, out_ptrs, n, views[0].dtype.itemsize, nd, sx, sy, sz,
                                        wx, wy, wz, int(bool(black_border)), flags, int(device)))
  return outs


# ---------------------------------------------------------------------------------------
# feature transform: WHERE the nearest boundary is (scipy's return_indices), and expand_labels
# ---------------------------------------------------------------------------------------

def _feature(v, black_border, flags, want_dist, budget=None, bound=None):
  """(distances or None, indices) of the resolved volume `v`, its order and weights set: the index planes
  from empty(planes=vnd), the distances zeroed first.  The entry point follows the arguments as in
  _transform, a one-shot host call that runs out of device memory included."""
  labels = v.labels()
  if labels is None:
    raise TypeError("feature_transform: unsupported label dtype %s" % v.dtype)
  planes = v.empty("int32", planes=v.vnd)
  dist = None
  if want_dist:
    dist = v.empty("float32").zero_() if v.on_device else v.shaped(np.zeros(v.size, dtype=np.float32))
  if v.size:
    lib = _lib()
    device, stream = v.where
    tail = (int(bool(black_border)), int(flags) | v.flags, v.ptr_of(dist), v.plane_ptrs(planes), device)
    if v.stacked:
      _check(lib.edtb200_feature_transform_stack(v.ptr_of(labels[0]), labels[1], *v.geometry, *tail, stream))
      return dist, planes
    args = (v.ptr_of(labels[0]), labels[1]) + v.volume_geometry + tail
    if bound is not None:
      _check(lib.edtb200_feature_transform_bounded(*args, stream, bound))
    elif budget is None:
      try:
        _check(lib.edtb200_feature_transform(*args, stream))
      except EDTError as e:
        if e.code != ENOMEM or v.on_device or v.nd not in (2, 3):
          raise
        budget = 0                          # too large for the device: stream it through in chunks
    if budget is not None:
      _check(lib.edtb200_feature_transform_chunked(*args, budget, stream))
  return dist, planes


def feature_transform(data, anisotropy=None, black_border=False, *, signed=False, return_distances=False, device=0,
                      max_device_bytes=None, stacked=False, max_distance=None):
  """The nearest site of every voxel: scipy.ndimage.distance_transform_edt(return_indices=True)
  for multi-label volumes, on the GPU.

  A site of voxel p is a voxel of another label, or with `black_border` a position just outside
  the volume (one coordinate -1 or n).  Foreground voxels get a nearest site; background voxels
  (label 0) get themselves, or with `signed=True` -- background as an ordinary label, as in sdf --
  their nearest voxel of a non-zero label.  Where there is no site at all (only possible without
  `black_border`) every coordinate is -1.  Among equally near sites, any one is returned, the same
  one on every run.

  Returns `indices`, int32 of shape (data.ndim,) + data.shape in scipy's layout (indices[k] is the
  coordinate along array axis k, each plane in the input's memory order), or with
  `return_distances=True` the pair (distances, indices), the distances equal to edt(data) (or
  sdf(data) with `signed=True`) bit for bit.  Arguments are handled as by edt(); device-resident
  input (a torch CUDA tensor or `__cuda_array_interface__`) returns torch CUDA tensors, computed on
  the current stream.

  `max_device_bytes=N` streams a 2-D / 3-D host array through one GPU in chunks that fit N bytes of
  device memory (0: what the GPU has free), with the one-shot result bit for bit; with None a one-shot
  call that runs out of device memory falls back to that once.

  `stacked=True` takes a 2-D to 4-D array whose slowest axis in memory indexes independent volumes,
  as edt(stacked=True) does: `indices` then has shape (data.ndim - 1,) + data.shape and holds the
  coordinates within each voxel's own volume.  The whole stack is staged on the GPU at once, so it
  cannot be combined with max_device_bytes.

  `max_distance=d` finds only the sites within d: inside that band the distances follow edt's bounded
  rule and the sites are as above; outside it every coordinate is -1 and the distance +inf (-inf on
  signed background).  Unsigned background still maps to itself.  It cannot be combined with stacked
  or max_device_bytes."""
  bound = _bound(max_distance, stacked=stacked, max_device_bytes=max_device_bytes)
  flags = FLAG_SQRT | (FLAG_SIGNED if signed else 0)
  v = _Volume("feature_transform", data, stacked, device=device)
  max_device_bytes = _feature_budget(v, max_device_bytes)
  anisotropy = _weights(v.vnd, anisotropy) if stacked else _single_weights(v, anisotropy)
  v.order(f_first=not (stacked or v.on_device))
  v.set_weights(anisotropy, positive=False, rule=None)
  dist, idx = _feature(v, black_border, flags, return_distances, max_device_bytes, bound)
  return (dist, idx) if return_distances else idx


def _feature_budget(v, max_device_bytes):
  """max_device_bytes of feature_transform and expand_labels, after rejecting a budget for a stack, which is
  staged on the GPU whole, and a stack of the wrong number of dimensions."""
  if v.stacked:
    _stack_dims(v.nd)
    return _chunk_budget(max_device_bytes, staged=True) if max_device_bytes is not None else None
  return None if max_device_bytes is None else _chunk_budget(max_device_bytes, v.on_device, None, v.nd)


def _single_weights(v, anisotropy):
  """The weights of one volume of feature_transform and expand_labels, taken as edt takes a host array."""
  if not 1 <= v.nd <= 3:
    raise TypeError(_TOO_MANY_DIMS.format(v.nd))
  return _weights(v.nd, anisotropy, "first")


def _expand_host(v, distance, anisotropy, max_device_bytes):
  """expand_labels of a resolved host volume through the chunked feature transform: the labels are
  gathered on the host, a bounded range of voxels at a time, at the background voxels that grow."""
  v.set_weights(_single_weights(v, anisotropy), positive=False, rule=None)
  dist, idx = _feature(v, False, FLAG_SIGNED, True, max_device_bytes)
  arr = v.arr
  order = "F" if arr.flags.f_contiguous and not arr.flags.c_contiguous else "C"
  out = arr.copy(order=order)
  # every array here is contiguous in `order`, so these flat views follow memory
  lab, sq, flat_out = arr.ravel(order=order), dist.ravel(order=order), out.ravel(order=order)
  planes = [idx[k].ravel(order=order) for k in range(arr.ndim)]
  limit = float(distance) ** 2
  step = 1 << 22
  for s in range(0, lab.size, step):
    e = min(lab.size, s + step)
    grow = np.flatnonzero((lab[s:e] == 0) & (planes[0][s:e] >= 0) & (np.abs(sq[s:e]).astype(np.float64) <= limit))
    if grow.size:
      site = np.ravel_multi_index(tuple(p[s:e][grow] for p in planes), arr.shape, order=order)
      flat_out[s + grow] = lab[site]
  return out


def _expand_device(v, distance, anisotropy):
  """expand_labels of a device volume (with `stacked`, a stack of volumes along its slowest axis in memory) on
  its current stream: the signed feature transform, then one gather kernel (edtb200_expand_gather) over the
  labels and index planes in the layout the transform used.  The result has the input's memory order."""
  if not v.stacked:
    anisotropy = _single_weights(v, anisotropy)
  v.order()
  v.set_weights(anisotropy, positive=False, rule=None)
  dist, idx = _feature(v, False, FLAG_SIGNED, True)
  if v.size == 0:
    return v.arr.clone()
  out = v.empty()
  flags = v.flags | (FLAG_LABELS_FLOAT if v.floating else 0)
  _check(_lib().edtb200_expand_gather(v.ptr, v.arr.element_size(), *v.geometry[:5], v.ptr_of(dist),
                                      v.plane_ptrs(idx), float(distance) ** 2, flags, v.ptr_of(out), *v.where))
  return out


def expand_labels(labels, distance=1.0, anisotropy=None, *, device=0, max_device_bytes=None, stacked=False):
  """skimage.segmentation.expand_labels on the GPU: every background voxel (label 0) whose nearest
  labelled voxel lies within `distance` takes that voxel's label; labelled voxels keep theirs.
  "Within" compares the squared distance (as sdfsq computes it, in float64) with distance**2, so a
  negative distance acts as its magnitude, NaN grows nothing and inf grows every background voxel of
  a volume that has a label.  For float labels background is the value 0 (-0.0 too), and every
  label, -0.0 and NaN payloads included, is copied bit for bit.  The result has the dtype, shape and
  memory order of `labels`; a torch CUDA tensor in gives one out, computed on the current stream.
  Built on feature_transform(signed=True); one CUDA kernel then gathers the labels on the device.

  `max_device_bytes=N` (2-D / 3-D host arrays) runs the feature transform in chunks that fit N bytes
  of device memory (0: what the GPU has free) and gathers the labels on the host; with None a host
  array too large for the device falls back to that once.

  `stacked=True` takes a 2-D to 4-D array whose slowest axis in memory indexes independent volumes,
  as edt(stacked=True) does: every volume grows on its own, with one launch per pass for the whole
  stack, and the result equals np.stack of the per-volume calls.  `anisotropy` has one entry per
  volume axis.  The whole stack is staged on the GPU at once: it cannot be combined with
  max_device_bytes, and a host stack that does not fit raises EDTError with code ENOMEM."""
  import torch
  v = _Volume("expand_labels", labels, stacked, device=device)
  max_device_bytes = _feature_budget(v, max_device_bytes)
  if stacked:
    anisotropy = _weights(v.vnd, anisotropy)
  if v.on_device:
    return _expand_device(v, distance, anisotropy)
  v.order(f_first=not stacked)
  if v.labels() is None:
    raise TypeError("expand_labels: unsupported label dtype %s" % v.dtype)
  if max_device_bytes is None:
    # host arrays go up through torch, are grown on the device and come back
    if stacked:
      if v.size == 0:
        return v.arr.copy(order="F" if v.fortran else "C")
      if device_count() == 0:
        raise EDTError("edt_b200 error %d: no usable CUDA device; this library has no CPU fallback" % ECUDA, ECUDA)
    arr = v.arr
    try:
      up = _Volume("expand_labels", v.upload(torch.device("cuda", int(device))), stacked)
      return _expand_device(up, distance, anisotropy).cpu().numpy().view(arr.dtype)
    except (EDTError, torch.cuda.OutOfMemoryError) as e:
      if stacked:
        if isinstance(e, EDTError):
          raise
        raise EDTError("edt_b200 error %d: the stack of %d bytes does not fit on the GPU (%s)"
                       % (ENOMEM, arr.nbytes, e), ENOMEM) from e
      if getattr(e, "code", ENOMEM) != ENOMEM or v.nd not in (2, 3):
        raise
    torch.cuda.empty_cache()                 # what the one-shot attempt left cached goes back to the device
    max_device_bytes = 0                     # too large for the device: the chunked path
  if v.size == 0:
    return v.arr.copy()
  return _expand_host(v, distance, anisotropy, max_device_bytes)


# ---------------------------------------------------------------------------------------
# spherical morphology: erosion, dilation, opening and closing with a Euclidean ball, each a threshold
# on a bounded transform whose last store writes labels (edtb200_morphology)
# ---------------------------------------------------------------------------------------

_ERODE, _DILATE, _OPEN, _CLOSE = 0, 1, 2, 3      # EDTB200_ERODE, _DILATE, _OPEN, _CLOSE


def _morph_label_bytes(dtype):
  """Label width of a numpy or torch dtype the morphology takes (None: not one)."""
  if isinstance(dtype, np.dtype):
    if dtype == np.bool_ or (dtype.kind in "iuf" and dtype.itemsize in (1, 2, 4, 8)):
      return None if dtype.kind == "f" and dtype.itemsize < 4 else dtype.itemsize
    return None
  import torch
  if dtype in (torch.float32, torch.float64):
    return 4 if dtype == torch.float32 else 8
  return _torch_label_bytes(torch).get(dtype)


def _morphology(op, labels, radius, anisotropy, black_border, device, stacked, name):
  """Every check before any device use, then one edtb200_morphology call: host arrays are staged whole
  (numpy out), device arrays run on the current stream (torch out)."""
  r = float(radius)
  if not (r >= 0.0 and r != float("inf")):
    raise ValueError("%s: radius must be finite and zero or more, got %r" % (name, radius))
  v = _Volume(name, labels, stacked, (1, 3), device)
  nbytes = _morph_label_bytes(v.dtype)
  if nbytes is None:
    raise TypeError("%s: unsupported label dtype %s" % (name, v.dtype))
  v.set_weights(anisotropy, positive=False)        # taken as edtb200_transform takes them
  out = v.empty("bool" if op in (_DILATE, _CLOSE) else None)
  if v.size:
    flags = v.flags | (FLAG_LABELS_FLOAT if v.floating else 0)
    _check(_lib().edtb200_morphology(v.ptr, nbytes, *v.geometry, op, r, int(bool(black_border)), flags,
                                     v.ptr_of(out), *v.where))
  return out


# Shared by the four functions below.  B is the ball {v in Z^n : sum_j (w_j v_j)^2 <= r^2}, w the
# anisotropy (one entry per axis of a volume, as for edt()), r the radius in the same units.  "Within r"
# compares the float32 squared distance that edtsq / sdfsq compute, in float64, with r * r -- the rule
# of max_distance= and expand_labels -- so each result is a threshold on one bounded transform
# (max_distance = r), whose last pass writes the labels directly.  Labels compare as edt() compares
# them: floats by value, so -0.0 is background.  A kept voxel keeps its exact bits (NaN payloads
# included); every other voxel is all-zero bits.  The result has the input's shape and memory order;
# numpy in gives numpy out, a torch CUDA tensor (or any __cuda_array_interface__ array) gives a torch
# CUDA tensor computed on the current stream without a host synchronisation.  `stacked=True` takes a 2-D
# to 4-D array whose slowest axis in memory indexes same-shaped volumes, as edt(stacked=True) does: the
# result equals np.stack of the per-volume calls, with one launch per pass for all of them; a host
# stack is staged on the GPU whole.  A radius that is negative, NaN or infinite is a ValueError, an
# unsupported dtype or number of dimensions a TypeError; a host array that does not fit on the GPU
# raises EDTError with code ENOMEM (there is no chunked path).

def spherical_erode(labels, radius, anisotropy=None, black_border=False, *, device=0, stacked=False):
  """Multi-label erosion by the ball of `radius`: a voxel keeps its label iff it is labelled (non-zero)
  and no voxel of another label (background included) lies within `radius`, i.e. its edtsq (with
  `black_border`: the volume's faces count as background) is not within radius; every other voxel
  becomes 0.  Per label k this is scipy.ndimage.binary_erosion(labels == k, B,
  border_value=0 if black_border else 1).  Radius 0 is the identity, and so is any radius for a volume
  of one label without black_border (it has no site at all).  Returns the input's dtype."""
  return _morphology(_ERODE, labels, radius, anisotropy, black_border, device, stacked, "spherical_erode")


def spherical_open(labels, radius, anisotropy=None, black_border=False, *, device=0, stacked=False):
  """Multi-label opening by the ball of `radius`: with E the spherical_erode result (with
  `black_border`), a voxel keeps its label iff it is labelled and the squared distance from it to the
  nearest voxel of E is within radius (that transform has no black border: no kept voxel lies outside
  the volume); every other voxel becomes 0.  Per label k this is
  scipy.ndimage.binary_dilation(eroded_k, B, border_value=0) -- not scipy's binary_opening with
  border_value=1, which dilates from outside the volume too.  Every label opens at once, without a
  loop over labels: the voxel q of E nearest p, if within radius, carries p's label, because the ball
  around q lies inside q's own label and contains p.  Both transforms run back to back on the GPU.
  Returns the input's dtype."""
  return _morphology(_OPEN, labels, radius, anisotropy, black_border, device, stacked, "spherical_open")


def spherical_dilate(labels, radius, anisotropy=None, *, device=0, stacked=False):
  """Binary dilation by the ball of `radius`: every non-zero voxel is foreground, and a voxel is set iff
  it is foreground or |sdfsq(labels)| there (the squared distance to the nearest foreground voxel) is
  within radius.  Equals scipy.ndimage.binary_dilation(labels != 0, B, border_value=0).  Returns a bool
  mask.  For a dilation that keeps the labels, see expand_labels."""
  return _morphology(_DILATE, labels, radius, anisotropy, False, device, stacked, "spherical_dilate")


def spherical_close(labels, radius, anisotropy=None, black_border=False, *, device=0, stacked=False):
  """Binary closing by the ball of `radius`: D = spherical_dilate(labels, radius), then D eroded as a
  two-label volume (with `black_border`: the faces count as background).  Equals
  scipy.ndimage.binary_erosion(D, B, border_value=0 if black_border else 1).  Both transforms run back to
  back on the GPU.  Returns a bool mask."""
  return _morphology(_CLOSE, labels, radius, anisotropy, black_border, device, stacked, "spherical_close")


# ---------------------------------------------------------------------------------------
# local thickness: the largest opening of a ladder of radii that still covers each voxel
# (edtb200_local_thickness)
# ---------------------------------------------------------------------------------------

THICKNESS_MAX_SIZES = 4096      # EDTB200_THICKNESS_MAX_SIZES


def _thickness_sizes(sizes, name):
  """An int n (default levels, as n) or the given radii as float64, sorted descending without repeats."""
  if isinstance(sizes, (bool, np.bool_)):
    raise TypeError("%s: sizes must be an integer or a 1-D sequence of radii, got %r" % (name, sizes))
  if isinstance(sizes, (int, np.integer)):
    if not 1 <= sizes <= THICKNESS_MAX_SIZES:
      raise ValueError("%s: sizes must be 1 to %d levels, got %d" % (name, THICKNESS_MAX_SIZES, sizes))
    return int(sizes)
  arr = np.asarray(sizes)
  if arr.dtype.kind not in "iuf":
    raise TypeError("%s: sizes must be an integer or a 1-D sequence of radii, got %r" % (name, sizes))
  if arr.ndim != 1 or arr.size == 0:
    raise ValueError("%s: sizes must be a non-empty 1-D sequence of radii, got shape %s" % (name, arr.shape))
  arr = arr.astype(np.float64)
  if not (np.all(np.isfinite(arr)) and np.all(arr >= 0.0)):
    raise ValueError("%s: every size must be finite and zero or more, got %r" % (name, sizes))
  arr = np.unique(arr)[::-1].copy()
  if arr.size > THICKNESS_MAX_SIZES:
    raise ValueError("%s: at most %d distinct sizes, got %d" % (name, THICKNESS_MAX_SIZES, arr.size))
  return arr


def local_thickness(labels, anisotropy=None, black_border=False, *, sizes=25, return_sizes=False, device=0,
                    stacked=False):
  """Local thickness of every label at once: for each labelled voxel, the largest radius of a ladder of sizes
  whose ball lies inside the voxel's own label and covers the voxel, as porespy's local_thickness defines it.

  Definition.  For labels L (0 is background), anisotropy w, black_border and levels r_1 > ... > r_m:
    1. D2 = edtsq(L, w, black_border), bit for bit;
    2. the seeds of level r are the voxels whose D2 is not within r ((double)D2 > r * r): the voxels
       spherical_erode(L, r, w, black_border) keeps;
    3. d2_r = edtsq of the mask that is 0 on the seeds and 1 elsewhere, without black border;
    4. out[p] = float32(max r_i with L(p) != 0 and (double)d2_r_i(p) <= r_i * r_i), or 0 where there is none.
  So out == max_i(np.where(spherical_open(L, r_i, w, black_border) != 0, r_i, 0)) bit for bit: every label is
  handled in one pass because the ball around a seed lies inside the seed's label.  The value is a RADIUS in
  the units of w; Hildebrand & Ruegsegger's thickness (BoneJ's Thickness) is twice it.  Labels compare as
  edt() compares them: floats by value, so -0.0 is background.  Exact Hildebrand thickness, with every
  distinct D2 as a level, is not offered: each level costs one transform of a 1-byte mask.

  Levels.  `sizes` is either
    - a sequence of radii, finite and >= 0: sorted descending without repeats, the same for every volume;
    - an integer n (default 25): per volume, in float64, with R = sqrt(the largest finite D2 over its
      labelled voxels) and h = min(w) (the least weight, rounded to float32 as every weight is),
      r_i = (h/2) * (2R/h)^(i/n) for i = 0 .. n-1.  Every labelled voxel gets at least h/2 and the top level
      stays below R; a volume with no finite labelled D2 (no labelled
      voxel, or one label without black_border) takes R = h/2.  These levels are computed on the GPU (pow
      may differ from numpy's in the last bit), so the result is defined relative to the levels used, which
      return_sizes=True returns: as out, sizes (shape (m,) descending, or (count, m) for a stack with
      default levels, whose volumes have their own levels).

  Input and output.  Labels of bool, any integer dtype, float32 or float64, 1-D to 3-D (2-D to 4-D with
  stacked=True, whose slowest axis in memory indexes same-shaped volumes as edt(stacked=True): the result
  equals np.stack of the per-volume calls).  Returns float32 with the input's shape and memory order.  numpy
  in gives numpy out; a torch CUDA tensor (or any __cuda_array_interface__ array) gives torch CUDA tensors
  computed on the current stream without a host synchronisation, default levels included.  Sizes that are
  empty, not 1-D, NaN, infinite or negative, an n below 1 or above THICKNESS_MAX_SIZES, and a weight that
  is not finite and > 0 are ValueErrors; an unsupported dtype or number of dimensions, or sizes of a
  non-numeric type, TypeErrors.  A host array that does not fit on the GPU raises EDTError with code ENOMEM
  (there is no chunked path).  Device memory beyond the input and output: 9 bytes per voxel (label bytes
  more for float labels)."""
  name = "local_thickness"
  levels = _thickness_sizes(sizes, name)
  if not isinstance(return_sizes, (bool, np.bool_)):
    raise TypeError("%s: return_sizes must be True or False, got %r" % (name, return_sizes))
  v = _Volume(name, labels, stacked, (1, 3), device)
  nbytes = _morph_label_bytes(v.dtype)
  if nbytes is None:
    raise TypeError("%s: unsupported label dtype %s" % (name, v.dtype))
  v.set_weights(anisotropy)
  out = v.empty("float32")
  count = v.geometry[4]
  by_default = isinstance(levels, int)
  m = levels if by_default else levels.size
  # the levels the C ABI writes: every default level, and the given ones only on the device (the host has them)
  used = None
  if return_sizes and (by_default or v.on_device):
    if v.on_device:
      import torch
      used = torch.empty((count, m), dtype=torch.float64, device=v.arr.device)
    else:
      used = np.empty((count, m), np.float64)
  if v.size:
    flags = v.flags | (FLAG_LABELS_FLOAT if v.floating else 0)
    _check(_lib().edtb200_local_thickness(v.ptr, nbytes, *v.geometry, int(bool(black_border)), flags,
                                          None if by_default else levels.ctypes.data, m, v.ptr_of(out),
                                          v.ptr_of(used), *v.where))
  elif used is not None:            # no voxel: every default level is h/2, and the given ones as they are
    used[...] = 0.5 * float(min(np.float32(x) for x in v.geometry[5:5 + v.vnd])) if by_default else \
        used.new_tensor(levels)
  if not return_sizes:
    return out
  if by_default:
    return out, (used if v.stacked else used[0])
  if not v.on_device:
    return out, levels
  return out, (used[0] if count else used.new_tensor(levels))


# ---------------------------------------------------------------------------------------
# parabolic erosion and dilation of float volumes: the distance transform of a sampled function
# (edtb200_parabolic)
# ---------------------------------------------------------------------------------------

_PARABOLIC_ERODE, _PARABOLIC_DILATE = 0, 1      # EDTB200_PARABOLIC_ERODE, _DILATE


def _parabolic(op, f, anisotropy, device, stacked, name, return_indices=False):
  """Every check before any device use, then one edtb200_parabolic call (edtb200_parabolic_sites with
  return_indices): host arrays are staged whole (numpy out), device arrays run on the current stream
  (torch out).  The index planes come back x first; indices[k], the coordinate along array axis k, is
  x-fastest plane vnd - 1 - k of a C-ordered array and plane k of an F-ordered one."""
  if not isinstance(return_indices, (bool, np.bool_)):
    raise TypeError("%s: return_indices must be True or False, got %r" % (name, return_indices))
  v = _Volume(name, f, stacked, (1, 3), device)
  if v.on_device:
    if v.arr.is_complex():
      raise TypeError("%s: it takes real or bool samples, got %s" % (name, v.dtype))
  elif v.dtype != np.bool_ and v.dtype.kind not in "iuf":
    raise TypeError("%s: it takes real or bool samples, got %s" % (name, v.dtype))
  v.set_weights(anisotropy)
  v.arr = v.arr.float() if v.on_device else v.arr.astype(np.float32, order="K", copy=False)   # memory order kept
  out = v.empty("float32")
  planes = v.empty("int32", planes=v.vnd) if return_indices else None
  if v.size:
    if return_indices:
      _check(_lib().edtb200_parabolic_sites(v.ptr, *v.geometry, op, v.flags, v.ptr_of(out), v.ptr_of(planes),
                                            *v.where))
    else:
      _check(_lib().edtb200_parabolic(v.ptr, *v.geometry, op, v.flags, v.ptr_of(out), *v.where))
  if not return_indices:
    return out
  # x first as written: an F-ordered caller's axis k is plane k, a C-ordered caller's is plane vnd - 1 - k
  return out, (planes if v.fortran else planes.flip(0) if v.on_device else planes[::-1])


_PARABOLIC_DOC = """

  Definition.  Volumes are x-fastest: for C-ordered input the last axis is x, as for edt().  Erosion
  starts from g = f as float32 and runs one pass per axis in the order x, y, z; each pass replaces every
  sample g(i) of a line by

      min( g(i), min_{j != i} fl32(fl64(fl64(w2 * (i-j)^2) + g(j))) ),   w2 = float32(w * w)

  -- w2 rounded in float32, the sum formed in float64 and rounded once to float32, which is what numpy
  gives in float64 followed by .astype(np.float32).  Lines never leave the volume and there are no
  border terms.  A NaN sample is never a site (read as +inf for erosion, -inf for dilation), every zero
  result is +0.0, a weight whose square overflows float32 leaves its pass's samples as they are, and
  (with a finite w2) one -inf sample makes its whole line -inf.  Dilation is -parabolic_erode(-f) with
  the same rules.  The result equals this definition bit for bit.

  Input and output.  Samples of any real dtype or bool are converted to float32 first (float64 rounds
  to float32 first).  The result is float32 with the input's shape and memory order; numpy in gives
  numpy out, a torch CUDA tensor (or any __cuda_array_interface__ array) gives a torch CUDA tensor
  computed on the current stream without a host synchronisation.  `stacked=True` takes a 2-D to 4-D
  array whose slowest axis in memory indexes same-shaped volumes, as edt(stacked=True) does: np.stack
  of the per-volume calls, one launch per pass for all of them.  A weight that is not finite and > 0 is
  a ValueError, a wrong number of dimensions or a non-real dtype a TypeError; a host array that does not
  fit on the GPU raises EDTError with code ENOMEM (there is no chunked path).

  return_indices=True returns (values, indices): the values bit for bit as without it, and the sample q
  that gives each value, int32 of shape (vnd,) + f.shape in scipy's layout (indices[k] is the coordinate
  along array axis k, each plane in the input's memory order; with stacked=True within each volume), as
  feature_transform returns them.  Each pass picks a site on every line among the candidates above (j = i
  included): on lines of at most 23170 samples the least j among the REAL minimisers of
  w2 * (i-j)^2 + g(j); on longer lines the least j among the minimisers of the float64 sum before its
  float32 rounding.  NaN and +inf samples are never sites; with a finite w2 a line holding -inf takes its
  least -inf position; with w2 = +inf every sample is its own site.  Dilation is the erosion of -f, so it
  names the least maximiser.  The sites compose as the feature transform's (q_z from the Z pass at p, q_y
  from the Y pass at (p_x, p_y, q_z), q_x from the X pass at (p_x, q_y, q_z)); where a line has no
  candidate at all every coordinate is -1 and the value +inf (-inf for dilation).  So f(q) is never NaN,
  and the value at p is the chain of rounded candidates from f(q): the X pass's, then Y's, then Z's.  It
  costs 4 bytes per voxel of device memory per pass but the last, and lines of more than 2^26 samples.

  Worked uses.
    edtsq of a mask, with integer weights w:
        parabolic_erode(np.where(mask, np.inf, 0), w) == edtsq(mask, w)          (bit for bit)
    the reverse distance transform -- the union of the balls of radius r at the medial points:
        parabolic_dilate(np.where(medial, r * r, -np.inf)) > 0
    ITK's ParabolicErode / DilateImageFilter at scale t with voxel spacing s:
        anisotropy = s / sqrt(2 t)
    the power (Laguerre) diagram of weighted seeds -- p's cell is the seed c least in |p - c|^2 - omega_c:
        f = np.where(seed_labels != 0, -omega, np.inf)
        _, idx = parabolic_erode(f, return_indices=True)
        cells = seed_labels[tuple(idx)]
    the best placement of a part (Felzenszwalb-Huttenlocher): q maximising score(q) - sum_a (w_a d_a)^2:
        best, idx = parabolic_dilate(score, w, return_indices=True)
    the medial ball that decides each voxel of the reverse distance transform (-1 off the union):
        cover, idx = parabolic_dilate(np.where(medial, r * r, -np.inf), return_indices=True)
        ball = np.where(cover > 0, ball_ids[tuple(idx)], -1)
  """


def parabolic_erode(f, anisotropy=None, *, device=0, stacked=False, return_indices=False):
  return _parabolic(_PARABOLIC_ERODE, f, anisotropy, device, stacked, "parabolic_erode", return_indices)


def parabolic_dilate(f, anisotropy=None, *, device=0, stacked=False, return_indices=False):
  return _parabolic(_PARABOLIC_DILATE, f, anisotropy, device, stacked, "parabolic_dilate", return_indices)


parabolic_erode.__doc__ = """Parabolic (grayscale) erosion: g(p) = min_q f(q) + sum_a (w_a (p_a - q_a))^2, computed as
  one exact lower envelope of parabolas per axis -- the distance transform of the sampled function f
  (Felzenszwalb-Huttenlocher).  Its cost per voxel does not depend on the weights.""" + _PARABOLIC_DOC
parabolic_dilate.__doc__ = """Parabolic (grayscale) dilation: g(p) = max_q f(q) - sum_a (w_a (p_a - q_a))^2, computed as
  -parabolic_erode(-f); NaN is never a site and zero results are +0.0.""" + _PARABOLIC_DOC


# ---------------------------------------------------------------------------------------
# the medial axis of every label: the power sites of its distance transform (edtb200_medial_axis)
# ---------------------------------------------------------------------------------------

def medial_axis(labels, anisotropy=None, black_border=False, *, return_distance=False, device=0, stacked=False):
  """The medial axis of every label at once: the voxels whose balls rebuild each label exactly.

  Definition.  For labels L (0 is background), anisotropy w and black_border:
    1. D2 = edtsq(L, w, black_border), bit for bit;
    2. V, q = parabolic_dilate(D2, w, return_indices=True) -- D2 as it is, 0 on the background -- so q(p)
       is p's power (Laguerre) site, the y maximising D2(y) - |p - y|^2_w;
    3. medial[y] is True iff y = q(p) for some voxel p with L(p) != 0.
  Labels compare as edt() compares them: floats by value, so -0.0 is background.  The tie rule is that of
  parabolic_dilate's indices: on lines of at most 23170 samples each pass takes the least j among the REAL
  maximisers, so with integer weights and values below 2^24 q(p) is the lexicographically least (z, y, x)
  among the maximisers over the whole volume.  Volumes are x-fastest, as for edt(): x is the last axis of a
  C-ordered array and the first of an F-ordered one, so where maximisers tie the two orders of the same
  labels can mark different (equally valid) voxels.  This is the reduced discrete medial axis of Coeurjolly &
  Montanvert: the balls B(y, sqrt(D2(y))) that are the power maximiser of at least one labelled voxel.  It is
  not thin and not connected: it is neither a topological skeleton (skimage's skeletonize, TEASAR) nor
  the minimal medial axis.

  Guarantees.  For any weights, at every voxel with L(p) != 0,
      parabolic_dilate(np.where(medial, D2, -np.inf), w) == V      (bit for bit, and > 0 there)
  because each pass is monotone (the restricted input gives no more than V) and q(p) is medial (its chain
  of rounded candidates gives V(p)).  With integer weights, moreover, that reconstruction is <= 0 on every
  background voxel, so `... > 0` equals `labels != 0` exactly; every site q(p) carries p's label; the balls
  of one label's medial voxels rebuild exactly that label; and every non-empty label has a medial voxel.
  Examples (1-D, background on both sides): a run of 5 has D2 = 1, 4, 9, 4, 1 and medial {2}; a run of 4
  has D2 = 1, 4, 4, 1 and medial {1, 2}.  A volume of one non-zero label without black_border has
  D2 = +inf, and its only medial voxel is its first voxel.

  Input and output.  Labels of bool, any integer dtype, float32 or float64, 1-D to 3-D (2-D to 4-D with
  stacked=True, whose slowest axis in memory indexes same-shaped volumes as edt(stacked=True); the result
  equals np.stack of the per-volume calls, one launch per pass for all of them).  Returns a bool array
  with the input's shape and memory order, and with return_distance=True also the distances
  edt(labels, anisotropy, black_border), bit for bit, as (medial, dist) -- as skimage's medial_axis returns
  them.  numpy in gives numpy out; a torch CUDA tensor (or any __cuda_array_interface__ array) gives torch
  CUDA tensors computed on the current stream without a host synchronisation.  A weight that is not finite
  and > 0 is a ValueError, an unsupported dtype or number of dimensions a TypeError; a host array that does
  not fit on the GPU raises EDTError with code ENOMEM (there is no chunked path).  Device memory beyond
  the input and the outputs: 4 + 4 * ndim bytes per voxel (16 in 3-D)."""
  name = "medial_axis"
  if not isinstance(return_distance, (bool, np.bool_)):
    raise TypeError("%s: return_distance must be True or False, got %r" % (name, return_distance))
  v = _Volume(name, labels, stacked, (1, 3), device)
  nbytes = _morph_label_bytes(v.dtype)
  if nbytes is None:
    raise TypeError("%s: unsupported label dtype %s" % (name, v.dtype))
  v.set_weights(anisotropy)
  medial = v.empty("bool")
  dist = v.empty("float32") if return_distance else None
  if v.size:
    flags = v.flags | (FLAG_LABELS_FLOAT if v.floating else 0)
    _check(_lib().edtb200_medial_axis(v.ptr, nbytes, *v.geometry, int(bool(black_border)), flags, v.ptr_of(medial),
                                      v.ptr_of(dist), *v.where))
  return (medial, dist) if return_distance else medial


# ---------------------------------------------------------------------------------------
# topology-preserving curve skeletons of every label, thinned in distance order (edtb200_skeletonize)
# ---------------------------------------------------------------------------------------

def skeletonize(labels, anisotropy=None, black_border=False, *, return_distance=False, device=0, stacked=False):
  """Topology-preserving curve skeletons of every label at once, thinned in distance order on the GPU.

  Definition.  Volumes are x-fastest, as for edt(): x is the last axis of a C-ordered array and the first of
  an F-ordered one; coordinates are taken within one volume.  The voxels of a label M are 26-connected
  (2-D: 8-); everything that is not M -- background, other labels and the voxels outside the volume -- is
  6-connected (2-D: 4-).  All labels are thinned at once, and deleting a voxel of M never changes the
  topology of another label.
    simple     p of label M is simple iff the M-voxels of N26(p) \\ {p} form exactly one 26-component and
               the non-M voxels of N18(p) \\ {p} have exactly one 6-component (within that set) that
               contains a 6-neighbour of p; in 2-D iff the M-pixels of N8(p) \\ {p} form one 8-component
               and the non-M pixels of N8(p) \\ {p} have exactly one 4-component 4-adjacent to p.
    end point  exactly one voxel of N26(p) \\ {p} (2-D: N8) has p's label.
    subfield   k = (x & 1) | (y & 1) << 1 | (z & 1) << 2 (2-D: (x & 1) | (y & 1) << 1).
  R = edtsq(labels, anisotropy, black_border), bit for bit; h = the least weight; theta_t = (t h)^2 in
  double for t = 1, 2, ...  Round t admits the labelled voxels still present with R <= theta_t; the rounds
  run up to the first t with theta_t >= the largest finite R, and a final round admits every voxel still
  present, R = +inf included (a label touching the volume's edge without black_border).  Inside a round,
  cycles repeat until one deletes nothing; a cycle runs the steps k = 0 .. 7 (2-D: 0 .. 3), and step k
  deletes at once every present admitted voxel of subfield k that is simple on the image at the start of
  the step and was not an end point at the start of the cycle.  The skeleton is what is left.  Peeling in
  the order of R centres the skeleton in physical units, also on voxels such as (4, 4, 40).
  Guarantees: every label keeps its number of components, the components of its complement (so its
  cavities and tunnels) and its Euler characteristic; the result is thin (no voxel of it is simple and not
  an end point) and lies within the labels.  The subfield order depends on the memory order, so an
  F-ordered array equals the C-ordered call on its transpose with the weights reversed, and the two orders
  of the same labels can give different, equally valid skeletons.
  Examples: a straight line one voxel thick is its own skeleton; an isolated voxel stays; a 3x3x3 cube in
  background gives exactly its centre; a hollow spherical shell keeps a closed surface around its cavity;
  a 4x6x12 box gives a line along its long axis; a 2-D disc gives one pixel.

  Input and output.  Labels of bool or integer dtypes of 1, 2, 4 or 8 bytes (float labels are a
  TypeError), 2-D or 3-D (3-D or 4-D with stacked=True, whose slowest axis in memory indexes same-shaped
  volumes as edt(stacked=True); the result equals np.stack of the per-volume calls).  Returns a bool array
  with the input's shape and memory order; the label of each skeleton voxel is labels[skeleton].  With
  return_distance=True it returns (skeleton, edt(labels, anisotropy, black_border)), the distances bit for
  bit, so the radius at each skeleton voxel is dist[skeleton].  numpy in gives numpy out; a torch CUDA
  tensor (or any __cuda_array_interface__ array) gives torch CUDA tensors computed on the current stream
  without a host synchronisation: the whole thinning is one cooperative kernel.  A weight that is not
  finite and > 0 is a ValueError, an unsupported dtype or number of dimensions a TypeError; a host array
  that does not fit on the GPU raises EDTError with code ENOMEM (there is no chunked path).  Device memory
  beyond the input and the outputs: 12 bytes per voxel for volumes of even sides (8 with
  return_distance=True)."""
  name = "skeletonize"
  if not isinstance(return_distance, (bool, np.bool_)):
    raise TypeError("%s: return_distance must be True or False, got %r" % (name, return_distance))
  v = _Volume(name, labels, stacked, (2, 3), device)
  try:
    nbytes = _nearest_label_bytes(v.dtype)
  except TypeError:
    raise TypeError("%s: unsupported label dtype %s: labels must be an integer or bool dtype"
                    % (name, v.dtype)) from None
  v.set_weights(anisotropy)
  skel = v.empty("bool")
  dist = v.empty("float32") if return_distance else None
  if v.size:
    _check(_lib().edtb200_skeletonize(v.ptr, nbytes, *v.geometry, int(bool(black_border)), v.flags, v.ptr_of(skel),
                                      v.ptr_of(dist), *v.where))
  return (skel, dist) if return_distance else skel


# ---------------------------------------------------------------------------------------
# shortest-path distances inside each label from seed voxels (edtb200_geodesic)
# ---------------------------------------------------------------------------------------

def _integer_bytes(dtype, what, name="geodesic_distance"):
  """Width of a numpy or torch bool / integer dtype of 1, 2, 4 or 8 bytes; TypeError for anything else."""
  try:
    return _nearest_label_bytes(dtype)
  except TypeError:
    raise TypeError("%s: unsupported %s dtype %s: it must be an integer or bool dtype"
                    % (name, what, dtype)) from None


def geodesic_distance(labels, seeds, anisotropy=None, *, return_indices=False, stacked=False, device=0):
  """Geodesic distance: the length of the shortest path from a seed to each voxel that stays inside the
  voxel's own label, on the GPU.

  Definition.  Volumes are x-fastest, as for edt(): x is the last axis of a C-ordered array and the first of
  an F-ordered one; coordinates are taken within one volume.
    graph     every voxel with a non-zero label is a node; two nodes are joined when they are 26-neighbours
              (2-D: 8, 1-D: 2) with the same label.  Label 0 and the outside of the volume cannot be crossed
              (there is no black_border).  A step (dx, dy, dz), each in {-1, 0, 1}, has the length
              sqrt((dx*wx)^2 + (dy*wy)^2 + (dz*wz)^2): each weight rounded to float32 (as the C ABI takes
              it) and promoted to double, the squares summed in double in the order x, y, z, the square root
              correctly rounded.
    seeds     a voxel is a seed when its seed value and its label are both non-zero; seeds on background are
              ignored.
    distance  D is the least fixed point of D[v] = min(D[v], fl64(D[u] + w(u, v))) over the graph neighbours
              u of v, from 0 on the seeds and +inf elsewhere -- exactly what Dijkstra computes in double
              (scipy.sparse.csgraph.dijkstra(G, indices=seeds, min_only=True) on this graph).  The result is
              float32(D), rounded once to nearest; label-0 voxels and voxels with no seed in their component
              are +inf.
    indices   with return_indices=True, S[v] is the least linear seed index c (x-fastest within the volume)
              with a tight path c = u0 .. uk = v, every step satisfying D[u_{i+1}] == fl64(D[u_i] + w): the
              seed v is reached from first, ties going to the least index, independent of any evaluation order.
  The result equals this definition bit for bit on every run.

  Examples.  A straight corridor: D is the number of steps times the step's weight,
      labels = np.zeros((3, 9), np.uint8); labels[1, 1:8] = 1
      seeds = np.zeros((3, 9), bool); seeds[1, 1] = True
      geodesic_distance(labels, seeds, (1.0, 0.5))[1, 1:8]  ->  [0, 0.5, 1, 1.5, 2, 2.5, 3]
  and +inf everywhere off the corridor.  An L-shaped corridor, where D is larger than the edt:
      labels = np.zeros((5, 5), np.uint8); labels[0, :] = 1; labels[:, 4] = 1
      seeds = np.zeros((5, 5), bool); seeds[0, 0] = True
      geodesic_distance(labels, seeds)[4, 4]  ->  np.float32(6 + np.sqrt(2)) = 7.4142137,
  three steps along the top, one diagonal step across the corner and three down, where the straight line
  is sqrt(32) = 5.656854.
  Seed splitting of touching objects: every voxel of a mask gets the marker it reaches first without
  leaving the mask (-1 indices, where no marker is reachable, masked to 0):
      dist, idx = geodesic_distance(mask, markers != 0, return_indices=True)
      split = np.where(idx[0] >= 0, markers[tuple(idx)], 0)

  Input and output.  `labels`: bool or integer dtypes of 1, 2, 4 or 8 bytes (float labels are a TypeError),
  1-D to 3-D, or with stacked=True 2-D to 4-D whose slowest axis in memory indexes same-shaped volumes, as
  edt(stacked=True); the result equals np.stack of the per-volume calls.  `seeds`: bool or integer dtypes (a
  TypeError otherwise) of the labels' shape (a ValueError otherwise); it is read in the labels' memory
  order, copied into it where its own differs, and moved to the labels' GPU when they are device-resident.
  `anisotropy`: one weight per volume axis, each finite and > 0 (a ValueError otherwise).  Returns `dist`,
  float32 with the input's shape and memory order, or with return_indices=True `(dist, indices)`, indices
  int32 of shape (vnd,) + labels.shape in scipy's return_indices layout (indices[k] is the coordinate along
  array axis k, each plane in the input's memory order, within each voxel's own volume for a stack), as
  feature_transform returns them, -1 in every plane where dist is +inf.  numpy in gives numpy out; a torch
  CUDA tensor (or any __cuda_array_interface__ array) gives torch CUDA tensors computed on the current stream
  without a host synchronisation: each phase is one cooperative kernel.  A host array that does not fit on
  the GPU raises EDTError with code ENOMEM (there is no chunked path).

  Cost.  The GPU relaxes 8x8x8 tiles (2-D 16x16, 1-D 256) in rounds, each round re-relaxing the tiles whose
  halo changed; the number of rounds grows with how often shortest paths turn across tile boundaries -- a
  handful for a convex object, thousands for a maze.  Device memory beyond the input and the outputs: 8 bytes
  per voxel for D, 8 more with return_indices, and 12 bytes per tile."""
  name = "geodesic_distance"
  if not isinstance(return_indices, (bool, np.bool_)):
    raise TypeError("%s: return_indices must be True or False, got %r" % (name, return_indices))
  v = _Volume(name, labels, stacked, (1, 3), device)
  nbytes = _integer_bytes(v.dtype, "label")
  sd = _device_array(seeds)
  if v.on_device:
    import torch
    sd = torch.as_tensor(seeds if sd is None else sd, device=v.arr.device)
  elif sd is not None:
    raise TypeError("%s: seeds are a GPU array but labels are a host array; pass both on the same side" % name)
  else:
    sd = np.asarray(seeds)
  seed_bytes = _integer_bytes(sd.dtype, "seed")
  if tuple(sd.shape) != v.shape:
    raise ValueError("%s: seeds must have the labels' shape %s, got %s" % (name, v.shape, tuple(sd.shape)))
  v.set_weights(anisotropy)
  # the seeds in the labels' memory order
  if not v.on_device:
    sd = np.asfortranarray(sd) if v.fortran else np.ascontiguousarray(sd)
  elif v.fortran:
    back = tuple(range(v.nd - 1, -1, -1))
    sd = sd.permute(*back).contiguous().permute(*back)
  else:
    sd = sd.contiguous()
  dist = v.empty("float32")
  planes = v.empty("int32", planes=v.vnd) if return_indices else None
  if v.size:
    ptrs = v.plane_ptrs(planes) if return_indices else None
    _check(_lib().edtb200_geodesic(v.ptr, nbytes, v.ptr_of(sd), seed_bytes, *v.geometry, v.flags, v.ptr_of(dist),
                                   ptrs, *v.where))
  if not return_indices:
    return dist
  return dist, planes


# ---------------------------------------------------------------------------------------
# marker-controlled flooding of an altitude image inside each label (edtb200_watershed)
# ---------------------------------------------------------------------------------------

def _like_volume(v, data, what, name):
  """`data` on the side and in the memory order of the volume `v`: host data is moved to v's GPU when v is
  device-resident; device data with a host volume is a TypeError; a shape other than v's a ValueError."""
  t = _device_array(data)
  if v.on_device:
    import torch
    x = torch.as_tensor(data if t is None else t, device=v.arr.device)
  elif t is not None:
    raise TypeError("%s: %s is a GPU array but the volume is a host array; pass every array on the same side"
                    % (name, what))
  else:
    x = np.asarray(data)
  if tuple(x.shape) != v.shape:
    raise ValueError("%s: %s must have the volume's shape %s, got %s" % (name, what, v.shape, tuple(x.shape)))
  return x


def _in_volume_order(v, x):
  """x (already on v's side and of v's shape) in v's memory order, contiguous."""
  if not v.on_device:
    return np.asfortranarray(x) if v.fortran else np.ascontiguousarray(x)
  if v.fortran:
    back = tuple(range(v.nd - 1, -1, -1))
    return x.permute(*back).contiguous().permute(*back)
  return x.contiguous()


def _real_float32(x, name):
  """x as float32 (once, where it is another real dtype); a TypeError for complex and non-numeric dtypes."""
  if isinstance(x, np.ndarray):
    if x.dtype.kind not in "biuf":
      raise TypeError("%s: unsupported image dtype %s: it must be a real dtype" % (name, x.dtype))
    return x if x.dtype == np.float32 else x.astype(np.float32)
  import torch
  if x.dtype.is_complex:
    raise TypeError("%s: unsupported image dtype %s: it must be a real dtype" % (name, x.dtype))
  return x if x.dtype == torch.float32 else x.to(torch.float32)


def watershed(image, markers, labels=None, *, connectivity=1, return_level=False, stacked=False, device=0):
  """Watershed: marker-controlled flooding of an altitude image inside each label, on the GPU.  The usual
  split of touching objects is
      dist = edt(mask); markers = <one marker per maximum of dist>; watershed(-dist, markers, mask)
  (skimage.segmentation.watershed's mask=m is labels=m here: flooding stays inside each label).

  Definition.  Volumes are x-fastest, as for edt(): x is the last axis of a C-ordered array and the first of
  an F-ordered one.
    graph     every voxel with a non-zero label is a node (labels=None: every voxel, all with one label); two
              nodes are joined when they are neighbours under `connectivity` with the same label: an offset
              counts when at most `connectivity` of its components are non-zero (3-D 1/2/3: 6/18/26
              neighbours, 2-D 1/2: 4/8), as in scipy and skimage.  Label 0 and the outside of the volume
              cannot be crossed.
    altitude  f = image as float32; NaN is read as +inf and -0.0 as +0.0; +inf and -inf are valid altitudes.
    seeds     a voxel is a seed when its marker and its label are both non-zero; markers on label 0 are
              ignored.  Marker values are compared as unsigned integers of the markers' width.
    level     L is the least fixed point of L[v] = min(L[v], max(f[v], L[u])) over the graph neighbours u of
              v, from f on the seeds and +inf elsewhere: the lowest flood level at which water from some seed
              reaches v.  It is exact: min and max round nothing.
    result    an edge u -> v is tight when v is not a seed and L[v] == max(f[v], L[u]).  W = the marker on
              the seeds; elsewhere W[v] is the least marker m with a tight path from a seed of marker m to v
              whose voxels after the first are non-seeds, and 0 where there is none and on label 0.
  The result equals this definition bit for bit on every run, whatever order the GPU floods in.  Ties: a
  voxel reached at the same level from two markers goes to the smaller marker value, and plateaus are not
  split by distance.  skimage breaks such ties by the order of its queue, so the two agree on every voxel
  but the tied ones.

  Examples.  Two basins in 1-D split at the ridge between them:
      image = np.array([0, 3, 1, 5, 2, 0], np.float32)
      markers = np.array([1, 0, 0, 0, 0, 2], np.uint8)
      watershed(image, markers)  ->  [1, 1, 1, 1, 2, 2]
  (the ridge voxel is reached at level 5 from both sides and goes to the smaller marker), and
      watershed(image, markers, return_level=True)[1]  ->  [0, 3, 3, 5, 2, 0]
  (the pit of altitude 1 fills up to the 3 that water from marker 1 must pass).
  Two touching discs split at the neck:
      dist = edt(mask); split = watershed(-dist, markers, mask)

  Input and output.  `image`: any real dtype, 1-D to 3-D, or with stacked=True 2-D to 4-D whose slowest axis
  in memory indexes same-shaped volumes, as edt(stacked=True); the result equals np.stack of the per-volume
  calls.  Anything but float32 is converted to float32 once (float64 altitudes that differ only below
  float32's precision become equal, and may tie).  `markers`: bool or integer dtypes of 1, 2, 4 or 8 bytes.
  `labels`: None, or bool or integer dtypes of 1, 2, 4 or 8 bytes (float labels are a TypeError).  Every
  array has the same shape (a ValueError otherwise) and is read in the memory order of `labels` (of `image`
  when labels is None), copied into it where its own differs.  `connectivity`: an int from 1 to the number
  of volume axes.  Returns W in the markers' dtype (bool markers give uint8) with the volume's shape and
  memory order, or with return_level=True `(W, level)`, level float32 (+inf on label 0 and where no seed
  is reachable at a finite level).  numpy in gives numpy out; a torch CUDA tensor (or any
  __cuda_array_interface__ array) gives torch CUDA tensors computed on the current stream without a host
  synchronisation: each phase is one cooperative kernel; host arrays passed with it are moved to its GPU.
  A host array that does not fit on the GPU raises EDTError with code ENOMEM (there is no chunked path).

  Cost.  The GPU floods 8x8x8 tiles (2-D 16x16, 1-D 256) in rounds, each round re-relaxing the tiles whose
  halo changed, first for the level and then for the markers over the tight edges.  Device memory beyond
  the inputs and the outputs: 4 bytes per voxel for the level, 4 for the markers (8 for 8-byte markers), and
  12 bytes per tile."""
  name = "watershed"
  if not isinstance(return_level, (bool, np.bool_)):
    raise TypeError("%s: return_level must be True or False, got %r" % (name, return_level))
  if isinstance(connectivity, (bool, np.bool_)) or not isinstance(connectivity, (int, np.integer)):
    raise TypeError("%s: connectivity must be an int, got %r" % (name, connectivity))
  ref = image if labels is None else labels
  v = _Volume(name, ref, stacked, (1, 3), device)
  if not 1 <= connectivity <= v.vnd:
    raise ValueError("%s: connectivity must be 1 to %d for %d-D volumes, got %d" % (name, v.vnd, v.vnd, connectivity))
  nbytes = 0 if labels is None else _integer_bytes(v.dtype, "label", name)
  mk = _like_volume(v, markers, "markers", name)
  marker_bytes = _integer_bytes(mk.dtype, "marker", name)
  img = v.arr if labels is None else _like_volume(v, image, "image", name)
  img = _in_volume_order(v, _real_float32(img, name))
  mk = _in_volume_order(v, mk)
  v.set_weights(None, positive=False)
  # W in the markers' dtype, bool as uint8
  if v.on_device:
    import torch
    out_dtype = "uint8" if mk.dtype == torch.bool else str(mk.dtype).split(".")[-1]
  else:
    out_dtype = "uint8" if mk.dtype == np.bool_ else mk.dtype.name
  out = v.empty(out_dtype)
  level = v.empty("float32") if return_level else None
  if v.size:
    vnd, sx, sy, sz, count = v.geometry[:5]
    _check(_lib().edtb200_watershed(None if labels is None else v.ptr, nbytes, v.ptr_of(mk), marker_bytes,
                                    v.ptr_of(img), vnd, sx, sy, sz, count, int(connectivity), v.flags, v.ptr_of(out),
                                    v.ptr_of(level), *v.where))
  return (out, level) if return_level else out


# ---------------------------------------------------------------------------------------
# connected components and extended maxima (edtb200_connected_components, edtb200_extended_maxima)
# ---------------------------------------------------------------------------------------

_COMPONENTS_GRAPH = """
    graph      every voxel with a non-zero label is a node (extended_maxima with labels=None: every voxel, all
               with one label); two nodes are joined when they are neighbours under `connectivity` with the
               same label: an offset counts when at most `connectivity` of its components are non-zero (3-D
               1/2/3: 6/18/26 neighbours, 2-D 1/2: 4/8), as in scipy and skimage.  Label 0 and the outside of
               the volume cannot be crossed.
    numbering  each component is numbered 1..n in increasing order of its least voxel index in memory order,
               everything else 0.  For a C-ordered array this is scipy.ndimage.label's numbering; for an
               F-ordered one it is that numbering of a.T, transposed back."""

_COMPONENTS_IO = """
  Input and output.  Volumes are x-fastest, as for edt(): x is the last axis of a C-ordered array and the first
  of an F-ordered one.  1-D to 3-D arrays, or with stacked=True 2-D to 4-D whose slowest axis in memory indexes
  same-shaped volumes; each volume is numbered on its own from 1, so the result equals np.stack of the
  per-volume calls bit for bit.  Labels are bool or integer dtypes of 1, 2, 4 or 8 bytes (float labels are a
  TypeError).  The result is int32 when each volume has fewer than 2^31 voxels, else int64, with the volume's
  shape and memory order.  numpy in gives numpy out; a torch CUDA tensor (or any __cuda_array_interface__
  array) gives a torch CUDA tensor computed on the current stream without a host synchronisation.  A host
  array that does not fit on the GPU raises EDTError with code ENOMEM (there is no chunked path)."""


def _components_out(v):
  """The result of a components call on the volume v (after set_weights): int32 when each volume has fewer
  than 2^31 voxels, else int64; and its width."""
  sx, sy, sz = v.geometry[1:4]
  out_bytes = 4 if sx * sy * sz < (1 << 31) else 8
  return v.empty("int32" if out_bytes == 4 else "int64"), out_bytes


def _connectivity(name, connectivity, v):
  if isinstance(connectivity, (bool, np.bool_)) or not isinstance(connectivity, (int, np.integer)):
    raise TypeError("%s: connectivity must be an int, got %r" % (name, connectivity))
  if not 1 <= connectivity <= v.vnd:
    raise ValueError("%s: connectivity must be 1 to %d for %d-D volumes, got %d" % (name, v.vnd, v.vnd, connectivity))
  return int(connectivity)


_CONNECTED_COMPONENTS_DOC = ("""Connected components of every label, numbered, on the GPU: cc3d.connected_components, or
  scipy.ndimage.label applied to each label at once.

  Definition.""" + _COMPONENTS_GRAPH + """
  The default connectivity=1 is scipy's and watershed's; cc3d's default of 26 is connectivity=3.

  Examples (2-D, C order):
      connected_components(np.array([[1, 1, 0, 2], [0, 1, 0, 2], [3, 0, 0, 1]]))
        ->  [[1, 1, 0, 2], [0, 1, 0, 2], [3, 0, 0, 4]]
      connected_components(np.array([[1, 0], [0, 1]]))                   ->  [[1, 0], [0, 2]]
      connected_components(np.array([[1, 0], [0, 1]]), connectivity=2)   ->  [[1, 0], [0, 1]]
""" + _COMPONENTS_IO + """

  Cost.  Union-find whose cost does not grow with a component's diameter: a tile pass in shared memory, a
  border pass of lock-free unions in global memory, a flatten pass, a prefix sum and a number pass.  Device
  memory beyond the input and the output: 4 bytes per voxel of parents and the scan's scratch.""")


def connected_components(labels, *, connectivity=1, stacked=False, device=0):
  name = "connected_components"
  v = _Volume(name, labels, stacked, (1, 3), device)
  conn = _connectivity(name, connectivity, v)
  nbytes = _integer_bytes(v.dtype, "label", name)
  v.set_weights(None, positive=False)
  out, out_bytes = _components_out(v)
  if v.size:
    vnd, sx, sy, sz, count = v.geometry[:5]
    _check(_lib().edtb200_connected_components(v.ptr, nbytes, vnd, sx, sy, sz, count, conn, v.flags, v.ptr_of(out),
                                               out_bytes, *v.where))
  return out


connected_components.__doc__ = _CONNECTED_COMPONENTS_DOC


_EXTENDED_MAXIMA_DOC = ("""Extended maxima: the regional maxima of the h-maxima transform (Soille's EMAX_h, MATLAB's imextendedmax),
  numbered, on the GPU.  They are the markers of the usual split of touching objects:
      dist = edt(mask); markers = extended_maxima(dist, h, mask); watershed(-dist, markers, mask)
  and extended_maxima(-f, h) gives the minima markers of an unseeded watershed(f, ...) (NaN, read as -inf here
  and as +inf by watershed, never becomes a marker).

  Definition.""" + _COMPONENTS_GRAPH + """
    image      f = image as float32, NaN read as -inf and -0.0 as +0.0.  `h` is a finite real >= 0 (a
               ValueError otherwise); m = fl32(fl64(f) - fl64(h)), -0.0 read as +0.0, so m <= f and h = 0
               gives m = f.
    R          the least fixed point of R[v] = max(R[v], min(f[v], R[u])) over the joined neighbours u of v,
               from m: the reconstruction by dilation of m under f.  It is exact: min and max round nothing.
    plateau    a component of the graph restricted to the edges with R[u] == R[v]; it is a maximum when no
               node in it has a joined neighbour with a larger R, and its R is not -inf.
    result     the maximum plateaus, numbered as above.
  When f - h is exact in float32, a peak survives exactly when its dynamic -- its height above the highest
  pass to a higher voxel of its label -- exceeds h.  skimage.morphology.h_maxima keeps dynamics >= h and
  returns only the top plateau of each survivor; here a peak whose dynamic equals h is merged, and a survivor
  is marked by the whole plateau of R at its top, which reaches h below the peak.

  Examples (1-D):
      extended_maxima(np.array([0, 3, 1, 5, 2, 0.]))         ->  [0, 1, 0, 2, 0, 0]   (h=1.9 the same)
      extended_maxima(np.array([0, 3, 1, 5, 2, 0.]), h=2)    ->  [0, 0, 0, 1, 0, 0]   (the peak at 1 has dynamic 2)
      extended_maxima(np.array([0, 4, 3.5, 4, 0.]), h=0.4)   ->  [0, 1, 0, 2, 0]
      extended_maxima(np.array([0, 4, 3.5, 4, 0.]), h=0.5)   ->  [0, 1, 1, 1, 0]
""" + _COMPONENTS_IO + """  The image may be any real dtype and is converted
  to float32 once; it is read in the memory order of `labels` (of `image` when labels is None).

  Cost.  With h = 0, R = f and the plateaus are labelled by the union-find passes of connected_components with
  the key (label, R), then a mark pass drops the plateaus with a larger neighbour.  With h > 0, R first comes
  from watershed's level phase on negated values, which floods 8x8x8 tiles in rounds (its cost grows with the
  distance R has to travel).  Device memory beyond the inputs and the output: 4 bytes per voxel of parents and
  the scan's scratch, and with h > 0 another 4 + 4 bytes per voxel and 12 bytes per tile.""")


def extended_maxima(image, h=0.0, labels=None, *, connectivity=1, stacked=False, device=0):
  name = "extended_maxima"
  if isinstance(h, (bool, np.bool_)) or not isinstance(h, (int, float, np.integer, np.floating)):
    raise TypeError("%s: h must be a real number, got %r" % (name, h))
  if not (math.isfinite(float(h)) and float(h) >= 0.0):
    raise ValueError("%s: h must be finite and >= 0, got %r" % (name, h))
  ref = image if labels is None else labels
  v = _Volume(name, ref, stacked, (1, 3), device)
  conn = _connectivity(name, connectivity, v)
  nbytes = 0 if labels is None else _integer_bytes(v.dtype, "label", name)
  img = v.arr if labels is None else _like_volume(v, image, "image", name)
  img = _in_volume_order(v, _real_float32(img, name))
  v.set_weights(None, positive=False)
  out, out_bytes = _components_out(v)
  if v.size:
    vnd, sx, sy, sz, count = v.geometry[:5]
    _check(_lib().edtb200_extended_maxima(None if labels is None else v.ptr, nbytes, v.ptr_of(img), vnd, sx, sy, sz,
                                          count, float(h), conn, v.flags, v.ptr_of(out), out_bytes, *v.where))
  return out


extended_maxima.__doc__ = _EXTENDED_MAXIMA_DOC


# ---------------------------------------------------------------------------------------
# hole filling and dust removal (edtb200_fill_holes, edtb200_dust)
# ---------------------------------------------------------------------------------------

_HOLES_IO = """
  Input and output.  Volumes are x-fastest, as for edt(): x is the last axis of a C-ordered array and the first
  of an F-ordered one.  1-D to 3-D arrays, or with stacked=True 2-D to 4-D whose slowest axis in memory indexes
  same-shaped volumes, each with its own faces, so the result equals np.stack of the per-volume calls.  Labels
  are bool or integer dtypes of 1, 2, 4 or 8 bytes and compare by their bits (float labels are a TypeError);
  volumes of 2^32 voxels or more raise EDTError with code ELIMIT.  The result has the input's dtype, shape and
  memory order.  numpy in gives numpy out; a torch CUDA tensor (or any __cuda_array_interface__ array) gives a
  torch CUDA tensor computed on the current stream without a host synchronisation.  A host array that does not
  fit on the GPU raises EDTError with code ENOMEM (there is no chunked path)."""


def _size_bound(name, what, value):
  if isinstance(value, (bool, np.bool_)) or not isinstance(value, (int, np.integer)):
    raise TypeError("%s: %s must be an int, got %r" % (name, what, value))
  if value < 0:
    raise ValueError("%s: %s must be >= 0, got %d" % (name, what, value))
  return min(int(value), (1 << 63) - 1)


_FILL_HOLES_DOC = ("""Fill the holes of every label, on the GPU: scipy.ndimage.binary_fill_holes for every label at once,
  fill_voids / kimimaro's fill_holes, porespy's blind pores.

  Definition.  The graph and `connectivity` are connected_components': an offset counts when at most
  `connectivity` of its components are non-zero (3-D 1/2/3: 6/18/26 neighbours, 2-D 1/2: 4/8).
    background component  a component of the label-0 voxels under `connectivity`.
    open                  it has a voxel on a face of its volume.
    bordering labels      the non-zero labels of the voxels that neighbour it under `connectivity`.
    hole of L             a background component that is not open, whose only bordering label is L, and, when
                          max_size is given, that has at most max_size voxels.
    result                the labels with every hole of L set to L; everything else unchanged.
  For a bool mask this is exactly scipy.ndimage.binary_fill_holes(mask, generate_binary_structure(ndim,
  connectivity)).  Per-label enclosure is fill_holes(labels == L): it fills L's mask whatever else L encloses.
  In one multi-label call a background gap bordered by two labels stays 0: the gap between a cell (label 1) and
  a nucleus (label 2) inside it borders both and is not filled, while a hole inside the nucleus becomes 2.

  Examples (C order):
      fill_holes(np.array([1, 0, 0, 1, 0]))                              ->  [1, 1, 1, 1, 0]
      fill_holes(np.array([2, 0, 1, 0, 1]))                              ->  [2, 0, 1, 1, 1]
      fill_holes(np.array([[0, 1, 0], [1, 0, 1], [0, 1, 0]]))            ->  [[0, 1, 0], [1, 1, 1], [0, 1, 0]]
      fill_holes(np.array([[0, 1, 0], [1, 0, 1], [0, 1, 0]]), connectivity=2)   ->  unchanged: the middle 0
        is joined to the corners, which are on the faces
      fill_holes(np.array([1, 0, 0, 1]), max_size=1)                     ->  [1, 0, 0, 1]

  `max_size`: None, or an int >= 0.  `return_fill_count=True` returns (result, filled): the number of voxels
  filled, an int for one volume (for device input that int waits for the GPU) and an int64 array with one entry
  per volume for a stack (a torch CUDA tensor for device input, without a host synchronisation).""" + _HOLES_IO + """

  Cost.  The union-find passes of connected_components on the background, a tally pass that points every
  background voxel at its root, sets OPEN and MIXED bits and claims the bordering labels at the root, and an
  apply pass.  Device memory beyond the input and the output: 4 bytes per voxel of parents, 4 bytes per voxel
  of claims (8 for 8-byte labels) and 1 byte per voxel of state, and with max_size another 4 bytes per voxel of
  sizes.""")


def fill_holes(labels, *, connectivity=1, max_size=None, return_fill_count=False, stacked=False, device=0):
  name = "fill_holes"
  if not isinstance(return_fill_count, (bool, np.bool_)):
    raise TypeError("%s: return_fill_count must be True or False, got %r" % (name, return_fill_count))
  bound = -1 if max_size is None else _size_bound(name, "max_size", max_size)
  v = _Volume(name, labels, stacked, (1, 3), device)
  conn = _connectivity(name, connectivity, v)
  nbytes = _integer_bytes(v.dtype, "label", name)
  v.set_weights(None, positive=False)
  out = v.empty()
  count = v.geometry[4]
  counts = None
  if return_fill_count:
    if v.on_device:
      import torch
      counts = torch.zeros(count, dtype=torch.int64, device=v.arr.device)
    else:
      counts = np.zeros(count, np.int64)
  if v.size:
    vnd, sx, sy, sz = v.geometry[:4]
    _check(_lib().edtb200_fill_holes(v.ptr, nbytes, vnd, sx, sy, sz, count, conn, bound, v.flags, v.ptr_of(out),
                                     v.ptr_of(counts), *v.where))
  if not return_fill_count:
    return out
  return out, (counts if stacked else int(counts[0]) if count else 0)


fill_holes.__doc__ = _FILL_HOLES_DOC


_DUST_DOC = ("""Remove the small components of every label, on the GPU: cc3d.dust, kimimaro's dust_threshold,
  skimage.morphology.remove_small_objects for every label at once.

  Definition.  The components are connected_components': voxels of the same non-zero label joined under
  `connectivity` (an offset counts when at most `connectivity` of its components are non-zero).  Every voxel of
  a component of FEWER than `threshold` voxels is set to 0, as in cc3d; a component of exactly `threshold`
  voxels is kept.  With invert=True only the components of fewer than `threshold` voxels are kept.  skimage
  versions disagree on whether their size bound is strict; this is the definition here.  cc3d's default of 26
  neighbours is connectivity=3.

  Examples (C order):
      dust(np.array([1, 1, 0, 2, 0, 1]), 2)                   ->  [1, 1, 0, 0, 0, 0]
      dust(np.array([1, 1, 0, 2, 0, 1]), 2, invert=True)      ->  [0, 0, 0, 2, 0, 1]
      dust(np.array([[1, 0], [0, 1]]), 2)                     ->  [[0, 0], [0, 0]]
      dust(np.array([[1, 0], [0, 1]]), 2, connectivity=2)     ->  [[1, 0], [0, 1]]

  `threshold`: an int >= 0 (0 keeps everything).""" + _HOLES_IO + """

  Cost.  The union-find passes of connected_components, a tally pass that adds every voxel to its root's size,
  and an apply pass.  Device memory beyond the input and the output: 4 bytes per voxel of parents and 4 bytes
  per voxel of sizes.""")


def dust(labels, threshold, *, connectivity=1, invert=False, stacked=False, device=0):
  name = "dust"
  threshold = _size_bound(name, "threshold", threshold)
  if not isinstance(invert, (bool, np.bool_)):
    raise TypeError("%s: invert must be True or False, got %r" % (name, invert))
  v = _Volume(name, labels, stacked, (1, 3), device)
  conn = _connectivity(name, connectivity, v)
  nbytes = _integer_bytes(v.dtype, "label", name)
  v.set_weights(None, positive=False)
  out = v.empty()
  if v.size:
    vnd, sx, sy, sz, count = v.geometry[:5]
    _check(_lib().edtb200_dust(v.ptr, nbytes, vnd, sx, sy, sz, count, conn, threshold, int(bool(invert)), v.flags,
                               v.ptr_of(out), *v.where))
  return out


dust.__doc__ = _DUST_DOC


# ---------------------------------------------------------------------------------------
# the k nearest distinct labels of every voxel within a distance (edtb200_nearest_labels)
# ---------------------------------------------------------------------------------------

FLAG_NEAREST_SQUARED = 32      # EDTB200_NEAREST_SQUARED


def _nearest_label_bytes(dtype):
  """Label width of a numpy or torch integer / bool dtype; TypeError for anything else (floats included)."""
  if isinstance(dtype, np.dtype):
    if dtype == np.bool_ or (dtype.kind in "iu" and dtype.itemsize in (1, 2, 4, 8)):
      return dtype.itemsize
  else:
    import torch
    nbytes = _torch_label_bytes(torch).get(dtype)
    if nbytes is not None:
      return nbytes
  raise TypeError("nearest_labels: labels must be an integer or bool dtype, got %s" % dtype)


def nearest_labels(labels, max_distance, anisotropy=None, *, k=2, squared=False, stacked=False, device=0):
  """The k nearest distinct labels of every voxel within max_distance, and how far away each is.

  Returns (distances, nearest): float32 distances and labels of the input's dtype, both of shape
  (k,) + labels.shape.  Entry q of a voxel is plane q, and each plane has the input's memory order (the
  layout of feature_transform's indices).  Entries come in ascending distance; ties are ordered by the
  label read as an unsigned integer of its width.  Where fewer than k labels lie within max_distance the
  missing entries are distance +inf and label 0.  A labelled voxel's entry 0 is (0, its own label).

  Definition.  Volumes are x-fastest: for C-ordered input the last axis is x, as for edt().  Every voxel
  with a non-zero label is a site of that label; label 0 is background, whose voxels ask the query but are
  never sites (there is no border term, so black_border does not apply).  For a voxel p and a label M,

      D_M(p) = parabolic_erode(np.where(labels == M, 0, np.inf), anisotropy)[p]      (bit for bit)

  -- one pass per axis in the order x, y, z, each candidate fl32(fl64(w2 * (i-j)^2) + fl64(g(j))) with
  w2 = float32(w * w).  With integer weights and values below 2^24 it is exactly the squared Euclidean
  distance from p to the nearest voxel of M.  B is the largest float32 with float64(B) <= max_distance^2
  (the cut of the bounded transforms); only labels with D_M(p) <= B count.
    values  the k distances of p are the k smallest D_M(p) over the distinct counted labels, exactly;
            squared=True returns D, otherwise np.sqrt of it in float32 (correctly rounded, as edt).
    labels  each pass keeps per voxel the k least (value, label) pairs with distinct labels: the X pass
            sees the voxel itself at 0 and each labelled voxel j != i of its row at fl32(w2 * (i-j)^2),
            every later pass its own row's list and row j's entries each raised to
            fl32(fl64(w2 * (i-j)^2) + fl64(v)); a label keeps its least value, ties go to the smaller
            unsigned label, pairs above B are dropped.  So the labels are the k least (D_M(p), M) pairs
            wherever rounding merges no two candidates -- always, for integer weights and values below
            2^24; otherwise a label can differ only among labels whose value equals the k-th value.
  The values are exact although each pass keeps only k entries: a label dropped at an intermediate voxel
  had k others no larger there, and each pass adds w2 * d^2 and rounds, which is monotone.

  Worked use: the U-Net weight map of touching cells, w(p) = w0 * exp(-(d1 + d2)^2 / (2 sigma^2)) on the
  background, d1 and d2 the distances to the nearest and second-nearest cell:
      (d, _) = nearest_labels(cells, max_distance=3 * sigma, k=2)
      w = np.where(cells == 0, w0 * np.exp(-(d[0] + d[1]) ** 2 / (2 * sigma ** 2)), 0)
  (+inf beyond max_distance makes the weight 0 there, where it is below w0 * exp(-4.5) anyway.)  Contacts
  between segments within r are the voxels where nearest[1] != 0 at max_distance=r, and Voronoi boundaries
  between instances lie where d[1] - d[0] is small.

  Arguments.  `labels`: 1-D to 3-D, or with stacked=True a 2-D to 4-D array whose slowest axis in memory
  indexes same-shaped volumes, each on its own with one launch per pass for all of them.  Integer and bool
  dtypes only: float labels raise TypeError.  `max_distance` must be finite and >= 0 (ValueError): each
  pass costs O(R) per voxel, R = max_distance / w rows, and R may not exceed 256 rows (EDTError ELIMIT).
  `anisotropy`: one weight per volume axis, finite and > 0.  `k`: 1 to 4.  numpy in gives numpy out, staged
  through the GPU whole (a host array that does not fit raises EDTError with code ENOMEM; there is no
  chunked path); a torch CUDA tensor (or any __cuda_array_interface__ array) gives torch CUDA tensors
  computed on the current stream.  Device memory beyond the labels and the outputs: k * (4 + itemsize)
  bytes per voxel in 2-D and 3-D, none in 1-D.
  """
  name = "nearest_labels"
  if isinstance(k, (bool, np.bool_)) or not isinstance(k, (int, np.integer)) or not 1 <= int(k) <= 4:
    raise ValueError("%s: k must be an integer from 1 to 4, got %r" % (name, k))
  k = int(k)
  d = float(max_distance)
  if not (d >= 0.0 and d != float("inf")):
    raise ValueError("%s: max_distance must be finite and zero or more, got %r" % (name, max_distance))
  v = _Volume(name, labels, stacked, (1, 3), device)
  nbytes = _nearest_label_bytes(v.dtype)
  v.set_weights(anisotropy)
  dist = v.empty("float32", planes=k)
  near = v.empty(planes=k)
  if v.size:
    flags = v.flags | (FLAG_NEAREST_SQUARED if squared else 0)
    _check(_lib().edtb200_nearest_labels(v.ptr, nbytes, *v.geometry, d, k, flags, v.ptr_of(dist), v.ptr_of(near),
                                         *v.where))
  return dist, near


# ---------------------------------------------------------------------------------------
# surface distances between two label volumes: Hausdorff distance, average surface distance and
# surface Dice (edtb200_surface_count, edtb200_surface_distances)
# ---------------------------------------------------------------------------------------

SurfaceDistances = collections.namedtuple("SurfaceDistances", "labels offsets values")
SurfaceDistances.__doc__ = """What surface_distances returns.  labels: the keys, in the caller's dtype;
offsets: int64, count * K * 2 + 1 entries, segment (volume * K + key) * 2 + direction from
values[offsets[s]] to values[offsets[s + 1]]; values: float32, each segment sorted ascending."""


def _surface_keys(labels, dtype):
  """labels= in the caller's dtype, checked: no 0 and no repeat."""
  keys = np.asarray(labels, dtype=dtype).reshape(-1)
  if np.any(keys == 0):
    raise ValueError("labels must not contain 0 (background)")
  raw = _label_view(keys)
  if raw is None:
    raise TypeError("unsupported label dtype %s" % dtype)
  if np.unique(raw).size != raw.size:
    raise ValueError("labels must be distinct")
  return keys


def _surface_run(a, b, anisotropy, labels, stacked, device, max_device_bytes):
  """The sorted surface distances of a against b: (keys, offsets, values, count, host) with torch CUDA
  offsets and values.  Host arrays go up through torch, as expand_labels' do."""
  import torch
  va, vb = (_Volume("surface_distances", x, stacked, device=device) for x in (a, b))
  host = not va.on_device and not vb.on_device
  if host:
    shape, dtype, nd = va.arr.shape, va.arr.dtype, va.nd
    if vb.arr.shape != shape:
      raise ValueError("a and b must have one shape, got %s and %s" % (shape, vb.arr.shape))
    if vb.arr.dtype != dtype:
      raise TypeError("a and b must have one dtype, got %s and %s" % (dtype, vb.arr.dtype))
    if _label_view(va.arr[:0]) is None:
      raise TypeError("unsupported label dtype %s" % dtype)
  else:
    if not va.on_device:
      va = _Volume(va.name, torch.as_tensor(va.arr, device=vb.arr.device), stacked)
    if not vb.on_device:
      vb = _Volume(vb.name, torch.as_tensor(vb.arr, device=va.arr.device), stacked)
    da, db = va.arr, vb.arr
    shape, nd = tuple(da.shape), da.dim()
    if tuple(db.shape) != shape:
      raise ValueError("a and b must have one shape, got %s and %s" % (shape, tuple(db.shape)))
    if db.dtype != da.dtype or db.device != da.device:
      raise TypeError("a and b must have one dtype and device, got %s on %s and %s on %s"
                      % (da.dtype, da.device, db.dtype, db.device))
    if _torch_label_bytes(torch).get(da.dtype) is None and da.dtype not in (torch.float32, torch.float64):
      raise TypeError("unsupported label dtype %s" % da.dtype)
    dtype = torch.empty(0, dtype=da.dtype).numpy().dtype
  if stacked:
    _stack_dims(nd)
  elif nd < 1 or nd > 3:
    raise TypeError("surface distances take 1-D to 3-D volumes, got %d-D" % nd)
  anisotropy = _weights(va.vnd, anisotropy)
  keys = None if labels is None else _surface_keys(labels, dtype)
  budget = 0 if max_device_bytes is None else _chunk_budget(max_device_bytes)
  if host:
    if np.prod(shape) == 0:
      count = (int(shape[0] if va.arr.flags.c_contiguous else shape[-1])) if stacked else 1
      keys = np.zeros(0, dtype) if keys is None else keys
      nseg = count * keys.size * 2
      return keys, torch.zeros(nseg + 1, dtype=torch.int64), torch.zeros(0, dtype=torch.float32), count, host
    if device_count() == 0:
      raise EDTError("edt_b200 error %d: no usable CUDA device; this library has no CPU fallback" % ECUDA, ECUDA)
    # host arrays go up through torch, as expand_labels' do
    dev = torch.device("cuda", int(device))
    va, vb = (_Volume(v.name, v.order().upload(dev), stacked) for v in (va, vb))
  # a's memory order decides the layout the C ABI reads; b is laid out the same way
  va.order()
  va.set_weights(anisotropy, positive=False, rule=None)
  rev = tuple(reversed(range(nd)))
  vb.arr = vb.arr.permute(*rev).contiguous().permute(*rev) if va.fortran else vb.arr.contiguous()
  (ta, nbytes), (tb, _) = va.labels(), vb.labels()
  vnd, sx, sy, sz, count, wx, wy, wz = va.geometry
  rtype = np.dtype("u%d" % ta.element_size())
  if keys is None:
    if ta.numel():
      raw = np.union1d(torch.unique(ta).cpu().numpy(), torch.unique(tb).cpu().numpy()).view(rtype)
    else:
      raw = np.zeros(0, rtype)
    raw = raw[raw != 0]
    keys = raw.view(dtype)[np.argsort(raw.view(dtype), kind="stable")]     # sorted by the caller's value
  raw_keys = (keys + 0 if keys.dtype.kind == "f" else keys).view(rtype)
  perm = np.argsort(raw_keys, kind="stable")             # the C ABI takes the keys ascending as raw bits
  sorted_keys = np.ascontiguousarray(raw_keys[perm])
  nkeys = keys.size
  nseg = count * nkeys * 2
  dev = ta.device
  counts = torch.zeros(nseg, dtype=torch.int64, device=dev)
  stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
  both = FLAG_LABELS_ON_DEVICE | FLAG_OUT_ON_DEVICE
  lib = _lib()
  _check(lib.edtb200_surface_count(ta.data_ptr(), tb.data_ptr(), ta.element_size(), vnd, sx, sy, sz, count,
                                   sorted_keys.ctypes.data, nkeys, both, counts.data_ptr(), dev.index, stream))
  offsets = torch.zeros(nseg + 1, dtype=torch.int64, device=dev)
  torch.cumsum(counts, 0, out=offsets[1:])
  total = int(offsets[-1].item())
  values = torch.empty(max(total, 1), dtype=torch.float32, device=dev)
  _check(lib.edtb200_surface_distances(
    ta.data_ptr(), tb.data_ptr(), ta.element_size(), vnd, sx, sy, sz, count, wx, wy, wz, sorted_keys.ctypes.data,
    nkeys, both, offsets.data_ptr(), values.data_ptr(), dev.index, budget, None, stream))
  values = values[:total]
  # Segment (v, r, d) of sorted key r is the caller's segment (v, perm[r], d).  One sort on
  # (segment << 32 | distance bits) -- non-negative floats order like their bits -- groups the
  # segments in the caller's order and sorts each ascending.
  new_of_old = (np.arange(count)[:, None, None] * nkeys + perm[None, :, None]) * 2 + np.arange(2)[None, None, :]
  new_of_old = torch.from_numpy(new_of_old.reshape(-1)).to(dev)
  seg_ids = torch.repeat_interleave(new_of_old, counts, output_size=total)
  key = (seg_ids << 32) | values.view(torch.int32).to(torch.int64)
  values = (torch.sort(key).values & 0xffffffff).to(torch.int32).view(torch.float32)
  new_counts = torch.zeros_like(counts)
  new_counts[new_of_old] = counts
  offsets = torch.zeros_like(offsets)
  torch.cumsum(new_counts, 0, out=offsets[1:])
  return keys, offsets, values, count, host


def surface_distances(a, b, anisotropy=None, *, labels=None, stacked=False, device=0, max_device_bytes=None):
  """The surface distances of two label volumes a (prediction) and b (reference) of one shape: what
  the Hausdorff distance, the average surface distance and surface Dice are formed from, on the GPU.

  For a volume v and key k, the surface S_v(k) is the voxels of label k with a face neighbour of
  another label or on a face of the volume (scipy's mask ^ binary_erosion(mask), border_value 0; in
  a stack neighbours never cross into the next volume).  d_v,k(q) is the float32 distance from q to
  the nearest voxel of S_v(k) under `anisotropy`, exactly edt(mask) of the mask that is 0 on S_v(k)
  and 1 elsewhere (+inf when S_v(k) is empty).  A->B for key k is {d_b,k(q) : q in S_a(k)}, B->A the
  other way round.

  `labels` (in the caller's dtype, distinct and non-zero) are the keys; the default is the sorted
  union of the non-zero labels of a and b.  Labels compare as edt() compares them (floats by value).
  `stacked=True` takes stacks of volumes along the slowest axis in memory, as edt(stacked=True) does.
  `max_device_bytes` bounds the device memory of the transforms (None or 0: what the GPU has free).

  Returns SurfaceDistances(labels, offsets, values): segment s = (volume * K + key) * 2 + direction
  (0: A->B, 1: B->A; volume 0 without `stacked`) is values[offsets[s]:offsets[s + 1]], sorted
  ascending.  numpy arrays for host input; torch CUDA tensors for device input, computed on the
  current stream."""
  import torch
  keys, offsets, values, _, host = _surface_run(a, b, anisotropy, labels, stacked, device, max_device_bytes)
  if host:
    return SurfaceDistances(keys, offsets.cpu().numpy(), values.cpu().numpy())
  return SurfaceDistances(torch.from_numpy(np.ascontiguousarray(keys)).to(offsets.device), offsets, values)


def _surface_metric(a, b, anisotropy, labels, stacked, device, max_device_bytes, reduce):
  """reduce(offsets, values, n) -> float64 (count, K) tensor from the sorted segments, with n the
  (count, K, 2) segment lengths; then the empty-surface rules and the caller's shape and type."""
  import torch
  keys, offsets, values, count, host = _surface_run(a, b, anisotropy, labels, stacked, device, max_device_bytes)
  nkeys = keys.size
  n = (offsets[1:] - offsets[:-1]).reshape(count, nkeys, 2)
  out = reduce(offsets, values.to(torch.float64), n) if values.numel() else \
      torch.zeros((count, nkeys), dtype=torch.float64, device=offsets.device)
  out = torch.where((n[..., 0] == 0) & (n[..., 1] == 0), torch.full_like(out, float("nan")), out)
  if not stacked:
    out = out[0]
  return out.cpu().numpy() if host else out


def _segment_sums(offsets, x):
  import torch
  return torch.segment_reduce(x, "sum", offsets=offsets, unsafe=True)


def hausdorff_distance(a, b, anisotropy=None, *, percentile=None, directed=False, labels=None, stacked=False, device=0,
                       max_device_bytes=None):
  """The Hausdorff distance between the surfaces of a (prediction) and b (reference) per key (see
  surface_distances for the definitions and arguments): the largest distance A->B, or with
  `percentile=p` np.percentile(A->B, p, method="linear"); with `directed=False` the larger of that over
  A->B and over B->A.  Per key it is NaN when both surfaces are empty and +inf when one is.

  Returns float64 of shape (K,), or (count, K) with `stacked`, in the order of `labels` (default: the
  sorted union of the non-zero labels): numpy for host input, a torch CUDA tensor for device input."""
  if percentile is not None:
    percentile = float(percentile)
    if not 0.0 <= percentile <= 100.0:
      raise ValueError("percentile must be within [0, 100], got %r" % (percentile,))

  def reduce(offsets, v, n):
    import torch
    start, length = offsets[:-1].reshape(n.shape), n
    if percentile is None:
      at = (start + length - 1).clamp(min=0)
      d = v[at.clamp(max=v.numel() - 1)]
    else:       # numpy's linear rule, its two-sided lerp included
      pos = (percentile / 100.0) * (length - 1).clamp(min=0).to(torch.float64)
      lo = pos.floor()
      t = pos - lo
      lo = lo.to(torch.int64)
      hi = torch.minimum(lo + 1, (length - 1).clamp(min=0))
      xa = v[(start + lo).clamp(max=v.numel() - 1)]
      xb = v[(start + hi).clamp(max=v.numel() - 1)]
      diff = xb - xa
      d = torch.where(t >= 0.5, xb - diff * (1 - t), xa + diff * t)
    d = d[..., 0] if directed else torch.maximum(d[..., 0], d[..., 1])
    return torch.where((n[..., 0] == 0) | (n[..., 1] == 0), torch.full_like(d, float("inf")), d)
  return _surface_metric(a, b, anisotropy, labels, stacked, device, max_device_bytes, reduce)


def average_surface_distance(a, b, anisotropy=None, *, symmetric=False, labels=None, stacked=False, device=0,
                             max_device_bytes=None):
  """The average surface distance per key (see surface_distances for the definitions and arguments):
  the mean of A->B, or with `symmetric=True` the mean of A->B and B->A taken together.  Per key it is
  NaN when both surfaces are empty and +inf when one is.  The sums are formed in float64 from the
  sorted segments, so the result does not depend on the order the GPU found the distances in.

  Returns float64 of shape (K,), or (count, K) with `stacked`, as hausdorff_distance does."""
  def reduce(offsets, v, n):
    import torch
    sums = _segment_sums(offsets, v).reshape(n.shape)
    if symmetric:
      m = sums.sum(-1) / n.sum(-1).to(torch.float64)
    else:
      m = sums[..., 0] / n[..., 0].to(torch.float64)
    return torch.where((n[..., 0] == 0) | (n[..., 1] == 0), torch.full_like(m, float("inf")), m)
  return _surface_metric(a, b, anisotropy, labels, stacked, device, max_device_bytes, reduce)


def surface_dice(a, b, tolerance, anisotropy=None, *, labels=None, stacked=False, device=0, max_device_bytes=None):
  """Surface Dice at `tolerance` per key (see surface_distances for the definitions and arguments):
  (#{A->B <= tolerance} + #{B->A <= tolerance}) / (|S_a| + |S_b|), the distances compared in float64.
  Per key it is NaN when both surfaces are empty and 0 when one is.

  Returns float64 of shape (K,), or (count, K) with `stacked`, as hausdorff_distance does."""
  tau = float(tolerance)
  if not tau >= 0.0:
    raise ValueError("tolerance must be zero or more, got %r" % (tolerance,))

  def reduce(offsets, v, n):
    import torch
    within = _segment_sums(offsets, (v <= tau).to(torch.float64)).reshape(n.shape)
    dice = within.sum(-1) / n.sum(-1).to(torch.float64)
    return torch.where((n[..., 0] == 0) | (n[..., 1] == 0), torch.zeros_like(dice), dice)
  return _surface_metric(a, b, anisotropy, labels, stacked, device, max_device_bytes, reduce)


# ---------------------------------------------------------------------------------------
# downstream helper of the reference's headline use case: one multi-label transform, then one
# masked image per label (src/edt.pyx:951-994; README.md:23, 204)
# ---------------------------------------------------------------------------------------

def label_stats_cuda(labels, dt):
  """Per-label statistics of a finished transform in ONE pass on the device: a dict of torch CUDA
  tensors sorted by label -- "labels" (int64, background 0 skipped), "count" (voxels), "max"
  (largest distance), "argmax" (smallest C-order linear index where it is attained), "box"
  (n x 6: inclusive bounding box, low corner then high corner, in ARRAY axis order).
  `labels` and `dt` are C-contiguous CUDA tensors of the same 1-3 dim shape (kernels:
  csrc/edt_each.cuh; the reference builds the same information from run lists,
  src/edt_voxel_graph.hpp:238-275)."""
  import torch
  if not (isinstance(labels, torch.Tensor) and labels.is_cuda and isinstance(dt, torch.Tensor) and dt.is_cuda):
    raise TypeError("label_stats_cuda expects torch CUDA tensors")
  if labels.shape != dt.shape or labels.device != dt.device:
    raise ValueError("labels and dt must have the same shape and device")
  nbytes = _torch_label_bytes(torch).get(labels.dtype)
  if nbytes is None:
    raise TypeError("label_stats_cuda: unsupported label dtype %s" % labels.dtype)
  labels = labels.contiguous()
  dt = dt.contiguous().to(torch.float32)
  nd = labels.dim()
  dims = [int(d) for d in labels.shape][::-1] + [1] * (3 - nd)          # sx, sy, sz
  dev = labels.device
  stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
  capacity = 1024
  while True:
    keys = torch.empty(capacity, dtype=torch.int64, device=dev)
    count = torch.empty(capacity, dtype=torch.int64, device=dev)
    mx = torch.empty(capacity, dtype=torch.float32, device=dev)
    argmax = torch.empty(capacity, dtype=torch.int64, device=dev)
    box = torch.empty((capacity, 6), dtype=torch.int32, device=dev)
    overflow = torch.zeros(1, dtype=torch.int32, device=dev)
    _check(_lib().edtb200_label_stats(labels.data_ptr(), nbytes, dt.data_ptr(), dims[0], dims[1], dims[2],
                                      capacity, keys.data_ptr(), count.data_ptr(), mx.data_ptr(),
                                      argmax.data_ptr(), box.data_ptr(), overflow.data_ptr(), dev.index, stream))
    used = int((keys != 0).sum().item())
    if int(overflow.item()) == 0 and 2 * used <= capacity:
      break
    capacity *= 4                                    # table too full (or full): again with more room
  sel = torch.nonzero(keys != 0).flatten()
  order = sel[torch.argsort(_unsigned_sort_key(torch, keys[sel], nbytes))]
  b = box[order].to(torch.int64)
  lo = b[:, :nd].flip(1)                             # x0 y0 z0 -> array axis order
  hi = b[:, 3:3 + nd].flip(1)
  return {"labels": keys[order], "count": count[order], "max": mx[order], "argmax": argmax[order],
          "box": torch.cat([lo, hi], dim=1)}


def _unsigned_sort_key(torch, keys, nbytes):
  """Sort key that orders int64-held label bits as the unsigned integers they are."""
  if nbytes < 8:
    return keys
  return keys ^ torch.tensor(-0x8000000000000000, dtype=torch.int64, device=keys.device)


def _label_scalar(torch, key, dtype):
  """The label value a table key (the label's raw bits, zero-extended) stands for."""
  nbytes = torch.empty((), dtype=dtype).element_size()
  raw = np.array([key & ((1 << (8 * nbytes)) - 1)], dtype=np.dtype("u%d" % nbytes))
  if dtype == torch.bool:
    return bool(raw[0])
  if dtype.is_floating_point:
    return float(raw.view(np.dtype("f%d" % nbytes))[0])
  if dtype == torch.uint8:
    return int(raw[0])
  return int(raw.view(np.dtype("i%d" % nbytes))[0])      # torch's other integer types are signed


def each_cuda(labels, dt, in_place=False, *, _stats=None):
  """Device-resident `each` (reference: edt.each, src/edt.pyx:951-994): iterator over
  (label, dt masked to that label) as torch CUDA tensors, labels in ascending order of their raw
  bits (the reference's order is that of a hash map), background skipped.
  One pass of `label_stats_cuda` finds every label's bounding box; each image is then drawn by a
  kernel that touches only that box (the device equivalent of the reference's run-list
  transfer).  in_place=True reuses ONE image: the previous label's box is erased, the next one
  drawn -- do not keep references to it between iterations (the reference marks it read-only)."""
  import torch
  stats = _stats if _stats is not None else label_stats_cuda(labels, dt)
  labels = labels.contiguous()
  dt = dt.contiguous().to(torch.float32)
  nbytes = _torch_label_bytes(torch)[labels.dtype]
  nd = labels.dim()
  dims = [int(d) for d in labels.shape][::-1] + [1] * (3 - nd)
  dev = labels.device
  keys = stats["labels"].tolist()
  boxes = stats["box"].tolist()
  lib = _lib()

  class DeviceImageIterator:
    def __len__(self):
      return len(keys)

    def __iter__(self):
      img = torch.zeros(labels.shape, dtype=torch.float32, device=dev) if in_place else None
      prev = None
      for key, bx in zip(keys, boxes):
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        lo, hi = bx[:nd][::-1] + [0] * (3 - nd), bx[nd:][::-1] + [0] * (3 - nd)      # -> x y z order
        cbox = (ctypes.c_int * 6)(*(lo + hi))
        out = img if in_place else torch.zeros(labels.shape, dtype=torch.float32, device=dev)
        if in_place and prev is not None:
          _check(lib.edtb200_label_extract(labels.data_ptr(), nbytes, dt.data_ptr(), dims[0], dims[1], dims[2],
                                           ctypes.c_uint64(0), prev, 1, out.data_ptr(), dev.index, stream))
        _check(lib.edtb200_label_extract(labels.data_ptr(), nbytes, dt.data_ptr(), dims[0], dims[1], dims[2],
                                         ctypes.c_uint64(key & 0xffffffffffffffff), cbox, 0, out.data_ptr(),
                                         dev.index, stream))
        prev = cbox
        yield (_label_scalar(torch, key, labels.dtype), out)

  return DeviceImageIterator()


def each(labels, dt, in_place=False, *, device=0):
  """Iterator over (label, distance transform of that label alone), labels in ascending order,
  background skipped -- same contract as the reference's edt.each (src/edt.pyx:951-994), which
  builds it from run lists (src/edt_voxel_graph.hpp:238-310).  Here labels and dt are uploaded
  ONCE, every label's bounding box comes from one device pass (`label_stats_cuda`), each masked
  image is drawn on the device inside that box, and only the box travels back to be pasted into
  the host image.  in_place=True reuses one read-only image between iterations, as the reference
  does.  Device-resident input (torch CUDA tensors) is handed to `each_cuda`."""
  try:
    import torch
  except ImportError:          # pragma: no cover
    torch = None
  if torch is not None and isinstance(labels, torch.Tensor) and labels.is_cuda:
    return each_cuda(labels, dt, in_place)
  labels = np.asarray(labels)
  dt = np.asarray(dt)
  if labels.shape != dt.shape:
    raise ValueError("labels and dt must have the same shape")
  if labels.ndim < 1 or labels.ndim > 3:
    raise TypeError("Multi-Label EDT library only supports up to 3 dimensions got {}.".format(labels.ndim))
  order = "F" if labels.flags.f_contiguous else "C"
  view = _label_view(labels)
  if view is None or torch is None:
    raise TypeError("each: unsupported label dtype %s" % labels.dtype)
  # memory order decides the axis roles on the device; the images are pasted back in array order
  mem = view.T if order == "F" else view
  dmem = dt.T if order == "F" else dt
  dev = torch.device("cuda", int(device))
  signed = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[view.dtype.itemsize]
  raw = np.ascontiguousarray(mem)
  lab_t = torch.from_numpy(raw.view(np.dtype("i%d" % raw.dtype.itemsize) if raw.dtype.itemsize > 1 else np.uint8)).to(dev)
  assert lab_t.dtype == signed
  dt_t = torch.from_numpy(np.ascontiguousarray(dmem, dtype=np.float32)).to(dev)
  stats = label_stats_cuda(lab_t, dt_t)
  keys = stats["labels"].tolist()
  boxes = stats["box"].tolist()
  nd = labels.ndim
  inner = each_cuda(lab_t, dt_t, in_place=True, _stats=stats)

  def key_value(key):
    # the device iterator reports the label's raw bits as an integer: back to the array's own dtype
    return np.array([key & ((1 << (8 * view.dtype.itemsize)) - 1)], dtype=view.dtype).view(labels.dtype)[0]

  class ImageIterator:
    def __len__(self):
      return len(keys)

    def __iter__(self):
      img = np.zeros(labels.shape, dtype=np.float32, order=order) if in_place else None
      prev = None
      for (key, dimg), bx in zip(inner, boxes):
        sl = tuple(slice(bx[a], bx[nd + a] + 1) for a in range(nd))          # box in device-array axis order
        sub = dimg[sl].cpu().numpy()
        host_sl, host_sub = (sl[::-1], sub.T) if order == "F" else (sl, sub)
        if in_place:
          img.setflags(write=1)
          if prev is not None:
            img[prev] = 0
          img[host_sl] = host_sub
          img.setflags(write=0)
          prev = host_sl
          yield (key_value(int(key)), img)
        else:
          out = np.zeros(labels.shape, dtype=np.float32, order=order)
          out[host_sl] = host_sub
          yield (key_value(int(key)), out)

  return ImageIterator()


def release():
  """Free cached device buffers held by the library, and the idle page-locked result blocks."""
  global _POOL_IDLE
  lib = _lib()
  with _POOL_LOCK:
    for size, ptrs in _POOL_FREE.items():
      while ptrs:
        lib.edtb200_host_free(ctypes.c_void_p(ptrs.pop()))
        _POOL_IDLE -= size
  _check(lib.edtb200_release())
