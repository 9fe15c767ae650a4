"""CPU tests: what the transform front doors -- the edt family, feature_transform, expand_labels' chunked
host path and transform_batch -- hand the C ABI, and how they map its results back to the caller's layout.

The library is replaced by a recording stub whose calls succeed.  Into every output it writes a known
pattern: distances get their x-fastest linear index, and x-fastest index plane j gets the coordinate
sx - 1 (sy - 1, sz - 1) of the volume's last voxel.  So each test checks the entry point, every scalar
argument, which buffer and plane each pointer points into, the label bits the C ABI reads, and the type,
shape, dtype, strides and values of what comes back.  The host and device paths still differ in a few
anisotropy and dtype rules; the tests at the end pin those as they are, so that a later change decides
them on purpose."""
import ctypes

import numpy as np
import pytest

SQRT, SIGNED, ON_DEVICE, FLOAT = 1, 2, 4 | 8, 16
FAMILY = {"edt": SQRT, "edtsq": 0, "sdf": SQRT | SIGNED, "sdfsq": SIGNED}

# entry point -> (index of the geometry, stacked geometry, index of the distances, index of the index planes)
LAYOUT = {
  "edtb200_transform": (2, False, 11, None),
  "edtb200_transform_bounded": (2, False, 11, None),
  "edtb200_transform_chunked": (2, False, 11, None),
  "edtb200_transform_multi": (2, False, 11, None),
  "edtb200_transform_stack": (2, True, 12, None),
  "edtb200_feature_transform": (2, False, 11, 12),
  "edtb200_feature_transform_bounded": (2, False, 11, 12),
  "edtb200_feature_transform_chunked": (2, False, 11, 12),
  "edtb200_feature_transform_stack": (2, True, 12, 13),
  "edtb200_transform_voxel_graph": (3, False, 12, None),
  "edtb200_transform_voxel_graph_chunked": (3, False, 12, None),
}


def _fill(ptr, n, ctype, values):
  np.ctypeslib.as_array((ctype * n).from_address(ptr))[:] = values


def _read(ptr, n, nbytes):
  return np.frombuffer(ctypes.string_at(ptr, n * nbytes), np.dtype("u%d" % nbytes)).copy()


class Call:
  def __init__(self, name, args):
    self.name = name
    self.args = tuple(list(a) if isinstance(a, ctypes.Array) else a for a in args)
    self.labels = self.graph = None


class Stub:
  """Records every edtb200_* call; each one succeeds and writes the pattern described above."""

  def __init__(self):
    self.calls = []

  def edtb200_host_alloc(self, nbytes):
    return 0

  def edtb200_last_error(self):
    return b""

  def edtb200_device_count(self):
    return 1

  def __getattr__(self, name):
    def call(*args):
      c = Call(name, args)
      self.calls.append(c)
      if name == "edtb200_transform_batch":
        n = c.args[5] * c.args[6] * c.args[7]
        c.labels = [_read(p, n, c.args[3]) for p in c.args[0]]
        for p in c.args[1]:
          _fill(p, n, ctypes.c_float, np.arange(n))
        return 0
      g, stacked, out, planes = LAYOUT[name]
      dims = c.args[g + 1:g + 4]
      n = dims[0] * dims[1] * dims[2] * (c.args[g + 4] if stacked else 1)
      c.labels = _read(c.args[0], n, c.args[1])
      if g == 3:
        c.graph = _read(c.args[2], n, 1)
      if c.args[out] is not None:
        _fill(c.args[out], n, ctypes.c_float, np.arange(n))
      if planes is not None:
        for j, p in enumerate(c.args[planes]):
          _fill(p, n, ctypes.c_int32, dims[j] - 1)
      return 0
    return call


@pytest.fixture
def stub(monkeypatch):
  import edt_b200
  s = Stub()
  monkeypatch.setattr(edt_b200, "_lib", lambda: s)
  monkeypatch.setenv("EDTB200_PINNED_POOL_MB", "0")
  return s


# ---------------------------------------------------------------------------------------------------------
# restatements of the layout rules the tests check against
# ---------------------------------------------------------------------------------------------------------

def _raw(x):
  """The label bits the C ABI reads: floats by value (-0.0 folded), signed and bool as unsigned."""
  x = np.asarray(x)
  if x.dtype.kind == "f":
    x = x + x.dtype.type(0)
  return x.view(np.dtype("u%d" % x.itemsize))


def _geometry(vshape, weights, order):
  """(sx, sy, sz), (wx, wy, wz) of a volume of `vshape` in memory order `order`."""
  dims, w = list(vshape), [float(a) for a in weights]
  if order == "C":
    dims, w = dims[::-1], w[::-1]
  return tuple(dims + [1] * (3 - len(dims))), tuple(w + [1.0] * (3 - len(w)))


def _pattern(shape, order, dtype=np.float32):
  """What a result holds when the C ABI wrote its x-fastest linear index, mapped back to `shape`."""
  return np.arange(int(np.prod(shape)), dtype=dtype).reshape(shape, order=order)


def _same(got, want):
  assert type(got) is type(want)
  assert got.shape == want.shape and got.dtype == want.dtype and got.strides == want.strides, \
      (got.shape, got.dtype, got.strides, want.shape, want.dtype, want.strides)
  assert got.tobytes(order="A") == want.tobytes(order="A")


def _labels_read(call, x, order):
  """The C ABI read x's label bits in its x-fastest order, from x's own buffer where no copy was needed."""
  x = np.asarray(x)
  np.testing.assert_array_equal(call.labels, _raw(x).ravel(order=order))
  contiguous = x.flags.c_contiguous if order == "C" else x.flags.f_contiguous
  if contiguous and x.dtype.kind != "f":
    assert call.args[0] == x.ctypes.data


def _volume(shape, dtype=np.int32, order="C", seed=0):
  rng = np.random.default_rng(seed)
  x = rng.integers(0, 3, shape).astype(dtype)
  return np.asfortranarray(x) if order == "F" else np.ascontiguousarray(x)


# ---------------------------------------------------------------------------------------------------------
# the edt family
# ---------------------------------------------------------------------------------------------------------

DTYPES = [np.bool_, np.int8, np.uint8, np.int16, np.uint16, np.int32, np.uint32, np.int64, np.uint64,
          np.float32, np.float64]


def _family_input(kind):
  """(input, the memory order it is transformed in)."""
  if kind == "C":
    return _volume((3, 4, 5)), "C"
  if kind == "F":
    return _volume((3, 4, 5), order="F"), "F"
  if kind == "strided":
    return _volume((3, 8, 5))[:, ::2], "C"
  if kind == "list":
    return _volume((3, 4)).tolist(), "C"
  if kind == "1d":
    return _volume((7,)), "F"                 # both orders apply: Fortran wins for the unstacked host path
  if kind == "2d_F":
    return _volume((4, 6), order="F"), "F"
  if kind == "row":
    return _volume((1, 6)), "F"
  raise KeyError(kind)


@pytest.mark.parametrize("fn", list(FAMILY))
@pytest.mark.parametrize("kind", ["C", "F", "strided", "list", "1d", "2d_F", "row"])
@pytest.mark.parametrize("weights", [None, "given"])
def test_edt_family_one_shot(edt, stub, fn, kind, weights):
  x, order = _family_input(kind)
  nd = np.ndim(x)
  aniso = None if weights is None else ((2.5,) if nd == 1 else (1.0, 2.0, 3.0)[:nd])
  got = getattr(edt, fn)(x, aniso, True)
  [call] = stub.calls
  shape = np.shape(x)
  (sx, sy, sz), (wx, wy, wz) = _geometry(shape, aniso or (1.0,) * nd, order)
  assert call.name == "edtb200_transform"
  assert call.args[1:] == (8 if kind == "list" else 4, nd, sx, sy, sz, wx, wy, wz, 1, FAMILY[fn], got.ctypes.data,
                           0, None)
  _labels_read(call, x, order)
  _same(got, _pattern(shape, order))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("order", ["C", "F"])
def test_edt_label_dtypes(edt, stub, dtype, order):
  x = _volume((3, 4, 5), dtype, order)
  if x.dtype.kind == "f":
    x[0, 0, :2] = -0.0
    x[1, 1, 1] = 1.5
  got = edt.sdf(x, device=3)
  [call] = stub.calls
  (sx, sy, sz), (wx, wy, wz) = _geometry(x.shape, (1.0,) * 3, order)
  assert call.name == "edtb200_transform"
  assert call.args[1:] == (x.itemsize, 3, sx, sy, sz, wx, wy, wz, 0, SQRT | SIGNED, got.ctypes.data, 3, None)
  _labels_read(call, x, order)
  _same(got, _pattern(x.shape, order))


@pytest.mark.parametrize("fn,dims", [("edt1d", 1), ("edt1dsq", 1), ("edt2d", 2), ("edt2dsq", 2), ("edt3d", 3),
                                     ("edt3dsq", 3)])
def test_fixed_dimension_aliases(edt, stub, fn, dims):
  x = _volume((5, 6, 7)[:dims])
  got = getattr(edt, fn)(x)
  [call] = stub.calls
  (sx, sy, sz), (wx, wy, wz) = _geometry(x.shape, (1.0,) * dims, "F" if dims == 1 else "C")
  assert call.name == "edtb200_transform"
  assert call.args[1:] == (4, dims, sx, sy, sz, wx, wy, wz, 0, 0 if fn.endswith("sq") else SQRT, got.ctypes.data, 0,
                           None)
  _same(got, _pattern(x.shape, "F" if dims == 1 else "C"))
  with pytest.raises(ValueError, match="expected a %d-D array, got %d-D" % (dims, dims % 3 + 1)):
    getattr(edt, fn)(_volume((5, 6, 7)[:dims % 3 + 1]))


@pytest.mark.parametrize("order", ["C", "F"])
def test_edt_max_distance(edt, stub, order):
  x = _volume((3, 4, 5), order=order)
  got = edt.sdfsq(x, (1.0, 2.0, 3.0), max_distance=2.5)
  [call] = stub.calls
  (sx, sy, sz), (wx, wy, wz) = _geometry(x.shape, (1.0, 2.0, 3.0), order)
  assert call.name == "edtb200_transform_bounded"
  assert call.args[1:] == (4, 3, sx, sy, sz, wx, wy, wz, 0, SIGNED, got.ctypes.data, 0, None, 2.5)
  _labels_read(call, x, order)
  _same(got, _pattern(x.shape, order))
  assert edt.edt(x, max_distance=float("inf")) is not None
  assert stub.calls[-1].name == "edtb200_transform"


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("budget", [0, 1 << 20])
def test_edt_max_device_bytes(edt, stub, order, budget):
  x = _volume((3, 4, 5), np.uint16, order)
  got = edt.edt3d(x, max_device_bytes=budget)
  [call] = stub.calls
  (sx, sy, sz), (wx, wy, wz) = _geometry(x.shape, (1.0,) * 3, order)
  assert call.name == "edtb200_transform_chunked"
  assert call.args[1:] == (2, 3, sx, sy, sz, wx, wy, wz, 0, SQRT, got.ctypes.data, 0, budget, None)
  _labels_read(call, x, order)
  _same(got, _pattern(x.shape, order))


def test_edt_devices(edt, stub):
  x = _volume((3, 4, 5), order="F")
  got = edt.edtsq(x, (1.0, 2.0, 3.0), devices=[0, 1])
  [call] = stub.calls
  (sx, sy, sz), (wx, wy, wz) = _geometry(x.shape, (1.0, 2.0, 3.0), "F")
  assert call.name == "edtb200_transform_multi"
  assert call.args[1:] == (4, 3, sx, sy, sz, wx, wy, wz, 0, 0, got.ctypes.data, [0, 1], 2)
  _labels_read(call, x, "F")
  _same(got, _pattern(x.shape, "F"))
  edt.edtsq(x, devices=[1])
  assert stub.calls[-1].name == "edtb200_transform" and stub.calls[-1].args[12] == 1


@pytest.mark.parametrize("dims", [2, 3, 4])
@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("fn", ["edt", "sdfsq"])
def test_edt_stacked(edt, stub, dims, order, fn):
  x = _volume((5, 3, 4, 6)[:dims], np.int64, order)
  if order == "C":
    count, vshape = x.shape[0], x.shape[1:]
  else:
    count, vshape = x.shape[-1], x.shape[:-1]
  weights = (1.0, 2.0, 3.0)[:dims - 1]
  got = getattr(edt, fn)(x, weights, True, stacked=True, max_device_bytes=None if fn == "edt" else 123)
  [call] = stub.calls
  (sx, sy, sz), (wx, wy, wz) = _geometry(vshape, weights, order)
  assert call.name == "edtb200_transform_stack"
  assert call.args[1:] == (8, dims - 1, sx, sy, sz, count, wx, wy, wz, 1, FAMILY[fn], got.ctypes.data, 0,
                           0 if fn == "edt" else 123, None, None)
  _labels_read(call, x, order)
  _same(got, _pattern(x.shape, order))


def test_edt_stacked_scalar_weight_of_1d_volumes(edt, stub):
  x = _volume((4, 6))
  edt.edt(x, 2.0, stacked=True)
  assert stub.calls[-1].args[7:10] == (2.0, 1.0, 1.0)


@pytest.mark.parametrize("kind", ["plain", "signed", "float", "F"])
def test_edt_voxel_graph(edt, stub, kind):
  x = _volume((4, 5), np.float32 if kind == "float" else np.int32, "F" if kind == "F" else "C")
  if kind == "float":
    x[0, :2] = -0.0
    x[1, 1] = np.nan
  order = "F" if kind == "F" else "C"
  graph = np.full(x.shape, 0x3f, np.uint8)
  graph[1, 2] = 0x15
  got = (edt.sdf if kind == "signed" else edt.edt)(x, (2.0, 3.0), voxel_graph=graph.astype(np.int32), devices=[1])
  (sx, sy, sz), (wx, wy, wz) = _geometry(x.shape, (2.0, 3.0), order)
  firsts = [x, x == 0] if kind == "signed" else [x]
  assert len(stub.calls) == len(firsts)
  for call, labels in zip(stub.calls, firsts):
    assert call.name == "edtb200_transform_voxel_graph"
    nbytes = np.asarray(labels).itemsize
    assert call.args[1] == nbytes and call.args[3:12] == (2, sx, sy, sz, wx, wy, wz, 0,
                                                          SQRT | (FLOAT if kind == "float" else 0))
    assert call.args[13:] == (1, None)
    raw = labels.view(np.dtype("u%d" % nbytes))     # float labels as they are: the C ABI compares them
    np.testing.assert_array_equal(call.labels, raw.ravel(order=order))
    np.testing.assert_array_equal(call.graph, graph.ravel(order=order))
  want = _pattern(x.shape, order)
  if kind == "signed":
    want = want - want
  assert got.ctypes.data == stub.calls[0].args[12]
  _same(got, want)


def test_edt_voxel_graph_checks(edt, stub):
  with pytest.raises(ValueError, match="voxel_graph must have the shape of data"):
    edt.edt(np.ones((4, 5), np.int32), voxel_graph=np.ones((5, 4), np.uint8))
  with pytest.raises(TypeError, match="only supported for 2D and 3D. Got 1"):
    edt.edt(np.ones(4, np.int32), voxel_graph=np.ones(4, np.uint8))
  got = edt.edt(np.ones((4, 5), np.complex64), voxel_graph=np.ones((4, 5), np.uint8))
  _same(got, np.zeros((4, 5), np.float32))
  assert stub.calls == []


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("dtype", [np.complex64, np.float16])
def test_sdf_voxel_graph_of_unsupported_labels(edt, stub, order, dtype):
  """f(data) - f(data == 0) with f(data) zeros: the background term is still transformed."""
  x = np.ones((4, 5), dtype, order=order)
  x[1, 2] = 0
  graph = np.full(x.shape, 0x3f, np.uint8)
  got = edt.sdfsq(x, (2.0, 3.0), voxel_graph=graph)
  [call] = stub.calls
  (sx, sy, sz), (wx, wy, wz) = _geometry(x.shape, (2.0, 3.0), order)
  assert call.name == "edtb200_transform_voxel_graph"
  assert call.args[1] == 1 and call.args[3:12] == (2, sx, sy, sz, wx, wy, wz, 0, 0) and call.args[13:] == (0, None)
  np.testing.assert_array_equal(call.labels, (x == 0).view(np.uint8).ravel(order=order))
  _same(got, np.zeros(x.shape, np.float32, order=order) - _pattern(x.shape, order))


@pytest.mark.parametrize("stacked", [False, True])
@pytest.mark.parametrize("order", ["C", "F"])
def test_edt_empty_and_unsupported(edt, stub, stacked, order):
  empty = np.ones((3, 0, 4), np.int32, order=order)
  got = edt.edt(empty, stacked=stacked)
  # an empty unstacked result is C-ordered whatever the input's order; a stack keeps its order
  _same(got, np.zeros(empty.shape, np.float32, order=order if stacked else "C"))
  x = np.ones((3, 4, 5), np.complex64, order=order)
  _same(edt.edt(x, stacked=stacked), np.zeros(x.shape, np.float32, order=order))
  assert stub.calls == []


def test_stacks_run_on_one_device(edt, stub):
  """A stack takes one device ordinal: a list for `device` is a TypeError, not a multi-GPU transform."""
  x = _volume((3, 4, 5))
  for fn in (edt.edt, edt.feature_transform):
    with pytest.raises(TypeError, match="not 'list'"):
      fn(x, stacked=True, device=[0, 1])
  assert stub.calls == []


def test_edt_zero_dimensional(edt, stub):
  for x in (np.array(3, np.int32), 3):
    with pytest.raises(TypeError, match="Multi-Label EDT library only supports up to 3 dimensions got 0."):
      edt.edt(x)
  with pytest.raises(TypeError, match="only supports up to 3 dimensions got 4."):
    edt.edt(np.ones((2, 2, 2, 2), np.int32))
  with pytest.raises(ValueError, match="stacked=True needs a 2-D to 4-D array"):
    edt.edt(np.ones(4, np.int32), stacked=True)
  assert stub.calls == []


def test_edt_argument_checks_precede_the_library(edt, stub):
  x = np.ones((3, 4, 5), np.uint8)
  cases = [
    (dict(max_distance=-1.0), ValueError, "max_distance must be zero or more"),
    (dict(max_distance=1.0, stacked=True), ValueError, "max_distance cannot be combined with stacked=True"),
    (dict(max_device_bytes=-1), ValueError, "non-negative"),
    (dict(max_device_bytes=-1, stacked=True), ValueError, "non-negative"),
    (dict(devices=[0, 1], max_device_bytes=0), ValueError, "max_device_bytes streams through one GPU"),
    (dict(devices=[0, 1], stacked=True), ValueError, "stacked=True runs on one GPU"),
    (dict(devices=[]), ValueError, "devices must name at least one GPU"),
    (dict(anisotropy=(1.0, 2.0)), ValueError, "anisotropy must have one entry per dimension"),
    (dict(anisotropy=(1.0, 2.0, 3.0), stacked=True), ValueError, r"one entry per volume axis \(2\), got 3"),
    (dict(voxel_graph=np.ones((3, 4, 5), np.uint8), stacked=True), ValueError, "cannot be combined with voxel_graph"),
    (dict(voxel_graph=np.ones((3, 4, 5), np.uint8), max_device_bytes=0), ValueError,
     "max_device_bytes cannot be combined with voxel_graph"),
  ]
  for kwargs, err, msg in cases:
    with pytest.raises(err, match=msg):
      edt.edt(x, **kwargs)
  with pytest.raises(ValueError, match="max_device_bytes needs a 2-D or 3-D array, got 1-D"):
    edt.edt(np.ones(5, np.uint8), max_device_bytes=0)
  assert stub.calls == []


# ---------------------------------------------------------------------------------------------------------
# feature_transform
# ---------------------------------------------------------------------------------------------------------

def _planes_checked(call, idx, vshape, order, plane_arg):
  """Index plane pointer j is the caller's axis j (F order) or vnd - 1 - j (C order) of `idx`, each plane
  holding the coordinate of the volume's last voxel along its axis."""
  vnd = len(vshape)
  assert idx.dtype == np.int32 and idx.shape[0] == vnd
  for j, p in enumerate(call.args[plane_arg]):
    assert p == idx[j if order == "F" else vnd - 1 - j].ctypes.data
  for k in range(vnd):
    assert (idx[k] == vshape[k] - 1).all()
  want = np.empty((vnd,) + (idx.shape[1:] if order == "C" else idx.shape[:0:-1]), np.int32)
  if order == "F":
    want = want.transpose((0,) + tuple(range(idx.ndim - 1, 0, -1)))
  assert idx.strides == want.strides


@pytest.mark.parametrize("kind", ["C", "F", "strided", "list", "1d", "2d_F", "row"])
@pytest.mark.parametrize("signed", [False, True])
@pytest.mark.parametrize("distances", [False, True])
def test_feature_transform(edt, stub, kind, signed, distances):
  x, order = _family_input(kind)
  nd = np.ndim(x)
  aniso = (2.5, 7.0) if nd == 1 else (1.0, 2.0, 3.0)[:nd]       # 1-D takes the first entry, as edt does
  got = edt.feature_transform(x, aniso, True, signed=signed, return_distances=distances, device=2)
  dist, idx = got if distances else (None, got)
  [call] = stub.calls
  shape = np.shape(x)
  (sx, sy, sz), (wx, wy, wz) = _geometry(shape, aniso[:nd], order)
  assert call.name == "edtb200_feature_transform"
  assert call.args[1:11] == (8 if kind == "list" else 4, nd, sx, sy, sz, wx, wy, wz, 1,
                            SQRT | (SIGNED if signed else 0))
  assert call.args[11] == (dist.ctypes.data if distances else None)
  assert call.args[13:] == (2, None)
  _labels_read(call, x, order)
  _planes_checked(call, idx, shape, order, 12)
  assert idx.shape[1:] == shape
  if distances:
    _same(dist, _pattern(shape, order))


@pytest.mark.parametrize("order", ["C", "F"])
def test_feature_transform_bounded_and_chunked(edt, stub, order):
  x = _volume((3, 4, 5), np.float64, order)
  x[0, 0, 0] = -0.0
  dist, idx = edt.feature_transform(x, return_distances=True, max_distance=1.5)
  dist2, idx2 = edt.feature_transform(x, return_distances=True, max_device_bytes=77)
  idx3 = edt.feature_transform(x, signed=True, max_device_bytes=0)
  (sx, sy, sz), (wx, wy, wz) = _geometry(x.shape, (1.0,) * 3, order)
  head = (8, 3, sx, sy, sz, wx, wy, wz, 0)
  names = [c.name for c in stub.calls]
  assert names == ["edtb200_feature_transform_bounded"] + ["edtb200_feature_transform_chunked"] * 2
  assert stub.calls[0].args[1:11] == head + (SQRT,) and stub.calls[0].args[13:] == (0, None, 1.5)
  assert stub.calls[1].args[1:11] == head + (SQRT,) and stub.calls[1].args[13:] == (0, 77, None)
  assert stub.calls[2].args[1:11] == head + (SQRT | SIGNED,) and stub.calls[2].args[11] is None
  assert stub.calls[2].args[13:] == (0, 0, None)
  for call, (d, i) in zip(stub.calls, [(dist, idx), (dist2, idx2), (None, idx3)]):
    _labels_read(call, x, order)
    _planes_checked(call, i, x.shape, order, 12)
    if d is not None:
      assert call.args[11] == d.ctypes.data
      _same(d, _pattern(x.shape, order))


@pytest.mark.parametrize("dims", [2, 3, 4])
@pytest.mark.parametrize("order", ["C", "F"])
def test_feature_transform_stacked(edt, stub, dims, order):
  x = _volume((5, 3, 4, 6)[:dims], np.uint32, order)
  if order == "C":
    count, vshape = x.shape[0], x.shape[1:]
  else:
    count, vshape = x.shape[-1], x.shape[:-1]
  weights = (1.0, 2.0, 3.0)[:dims - 1]
  dist, idx = edt.feature_transform(x, weights, signed=True, return_distances=True, stacked=True)
  [call] = stub.calls
  (sx, sy, sz), (wx, wy, wz) = _geometry(vshape, weights, order)
  assert call.name == "edtb200_feature_transform_stack"
  assert call.args[1:12] == (4, dims - 1, sx, sy, sz, count, wx, wy, wz, 0, SQRT | SIGNED)
  assert call.args[12] == dist.ctypes.data and call.args[14:] == (0, None)
  _labels_read(call, x, order)
  _planes_checked(call, idx, vshape, order, 13)
  assert idx.shape == (dims - 1,) + x.shape
  _same(dist, _pattern(x.shape, order))


@pytest.mark.parametrize("stacked", [False, True])
@pytest.mark.parametrize("order", ["C", "F"])
def test_feature_transform_empty_and_unsupported(edt, stub, stacked, order):
  x = np.ones((3, 0, 4), np.int16, order=order)
  dist, idx = edt.feature_transform(x, return_distances=True, stacked=stacked)
  # an empty array is contiguous in both orders: Fortran wins for one volume, C for a stack
  _same(dist, _pattern(x.shape, "C" if stacked else "F"))
  assert idx.shape == (2 if stacked else 3,) + x.shape and idx.dtype == np.int32
  with pytest.raises(TypeError, match="feature_transform: unsupported label dtype complex64"):
    edt.feature_transform(np.ones((3, 4, 5), np.complex64, order=order), stacked=stacked)
  with pytest.raises(TypeError, match="only supports up to 3 dimensions got 4"):
    edt.feature_transform(np.ones((2, 2, 2, 2), np.int32))
  with pytest.raises(ValueError, match="stacked=True stages the whole stack"):
    edt.feature_transform(np.ones((2, 2, 2), np.int32), stacked=True, max_device_bytes=0)
  with pytest.raises(ValueError, match="stacked=True needs a 2-D to 4-D array"):
    edt.feature_transform(np.ones(2, np.int32), stacked=True)
  assert stub.calls == []


# ---------------------------------------------------------------------------------------------------------
# expand_labels' chunked host path: the feature transform in chunks, the labels gathered on the host
# ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [np.uint8, np.int32, np.float32])
@pytest.mark.parametrize("order", ["C", "F", "strided"])
@pytest.mark.parametrize("dims", [2, 3])
def test_expand_labels_chunked(edt, stub, dtype, order, dims):
  x = _volume((4, 10, 5)[:dims], dtype, "F" if order == "F" else "C", seed=dims)
  if order == "strided":
    x = x[:, ::2]
  mem = "F" if order == "F" else "C"
  if np.dtype(dtype).kind == "f":
    x[(0,) * dims] = -0.0
  x[(-1,) * dims] = 7
  got = edt.expand_labels(x, 3.0, (1.0, 2.0, 3.0)[:dims], max_device_bytes=0, device=1)
  [call] = stub.calls
  (sx, sy, sz), (wx, wy, wz) = _geometry(x.shape, (1.0, 2.0, 3.0)[:dims], mem)
  assert call.name == "edtb200_feature_transform_chunked"
  assert call.args[1:11] == (x.itemsize, dims, sx, sy, sz, wx, wy, wz, 0, SIGNED)
  assert call.args[13:] == (1, 0, None)
  _labels_read(call, x, mem)
  # distances 0, 1, 2, ... in memory order: the first nine background voxels in memory take the label of
  # the site every index plane names, the last voxel
  flat = np.ascontiguousarray(x).ravel(order=mem) if mem == "C" else x.ravel(order="F")
  want = flat.copy()
  grow = (flat == 0) & (np.arange(flat.size) <= 9)
  want[grow] = flat[-1]
  _same(got, want.reshape(x.shape, order=mem))


def test_expand_labels_chunked_checks(edt, stub):
  with pytest.raises(ValueError, match="max_device_bytes needs a 2-D or 3-D array, got 1-D"):
    edt.expand_labels(np.ones(5, np.int32), max_device_bytes=0)
  with pytest.raises(ValueError, match="non-negative"):
    edt.expand_labels(np.ones((4, 5), np.int32), max_device_bytes=-1)
  with pytest.raises(TypeError, match="expand_labels: unsupported label dtype complex64"):
    edt.expand_labels(np.ones((4, 5), np.complex64), max_device_bytes=0)
  with pytest.raises(ValueError, match="stacked=True stages the whole stack"):
    edt.expand_labels(np.ones((4, 5), np.int32), max_device_bytes=0, stacked=True)
  got = edt.expand_labels(np.ones((4, 0), np.int16, order="F"), max_device_bytes=0)
  _same(got, np.ones((4, 0), np.int16))
  assert stub.calls == []


# ---------------------------------------------------------------------------------------------------------
# transform_batch
# ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("given", [False, True])
def test_transform_batch(edt, stub, order, given):
  vols = [_volume((3, 4, 5), np.int16, order, seed=s) for s in range(3)]
  vols[2] = np.ascontiguousarray(vols[2][:, :, ::-1]) if order == "C" else vols[2]
  outs = [np.empty((3, 4, 5), np.float32, order=order) for _ in vols] if given else None
  got = edt.transform_batch(vols, (1.0, 2.0, 3.0), True, sqrt=True, signed=True, outs=outs, device=1)
  [call] = stub.calls
  (sx, sy, sz), (wx, wy, wz) = _geometry((3, 4, 5), (1.0, 2.0, 3.0), order)
  assert call.name == "edtb200_transform_batch"
  assert call.args[0] == [v.ctypes.data for v in vols]
  assert call.args[1] == [o.ctypes.data for o in got]
  assert call.args[2:] == (3, 2, 3, sx, sy, sz, wx, wy, wz, 1, SQRT | SIGNED, 1)
  for labels, v in zip(call.labels, vols):
    np.testing.assert_array_equal(labels, _raw(v).ravel(order=order))
  if given:
    assert all(g is o for g, o in zip(got, outs))
  for g in got:
    _same(g, _pattern((3, 4, 5), order))


def test_transform_batch_edges(edt, stub):
  assert edt.transform_batch([]) == []
  x = np.ones(6, np.int32)
  edt.transform_batch([x], 2.0)
  assert stub.calls[-1].args[2:] == (1, 4, 1, 6, 1, 1, 2.0, 1.0, 1.0, 0, 0, 0)
  edt.transform_batch([np.asfortranarray(np.ones((4, 5), np.int32)), np.ones((4, 5), np.int32)])
  assert stub.calls[-1].args[5:8] == (4, 5, 1)
  with pytest.raises(TypeError, match="'float' object is not iterable"):
    edt.transform_batch([np.ones((4, 5), np.int32)], 2.0)
  with pytest.raises(ValueError, match="one entry per dimension"):
    edt.transform_batch([np.ones((4, 5), np.int32)], (1.0,))
  with pytest.raises(ValueError, match="one shape and dtype"):
    edt.transform_batch([np.ones((4, 5), np.int32), np.ones((4, 5), np.int16)])
  for out in edt.transform_batch([np.ones((4, 5), np.complex64)] * 2) + edt.transform_batch([np.ones((0, 5))]):
    assert not out.any()
  assert len(stub.calls) == 2


# ---------------------------------------------------------------------------------------------------------
# where host and device paths differ today
# ---------------------------------------------------------------------------------------------------------

def _fake_device(x):
  """A CPU tensor that _device_array takes for device-resident input; fine until the first CUDA call."""
  import torch

  class FakeCuda(torch.Tensor):
    @property
    def is_cuda(self):
      return True
  FakeCuda.__module__ = "torch.fake"
  return torch.from_numpy(x).as_subclass(FakeCuda)


def test_two_weights_for_one_dimension(edt, stub):
  x = np.ones(5, np.uint8)
  edt.edt(x, anisotropy=(2.0, 3.0))
  assert stub.calls[-1].args[6:9] == (2.0, 1.0, 1.0)
  edt.feature_transform(x, anisotropy=(2.0, 3.0))
  assert stub.calls[-1].args[6:9] == (2.0, 1.0, 1.0)
  pytest.importorskip("torch")
  with pytest.raises(ValueError, match="anisotropy must have one entry per dimension"):
    edt.edt(_fake_device(x), anisotropy=(2.0, 3.0))
  assert len(stub.calls) == 2


def test_one_weight_for_two_dimensions(edt, stub):
  x = np.ones((4, 5), np.uint8)
  with pytest.raises(TypeError, match="'float' object is not iterable"):
    edt.edt(x, anisotropy=2.0)
  pytest.importorskip("torch")
  with pytest.raises(ValueError, match="anisotropy must have one entry per dimension"):
    edt.edt(_fake_device(x), anisotropy=2.0)
  assert stub.calls == []


def test_unsupported_label_dtype(edt, stub):
  x = np.ones((4, 5), np.complex64)
  _same(edt.edt(x), np.zeros((4, 5), np.float32))
  with pytest.raises(TypeError, match="feature_transform: unsupported label dtype complex64"):
    edt.feature_transform(x)
  pytest.importorskip("torch")
  with pytest.raises(TypeError, match="edt_cuda: unsupported label dtype torch.complex64"):
    edt.edt(_fake_device(x))
  with pytest.raises(TypeError, match="feature_transform: unsupported label dtype torch.complex64"):
    edt.feature_transform(_fake_device(x))
  assert stub.calls == []
