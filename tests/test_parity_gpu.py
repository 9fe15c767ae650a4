"""GPU parity tests (-m gpu): the CUDA path, called through the C ABI, against the oracle.

Bar (BASELINE.json north_star): edtsq bit-exact on the integer squared-distance path;
edt / sdf within 1 ULP after sqrt (0 expected: IEEE sqrt on identical inputs).  For
non-integer anisotropy the kernels use one fused multiply-add per candidate only where the
host has proven the double sum exact (and the double form elsewhere), so the same exact
comparison is applied there; tests/test_envelope_gpu.py covers the rounding edges.
"""
import os
import zlib

import numpy as np
import pytest

import cases

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_vectors.npz")


def ulp_diff(a, b):
  """Max distance in float32 ULPs (inf/nan must match exactly)."""
  a = np.asarray(a, np.float32).ravel()
  b = np.asarray(b, np.float32).ravel()
  special = ~np.isfinite(a) | ~np.isfinite(b)
  if not np.array_equal(a[special], b[special], equal_nan=True):
    return np.inf
  ai = a[~special].view(np.int32).astype(np.int64)
  bi = b[~special].view(np.int32).astype(np.int64)
  ai = np.where(ai < 0, np.int64(-2**31) - ai, ai)
  bi = np.where(bi < 0, np.int64(-2**31) - bi, bi)
  return 0 if ai.size == 0 else int(np.abs(ai - bi).max())


def assert_same(got, want, what):
  assert got.shape == want.shape, (what, got.shape, want.shape)
  assert got.dtype == np.float32
  if not np.array_equal(got, want, equal_nan=True):
    bad = np.argwhere(~((got == want) | (np.isnan(got) & np.isnan(want))))
    first = tuple(bad[0])
    raise AssertionError("%s: %d of %d voxels differ; first at %s: got %r want %r (max ulp %s)" % (
      what, len(bad), got.size, first, got[first], want[first], ulp_diff(got, want)))


# ---- the reference's own golden vectors -------------------------------------------------

@pytest.mark.parametrize("case", cases.KNOWN_ANSWERS, ids=[c[0] for c in cases.KNOWN_ANSWERS])
def test_known_answers(edt, case):
  for dtype in case[4]:
    labels, kwargs, expected = cases.known_answer_arrays(case, dtype)
    for parallel in (1, 2):
      assert_same(edt.edtsq(labels, parallel=parallel, **kwargs), expected, (case[0], dtype))


def test_one_d_simple(edt):
  # automated_test.py:17-60
  for dtype in cases.ALL:
    for labels in ([0], [0, 1], [1, 0], [0, 1, 0], [0, 1, 1, 0]):
      arr = np.array(labels, dtype=dtype)
      for bb in (True, False):
        assert np.all(edt.edt(arr, black_border=bb) == arr)
    one = np.array([1], dtype=dtype)
    assert np.all(edt.edt(one, black_border=True) == one)
    assert np.all(edt.edt(one, black_border=False) == np.array([np.inf]))


def test_golden_fixtures(edt):
  z = np.load(GOLDEN)
  for seed in z["seeds"]:
    key = "s%d" % seed
    labels = z[key + "_labels"]
    an = z[key + "_aniso"]
    an = float(an[0]) if labels.ndim == 1 else tuple(an)
    bb = bool(z[key + "_border"])
    assert_same(edt.edtsq(labels, anisotropy=an, black_border=bb), z[key + "_edtsq"], ("edtsq", seed))
    assert ulp_diff(edt.edt(labels, anisotropy=an, black_border=bb), z[key + "_edt"]) <= 1, seed
    assert ulp_diff(edt.sdf(labels, anisotropy=an, black_border=bb), z[key + "_sdf"]) <= 1, seed
  cfg1 = np.ones((64, 64, 64), dtype=np.uint32, order="F")      # BASELINE.json configs[0]
  got = edt.edtsq(cfg1, black_border=True, parallel=1)
  assert_same(got, z["cfg1_edtsq"], "cfg1")
  assert got.max() == 1024.0 and got.flags.f_contiguous


# ---- voxel_graph= path (src/edt_voxel_graph.hpp:54-236, edt.pyx:514-620, 736-844) --------------

def test_voxel_graph_golden_fixtures(edt):
  z = np.load(GOLDEN)
  for seed in z["graph_seeds"]:
    key = "g%d" % seed
    labels, graph = z[key + "_labels"], z[key + "_graph"]
    kw = dict(anisotropy=tuple(z[key + "_aniso"]), black_border=bool(z[key + "_border"]), voxel_graph=graph)
    got = edt.edtsq(labels, **kw)
    assert_same(got, z[key + "_edtsq"], ("edtsq", seed))
    assert got.flags.f_contiguous == z[key + "_edtsq"].flags.f_contiguous
    with np.errstate(invalid="ignore"):
      assert ulp_diff(edt.edt(labels, **kw), z[key + "_edt"]) <= 1, seed
      assert ulp_diff(edt.sdf(labels, **kw), z[key + "_sdf"]) <= 1, seed


def test_voxel_graph_known_answer_and_random(edt, oracle):
  labels = np.ones((5, 6), dtype=np.int64)                       # automated_test.py:736-789
  graph = np.full((5, 6), 0b111111, dtype=np.uint8)
  assert np.all(edt.edt(labels, voxel_graph=graph) == np.inf)
  ring = np.array([[0.5] * 6, [0.5, 1.5, 1.5, 1.5, 1.5, 0.5], [0.5, 1.5, 2.5, 2.5, 1.5, 0.5],
                   [0.5, 1.5, 1.5, 1.5, 1.5, 0.5], [0.5] * 6], dtype=np.float32)
  assert_same(edt.edt(labels, voxel_graph=graph, black_border=True), ring, "ring")
  graph[2, 2], graph[2, 3] = 0b111110, 0b111101
  for g in (graph, np.asfortranarray(graph)):
    assert_same(edt.edt(labels, voxel_graph=g, black_border=True),
                oracle.edt(labels, voxel_graph=g, black_border=True), "blocked edge")
  for seed in range(200, 260):
    labels, graph, kwargs = cases.random_graph_case(seed)
    what = (seed, labels.shape, labels.dtype.name, kwargs)
    assert_same(edt.edtsq(labels, voxel_graph=graph, **kwargs),
                oracle.edtsq(labels, voxel_graph=graph, **kwargs), ("edtsq",) + what)
    if seed % 4 == 0:
      with np.errstate(invalid="ignore"):
        assert_same(edt.sdfsq(labels, voxel_graph=graph, **kwargs),
                    oracle.sdfsq(labels, voxel_graph=graph, **kwargs), ("sdfsq",) + what)
  # a volume large enough for the tile kernels on the doubled grid (2 * 96 = 192 rows per axis)
  rng = np.random.default_rng(11)
  labels = (rng.random((96, 80, 72)) < 0.995).astype(np.uint16)
  graph = np.where(rng.random(labels.shape) < 0.98, 63, rng.integers(0, 64, labels.shape)).astype(np.uint8)
  assert_same(edt.edt(labels, anisotropy=(4, 4, 40), black_border=True, voxel_graph=graph),
              oracle.edt(labels, anisotropy=(4, 4, 40), black_border=True, voxel_graph=graph), "96x80x72")
  with pytest.raises(TypeError):
    edt.edtsq(np.ones(5, np.uint8), voxel_graph=np.ones(5, np.uint8))
  import torch                                                       # device-resident entry
  got = edt.edt_cuda(torch.from_numpy(labels.astype(np.int16)).cuda(), (4, 4, 40), True, sqrt=True,
                     voxel_graph=torch.from_numpy(graph).cuda())
  assert_same(got.cpu().numpy(), oracle.edt(labels, anisotropy=(4, 4, 40), black_border=True, voxel_graph=graph),
              "edt_cuda voxel_graph")


# ---- randomized differential tests against the oracle -----------------------------------

@pytest.mark.parametrize("block", range(8))
def test_random_vs_oracle(edt, oracle, block):
  for seed in range(block * 40, block * 40 + 40):
    labels, kwargs = cases.random_case(seed)
    what = (seed, labels.shape, labels.dtype.name, kwargs)
    assert_same(edt.edtsq(labels, **kwargs), oracle.edtsq(labels, **kwargs), ("edtsq",) + what)
    if seed % 2 == 0:
      assert_same(edt.edt(labels, **kwargs), oracle.edt(labels, **kwargs), ("edt",) + what)
    if seed % 3 == 0:
      assert_same(edt.sdf(labels, **kwargs), oracle.sdf(labels, **kwargs), ("sdf",) + what)
      assert_same(edt.sdfsq(labels, **kwargs), oracle.sdfsq(labels, **kwargs), ("sdfsq",) + what)


@pytest.mark.parametrize("shape", [(33, 65, 97), (1, 1, 300), (300, 1, 1), (1, 300, 1), (7, 513, 3),
                                   (70, 3, 600), (128, 128, 128), (31, 1030), (1030, 31), (5000,),
                                   (2, 2, 2), (32, 32, 32), (64, 96, 33)])
@pytest.mark.parametrize("kind", ["blocks", "sparse_zero", "iid", "balls"])
def test_shapes_vs_oracle(edt, oracle, shape, kind):
  rng = np.random.default_rng(zlib.crc32(repr((shape, kind)).encode()))
  for dtype, order in ((np.uint32, "F"), (np.uint8, "C")):
    labels = cases.random_volume(rng, shape, kind, dtype)
    labels = np.asfortranarray(labels) if order == "F" else np.ascontiguousarray(labels)
    nd = labels.ndim
    for an in ((1.0, 1.0, 1.0), (4.0, 4.0, 40.0), (0.7, 1.3, 2.9)):
      a = an[0] if nd == 1 else an[:nd]
      for bb in (False, True):
        assert_same(edt.edtsq(labels, anisotropy=a, black_border=bb),
                    oracle.edtsq(labels, anisotropy=a, black_border=bb), (shape, kind, dtype, order, a, bb))


def test_long_axes(edt, oracle):
  """Lines longer than one shared-memory tile (the out-of-place long-line kernel), a first
  axis of 46342 voxels (automated_test.py:819-823) and >4096-voxel distances."""
  arr = np.ones((46342, 1))
  arr[0, 0] = 0
  got = edt.edt(arr)
  assert not np.any(np.isnan(got))
  assert_same(got, oracle.edt(arr), "46342x1 float64")
  col = np.ascontiguousarray(np.ones((1, 46342), dtype=np.uint8).T)       # C order: sx=1, sy=46342
  col[17, 0] = 0
  assert_same(edt.edtsq(col, anisotropy=(3.0, 1.0)), oracle.edtsq(col, anisotropy=(3.0, 1.0)), "1x46342")
  rng = np.random.default_rng(11)
  for shape in ((3, 5, 2500), (2500, 5, 3), (4, 2100), (40, 1100, 3), (3, 1100, 40), (9, 4096), (9, 4097),
                (4096, 9), (2, 3000, 2)):
    lab = cases.random_volume(rng, shape, "blocks", np.uint16)
    lab[lab == 0] = 7        # long runs, no background: inf-rich without a border
    lab.flat[5] = 0
    for bb in (False, True):
      assert_same(edt.edtsq(lab, black_border=bb), oracle.edtsq(lab, black_border=bb), (shape, bb))
  # a big 2-D image whose lines (5000 and 4500 pixels) are longer than a shared-memory tile on the
  # second axis, almost all foreground: the long-line kernel must stay O(n) per line
  img = cases.random_volume(rng, (5000, 4500), "sparse_zero", np.uint8)
  assert_same(edt.edt(img, anisotropy=(1.0, 2.0)), oracle.edt(img, anisotropy=(1.0, 2.0)), "5000x4500 sparse")


def test_label_widths_and_float_labels(edt, oracle):
  rng = np.random.default_rng(2)
  base = rng.integers(0, 4, (19, 23, 29))
  for dtype in (np.uint8, np.int8, np.uint16, np.int16, np.uint32, np.int32, np.uint64, np.int64,
                np.float32, np.float64, bool):
    lab = (base != 0) if dtype is bool else base.astype(dtype)
    assert_same(edt.edtsq(lab, black_border=True), oracle.edtsq(lab, black_border=True), dtype)
  # labels that differ only in high bits / only in sign
  wide = np.where(base == 1, np.uint64(1) << np.uint64(63), np.uint64(base)).astype(np.uint64)
  wide[base == 2] = (np.uint64(1) << np.uint64(63)) + np.uint64(1) << np.uint64(0)
  assert_same(edt.edtsq(wide), oracle.edtsq(wide), "uint64 high bits")
  neg = np.where(base == 1, -1, base).astype(np.int32)
  assert_same(edt.edtsq(neg), oracle.edtsq(neg), "negative int32")
  fl = base.astype(np.float32)
  fl[base == 0] = -0.0                                   # -0.0 is background too
  assert_same(edt.edtsq(fl), oracle.edtsq(fl), "negative zero")
  # bool path == uint8 path (SURVEY.md section 8a: bit-identical in the reference)
  assert_same(edt.edtsq(base != 0), edt.edtsq((base != 0).astype(np.uint8)), "bool vs uint8")
  # unsupported dtype: the reference silently returns zeros (no else branch, src/edt.pyx:670-732)
  assert np.all(edt.edtsq(base.astype(np.float16)) == 0)


def test_non_contiguous_and_lists(edt, oracle):
  rng = np.random.default_rng(4)
  big = rng.integers(0, 3, (20, 30, 14)).astype(np.uint8)
  view = big[::2, 1:-1, ::-1]
  assert not view.flags.c_contiguous and not view.flags.f_contiguous
  assert_same(edt.edtsq(view), oracle.edtsq(view), "strided view")
  before = big.copy()
  edt.edt(big)
  assert np.array_equal(big, before)                       # input never mutated
  assert_same(edt.edtsq([[1, 1, 0], [1, 2, 2]]), oracle.edtsq([[1, 1, 0], [1, 2, 2]]), "list input")
  res = edt.edtsq(np.zeros((128, 128, 128), np.uint32), anisotropy=np.array([4, 4, 40]))   # automated_test.py:729-734
  assert res.shape == (128, 128, 128)


def test_reference_metamorphic_cases(edt, oracle):
  # automated_test.py:723-727
  assert np.all(edt.edt(np.ones((128, 128, 128), np.uint8), black_border=False, anisotropy=(1, 1, 1)) == np.inf)
  # automated_test.py:641-649
  box = np.zeros((15, 15, 15), dtype=bool, order="F")
  box[2:12, 2:12, 5:10] = True
  img = edt.edt(box, anisotropy=(1, 1, 1))
  for i in range(1, 150, 7):
    w = float(i)
    assert np.all(w * img == edt.edt(box, anisotropy=(w, w, w)))
  # automated_test.py:685-700 (C vs F order, lopsided multi-label)
  for size in ((150, 150, 150), (150, 75, 23), (75, 150, 37)):
    def gen(order):
      x = np.zeros(size, dtype=np.uint32, order=order)
      x[0:25, 5:50, 0:25] = 3
      x[25:50, 5:50, 0:25] = 1
      x[60:110, 5:50, 0:25] = 2
      return x
    c, f = edt.edt(gen("C")), edt.edt(gen("F"))
    assert np.array_equal(c, f)
    assert_same(c, oracle.edt(gen("C")), size)
  # automated_test.py:800-817 anisotropy magnitudes
  img = np.ones((100, 97, 99), dtype=np.uint8)
  img[0, 0, 0] = 0
  for weight in (1e-7, 1e-3, 0.1, 1.0, 1000.0, 1e8):
    res = edt.edt(img, anisotropy=(weight,) * 3)
    expected = np.sqrt(sum((weight * (s - 1)) ** 2 for s in img.shape))
    assert np.isclose(res[99, 96, 98], expected, rtol=1e-6)
    assert ulp_diff(res, oracle.edt(img, anisotropy=(weight,) * 3)) <= 1
  # automated_test.py:702-721
  lab = np.ones((256, 256, 256), dtype=np.uint8)
  lab[0, 0, 0] = 0
  lab[-1, -1, -1] = 0
  res = edt.edt(lab, anisotropy=(1000000, 1200000, 40))
  assert np.isfinite(res.max())
  assert ulp_diff(res, oracle.edt(lab, anisotropy=(1000000, 1200000, 40))) <= 1
  # automated_test.py:879-895
  lab2 = np.zeros((9, 7), dtype=np.uint16)
  lab2[3:6, 2:5] = 1
  assert np.array_equal(edt.sdf(lab2), edt.edt(lab2) - edt.edt(lab2 == 0))


# ---- device-resident path and the per-axis entry points ---------------------------------

def test_torch_device_path(edt, oracle):
  import torch
  rng = np.random.default_rng(9)
  lab = cases.random_volume(rng, (40, 50, 60), "blocks", np.int32)
  t = torch.from_numpy(lab).cuda()
  for sqrt, signed, fn in ((False, False, oracle.edtsq), (True, False, oracle.edt),
                           (True, True, oracle.sdf), (False, True, oracle.sdfsq)):
    got = edt.edt_cuda(t, (2.0, 3.0, 5.0), True, sqrt=sqrt, signed=signed)
    assert got.is_cuda and got.dtype == torch.float32
    assert_same(got.cpu().numpy(), fn(lab, anisotropy=(2.0, 3.0, 5.0), black_border=True), (sqrt, signed))
  out = torch.empty(t.shape, dtype=torch.float32, device="cuda")
  again = edt.edt_cuda(t, (2.0, 3.0, 5.0), True, out=out)
  assert again.data_ptr() == out.data_ptr()
  u8 = torch.from_numpy((lab != 0)).cuda()
  assert_same(edt.edt_cuda(u8).cpu().numpy(), oracle.edtsq(lab != 0), "bool tensor")
  # the reference-named functions take device-resident input as it is and answer on the device
  got = edt.sdf(t, anisotropy=(2.0, 3.0, 5.0), black_border=True)
  assert isinstance(got, torch.Tensor) and got.is_cuda
  assert_same(got.cpu().numpy(), oracle.sdf(lab, anisotropy=(2.0, 3.0, 5.0), black_border=True), "sdf(tensor)")

  class Foreign:                         # e.g. a CuPy / Numba array: only __cuda_array_interface__
    def __init__(self, tensor):
      self.keep = tensor
      self.__cuda_array_interface__ = tensor.__cuda_array_interface__

  flab = np.asfortranarray(lab.astype(np.float32) - 1.0)          # float labels, Fortran order, a -0.0 or two
  flab[flab == 0] = -0.0
  ft = torch.from_numpy(flab).cuda()
  assert ft.stride() == torch.from_numpy(flab).stride()
  got = edt.edtsq(Foreign(ft), anisotropy=(2.0, 3.0, 5.0))
  assert got.is_cuda and got.stride() == ft.stride()               # memory order preserved, no copy
  assert_same(got.cpu().numpy(), oracle.edtsq(flab, anisotropy=(2.0, 3.0, 5.0)), "edtsq(F-ordered device array)")
  plane, graph = lab[3] != 0, np.full(lab[3].shape, 63, np.uint8)
  graph[::3, ::4] = 0b111010
  got = edt.edt(torch.from_numpy(plane).cuda(), black_border=True, voxel_graph=torch.from_numpy(graph).cuda())
  assert_same(got.cpu().numpy(), oracle.edt(plane, black_border=True, voxel_graph=graph), "edt(tensor, voxel_graph)")


def test_per_axis_entry_points(edt, oracle):
  """pass_first + pass_later(Y) + pass_later(Z) == transform (the slab-split building blocks)."""
  import ctypes
  import torch
  rng = np.random.default_rng(10)
  lab = np.asfortranarray(cases.random_volume(rng, (37, 41, 29), "blocks", np.uint32))
  sx, sy, sz = lab.shape
  t = torch.from_numpy(np.ascontiguousarray(lab.T)).cuda()        # memory = x fastest
  f = torch.empty(t.shape, dtype=torch.float32, device="cuda")
  lib = edt._lib()
  s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  assert lib.edtb200_pass_first(t.data_ptr(), 4, sx, sy, sz, 2.0, 1, 0, f.data_ptr(), 0, s) == 0
  assert lib.edtb200_pass_later(t.data_ptr(), 4, 1, sx, sy, sz, 3.0, 1, 1, 0, f.data_ptr(), 0, s) == 0
  assert lib.edtb200_pass_later(t.data_ptr(), 4, 2, sx, sy, sz, 5.0, 1, 1, 1, f.data_ptr(), 0, s) == 0
  torch.cuda.synchronize()
  got = np.asfortranarray(f.cpu().numpy().T)
  assert_same(got, oracle.edt(lab, anisotropy=(2.0, 3.0, 5.0), black_border=True), "per-axis")


# ---- BASELINE.json sizes: closed forms and size-independent properties ------------------

def box_closed_form(shape, anisotropy):
  """edtsq of an all-foreground box with black_border=True: the nearest background is the
  closest face, so the value is (min over axes of w*min(i+1, n-i))^2 -- exact in float32 for
  integer weights."""
  axes = []
  for n, w in zip(shape, anisotropy):
    i = np.arange(n, dtype=np.float32)
    axes.append((np.float32(w) * np.minimum(i + 1, n - i)) ** 2)
  gx, gy, gz = np.meshgrid(*axes, indexing="ij", sparse=True)
  return np.minimum(np.minimum(gx, gy), gz)


def test_cfg3_box_512_uint8(edt):
  # BASELINE.json configs[2]: 512^3 uint8 ones, anisotropy (6,6,30), black_border, edt vs edtsq
  lab = np.ones((512, 512, 512), dtype=np.uint8, order="F")
  want = np.asfortranarray(np.broadcast_to(box_closed_form(lab.shape, (6, 6, 30)), lab.shape))
  got = edt.edtsq(lab, anisotropy=(6, 6, 30), black_border=True)
  assert got.max() == 2359296.0
  assert np.array_equal(got, want)
  got = edt.edt(lab, anisotropy=(6, 6, 30), black_border=True)
  assert np.array_equal(got, np.sqrt(want))


def test_cfg2_512_uint32_properties(edt, oracle):
  # BASELINE.json configs[1]: 512^3 uint32 random 0..255, anisotropy (1,1,1)
  rng = np.random.default_rng(0)
  lab = np.asfortranarray(rng.integers(0, 256, (512, 512, 512), dtype=np.uint32))
  got = edt.edtsq(lab, anisotropy=(1, 1, 1))
  assert got.flags.f_contiguous and got.shape == lab.shape
  assert np.all(got[lab == 0] == 0) and np.all(got[lab != 0] >= 1)
  # a slab of full x/y extent against the oracle (z-faces differ, so compare an interior band
  # of a transform recomputed on the slab with the same neighbours: use black_border on both)
  slab = np.asfortranarray(lab[:, :, :24])
  assert_same(edt.edtsq(slab, black_border=True), oracle.edtsq(slab, black_border=True), "512x512x24 slab")
  # relabelling invariance: any injective map on non-zero labels leaves the result unchanged
  perm = rng.permutation(np.arange(1, 256, dtype=np.uint32)) * np.uint32(16777259)
  lut = np.concatenate([[np.uint32(0)], perm]).astype(np.uint32)
  assert np.array_equal(edt.edtsq(np.asfortranarray(lut[lab])), got)
  # axis-order invariance: the C-ordered transpose holds the same bytes with axes reversed
  assert np.array_equal(edt.edtsq(lab.T), got.T)
  # exact scaling by a power of two
  assert np.array_equal(edt.edtsq(lab, anisotropy=(4, 4, 4)), got * np.float32(16))


def test_blocks_256_vs_oracle(edt, oracle):
  rng = np.random.default_rng(0)
  small = rng.integers(0, 256, (8, 8, 8), dtype=np.uint32)
  lab = np.asfortranarray(np.repeat(np.repeat(np.repeat(small, 32, 0), 32, 1), 32, 2))   # 256^3, 32^3 blocks
  for bb in (False, True):
    assert_same(edt.edtsq(lab, anisotropy=(1, 1, 1), black_border=bb),
                oracle.edtsq(lab, anisotropy=(1, 1, 1), black_border=bb), ("blocks256", bb))
  assert_same(edt.sdf(lab, anisotropy=(4, 4, 40)), oracle.sdf(lab, anisotropy=(4, 4, 40)), "blocks256 sdf")


def test_cpp_shim_header(edt, oracle, tmp_path):
  """include/edt.hpp: edt::edt<T> / edt::edtsq<T> with the reference's C++ signature
  (src/edt.hpp:836-844, 907-922), compiled with g++ against libedt_b200.so."""
  import shutil
  import subprocess
  if shutil.which("g++") is None:
    pytest.skip("no g++")
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  src = tmp_path / "shim.cpp"
  src.write_text(r'''
#include "edt.hpp"
#include <cstdio>
#include <cstdlib>
int main(int argc, char** argv) {
  const int sx = 19, sy = 11, sz = 7;
  std::vector<uint16_t> lab(sx * sy * sz);
  FILE* fi = fopen(argv[1], "rb"); if (!fi || fread(lab.data(), 2, lab.size(), fi) != lab.size()) return 2; fclose(fi);
  float* a = edt::edtsq<uint16_t>(lab.data(), sx, sy, sz, 2.f, 3.f, 5.f, true);
  float* b = edt::edt<uint16_t>(lab.data(), sx, sy, sz, 2.f, 3.f, 5.f, false, 4);
  std::vector<float> c(lab.size());
  float* cret = edt::edtsq<uint16_t>(lab.data(), sx, sy, sz, 2.f, 3.f, 5.f, true, 1, c.data());
  if (cret != c.data()) return 3;
  FILE* fo = fopen(argv[2], "wb");
  fwrite(a, 4, lab.size(), fo); fwrite(b, 4, lab.size(), fo); fwrite(c.data(), 4, lab.size(), fo); fclose(fo);
  delete[] a; delete[] b;
  return 0;
}
''')
  exe = tmp_path / "shim"
  libdir = os.path.dirname(edt.library_path())
  subprocess.run(["g++", "-std=c++17", "-I", os.path.join(root, "include"), str(src), "-L", libdir,
                  "-ledt_b200", "-Wl,-rpath," + libdir, "-o", str(exe)], check=True)
  rng = np.random.default_rng(21)
  lab = np.asfortranarray(rng.integers(0, 4, (19, 11, 7)).astype(np.uint16))      # x fastest
  (tmp_path / "in.bin").write_bytes(lab.tobytes(order="F"))
  subprocess.run([str(exe), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], check=True)
  out = np.fromfile(tmp_path / "out.bin", dtype=np.float32).reshape(3, -1)
  sq = oracle.edtsq(lab, anisotropy=(2, 3, 5), black_border=True).ravel(order="F")
  assert np.array_equal(out[0], sq) and np.array_equal(out[2], sq)
  assert np.array_equal(out[1], oracle.edt(lab, anisotropy=(2, 3, 5), black_border=False).ravel(order="F"))


def test_cpp_voxel_graph_shim(edt, oracle, tmp_path):
  """include/edt_voxel_graph.hpp: pyedt::_edt3dsq_voxel_graph / _edt2dsq_voxel_graph with the
  reference's signatures (src/edt_voxel_graph.hpp:54-236), compiled with g++."""
  import shutil
  import subprocess
  if shutil.which("g++") is None:
    pytest.skip("no g++")
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  src = tmp_path / "vg.cpp"
  src.write_text(r'''
#include "edt_voxel_graph.hpp"
#include <cstdio>
#include <vector>
int main(int argc, char** argv) {
  const int sx = 13, sy = 9, sz = 6;
  std::vector<float> lab(sx * sy * sz);
  std::vector<uint8_t> graph(lab.size());
  FILE* fi = fopen(argv[1], "rb");
  if (!fi || fread(lab.data(), 4, lab.size(), fi) != lab.size()) return 2;
  if (fread(graph.data(), 1, graph.size(), fi) != graph.size()) return 2;
  fclose(fi);
  float* a = pyedt::_edt3dsq_voxel_graph<float, uint8_t>(lab.data(), graph.data(), sx, sy, sz, 2.f, 3.f, 5.f, true);
  float* b = pyedt::_edt3d_voxel_graph<float>(lab.data(), graph.data(), sx, sy, sz, 2.f, 3.f, 5.f, true);
  std::vector<float> c(sx * sy);
  float* cret = pyedt::_edt2dsq_voxel_graph<float>(lab.data(), graph.data(), sx, sy, 1.f, 1.f, false, c.data());
  if (cret != c.data()) return 3;
  FILE* fo = fopen(argv[2], "wb");
  fwrite(a, 4, lab.size(), fo); fwrite(b, 4, lab.size(), fo); fwrite(c.data(), 4, c.size(), fo); fclose(fo);
  delete[] a; delete[] b;
  return 0;
}
''')
  exe = tmp_path / "vg"
  libdir = os.path.dirname(edt.library_path())
  subprocess.run(["g++", "-std=c++17", "-I", os.path.join(root, "include"), str(src), "-L", libdir,
                  "-ledt_b200", "-Wl,-rpath," + libdir, "-o", str(exe)], check=True)
  rng = np.random.default_rng(23)
  lab = np.asfortranarray((rng.integers(-1, 3, (13, 9, 6)) * (rng.random((13, 9, 6)) < 0.9)).astype(np.float32))
  graph = np.asfortranarray(np.where(rng.random(lab.shape) < 0.7, 63, rng.integers(0, 64, lab.shape)).astype(np.uint8))
  (tmp_path / "in.bin").write_bytes(lab.tobytes(order="F") + graph.tobytes(order="F"))
  subprocess.run([str(exe), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], check=True)
  out = np.fromfile(tmp_path / "out.bin", dtype=np.float32)
  n = lab.size
  sq = oracle.edtsq(lab, anisotropy=(2, 3, 5), black_border=True, voxel_graph=graph)
  assert np.array_equal(out[:n], sq.ravel(order="F"))
  assert np.array_equal(out[n:2 * n], np.sqrt(sq).ravel(order="F"))
  plane = oracle.edtsq(lab[:, :, 0], anisotropy=(1, 1), black_border=False, voxel_graph=graph[:, :, 0])
  assert np.array_equal(out[2 * n:], plane.ravel(order="F"), equal_nan=True)


def test_cfg4_1024_device_resident(edt):
  """BASELINE.json configs[3] size (1024^3), entirely on the device (8 GiB resident): closed
  form for the all-foreground box, and label-permutation / power-of-two scaling invariance for
  iid uint32 labels (size-independent properties; the oracle would need minutes here)."""
  import torch
  n = 1024
  dev = torch.device("cuda", 0)
  ones = torch.ones((n, n, n), dtype=torch.uint8, device=dev)
  got = edt.edt_cuda(ones, (3.0, 2.0, 1.0), True)
  del ones
  i = torch.arange(n, device=dev, dtype=torch.float32)
  edge = torch.minimum(i + 1, n - i)
  want = torch.minimum(torch.minimum(((3.0 * edge) ** 2).view(n, 1, 1), ((2.0 * edge) ** 2).view(1, n, 1)),
                       (edge ** 2).view(1, 1, n))
  assert bool((got == want).all())
  del got, want
  g = torch.Generator(device=dev)
  g.manual_seed(0)
  lab = torch.randint(0, 256, (n, n, n), dtype=torch.int32, device=dev, generator=g)
  base = edt.edt_cuda(lab)
  assert bool((base[lab == 0] == 0).all()) and float(base.max()) < 64.0
  lut = torch.cat([torch.zeros(1, dtype=torch.int32, device=dev),
                   (torch.randperm(255, device=dev, generator=g).to(torch.int32) + 1) * 16777259])
  relabelled = lut[lab]
  assert bool((edt.edt_cuda(relabelled) == base).all())
  del relabelled
  assert bool((edt.edt_cuda(lab, (4.0, 4.0, 4.0)) == base * 16.0).all())


def test_transform_batch_pipeline(edt, oracle):
  """edtb200_transform_batch: many host volumes through two device slots; every result must equal
  the single-call result (and the oracle's), for pageable and pinned buffers, odd counts, count 1."""
  import torch
  rng = np.random.default_rng(41)
  shape = (70, 96, 130)                      # 3.5 MB of uint32: above the direct-copy threshold for float32 too
  vols = [cases.random_volume(rng, shape, kind, np.uint32) for kind in ("blocks", "iid", "balls", "few", "blocks")]
  vols = [np.asfortranarray(v) for v in vols]
  for count in (5, 1, 2):
    got = edt.transform_batch(vols[:count], (2.0, 1.0, 3.0), True, sqrt=True)
    assert len(got) == count
    for v, g in zip(vols, got):
      assert g.flags.f_contiguous
      assert_same(g, oracle.edt(v, anisotropy=(2.0, 1.0, 3.0), black_border=True), ("batch", count))
  # bigger volumes (staged copies, 3 x 32 MiB buffers per direction), pageable and pinned outputs
  big = [np.ascontiguousarray(rng.integers(0, 5, (160, 256, 320), dtype=np.int64).astype(np.uint16)) for _ in range(4)]
  want = [edt.sdfsq(v, anisotropy=(1.0, 2.0, 1.0)) for v in big]
  got = edt.transform_batch(big, (1.0, 2.0, 1.0), signed=True)
  pinned = [torch.empty(big[0].shape, dtype=torch.float32, pin_memory=True).numpy() for _ in big]
  got_pinned = edt.transform_batch(big, (1.0, 2.0, 1.0), signed=True, outs=pinned)
  for w, g, gp in zip(want, got, got_pinned):
    assert_same(g, w, "batch pageable")
    assert_same(gp, w, "batch pinned")
  assert got_pinned[0] is pinned[0]
  assert edt.transform_batch([]) == []
  with pytest.raises(ValueError):
    edt.transform_batch([vols[0], vols[1][:10]])


def test_more_than_2_31_voxels(edt):
  """528 x 2048 x 2048 = 2.2e9 voxels (64-bit voxel indices everywhere), device-resident, against
  closed forms: isolated boxes of edge 48 (long runs: chunk hulls + stitching) and 16 (short runs),
  anisotropic, black border; labels of neighbouring boxes always differ."""
  import torch
  dev = torch.device("cuda", 0)
  shape = (528, 2048, 2048)
  w = (3.0, 1.0, 2.0)

  def axis_terms(n, edge, weight):
    i = torch.arange(n, device=dev, dtype=torch.int64)
    p = i % edge
    length = torch.minimum(torch.full_like(i, edge), n - (i - p))      # the last box may be cut by the volume
    d = torch.minimum(p + 1, length - p).to(torch.float32)
    return (weight * d) ** 2, (i // edge)

  for edge in (48, 16):
    (tz, bz), (ty, by), (tx, bx) = (axis_terms(n, edge, wt) for n, wt in zip(shape, w))
    lab = (1 + (bz.view(-1, 1, 1) + 2 * by.view(1, -1, 1) + 4 * bx.view(1, 1, -1)) % 8).to(torch.uint8)
    assert lab.numel() > 2**31
    got = edt.edt_cuda(lab, w, True)
    del lab
    want = torch.minimum(torch.minimum(tz.view(-1, 1, 1), ty.view(1, -1, 1)).expand(shape), tx.view(1, 1, -1))
    bad = int((got != want).sum().item())
    assert bad == 0, (edge, bad)
    del got, want
    torch.cuda.empty_cache()


def test_current_device_and_threads(edt, oracle):
  """The library must leave the caller's current CUDA device alone and survive concurrent calls."""
  import threading
  import torch
  before = torch.cuda.current_device()
  rng = np.random.default_rng(31)
  labs = [cases.random_volume(rng, (40, 33, 29), kind, np.uint16) for kind in ("blocks", "iid", "balls", "few")]
  want = [oracle.edtsq(l, anisotropy=(1, 2, 3), black_border=True) for l in labs]
  got = [None] * len(labs)

  def work(i):
    for _ in range(3):
      got[i] = edt.edtsq(labs[i], anisotropy=(1, 2, 3), black_border=True)

  threads = [threading.Thread(target=work, args=(i,)) for i in range(len(labs))]
  for t in threads:
    t.start()
  for t in threads:
    t.join()
  for g, w in zip(got, want):
    assert_same(g, w, "concurrent")
  assert torch.cuda.current_device() == before
