"""GPU tests (-m gpu) of the run-start bit planes: on predicted label noise with labels of 4 or 8
bytes, the X pass writes one run-start bit per voxel and later axis, and the later passes read those
instead of the labels.  The prediction comes from the previous transform on the device, so every
volume here is transformed twice in a row and the second result is compared with the oracle bit for
bit: ragged extents (sx, sy, sz not multiples of 32 or 128), 2-D and 3-D, black_border, sqrt, both
label widths, the device-resident and batch entry points, shapes in turn, and a structured volume
right after noise (planes written for a prediction that turns out wrong).

At the edges of the plane-writing X kernel's work (bands of 8 slices, y-chunks, 32-voxel words of a
row), volumes with random runs of 1 to 4 equal labels along y and z (so that a wrong start bit changes
the result) and noise along x, each transformed right after a noise volume.
"""
import numpy as np
import pytest

from noise_cases import BAND, WIDE, noise, twice

pytestmark = pytest.mark.gpu

# around the band edges, and sy = 134 cut into two y-chunks
SY = (1, 7, 8, 9, 29, 134)
SZ = (1, 2, 3, BAND - 1, BAND, BAND + 1, 2 * BAND + 1, 257)
SX = (4, 128, 132, 508, 512)


def blocky(shape, dtype, seed, cell=3):
  rng = np.random.default_rng(seed)
  out = rng.integers(0, 5, [-(-s // cell) for s in shape]).astype(dtype)
  for ax in range(len(shape)):
    out = np.repeat(out, cell, axis=ax)
  return np.ascontiguousarray(out[tuple(slice(0, s) for s in shape)])


# C order: the last extent is x
SHAPES_3D = [(33, 37, 44), (17, 70, 132), (40, 33, 256), (9, 65, 100), (20, 31, 512), (5, 6, 4)]


@pytest.mark.parametrize("shape", SHAPES_3D, ids=["x".join(map(str, s)) for s in SHAPES_3D])
@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_3d_noise_bit_exact(edt, oracle, shape, dtype):
  lab = noise(shape, dtype, sum(shape))
  for border in (False, True):
    for fn in ("edtsq", "edt"):
      got = twice(getattr(edt, fn), lab, anisotropy=(1.0, 2.0, 3.0), black_border=border)
      want = getattr(oracle, fn)(lab, anisotropy=(1.0, 2.0, 3.0), black_border=border)
      assert np.array_equal(got, want), (fn, border, int((got != want).sum()))


def test_noise_takes_the_label_noise_plan(edt):
  lab = noise((16, 40, 256), np.uint32, 1)
  twice(edt.edtsq, lab)
  info = edt.last_later_launch()
  assert info["kernel"] == "tile" and info["ctas"] == 2, info


SHAPES_2D = [(37, 44), (70, 132), (65, 512), (3, 4)]


@pytest.mark.parametrize("shape", SHAPES_2D, ids=["x".join(map(str, s)) for s in SHAPES_2D])
@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_2d_noise_bit_exact(edt, oracle, shape, dtype):
  lab = noise(shape, dtype, sum(shape) + 7)
  for border in (False, True):
    got = twice(edt.edtsq, lab, anisotropy=(1.5, 1.0), black_border=border)
    assert np.array_equal(got, oracle.edtsq(lab, anisotropy=(1.5, 1.0), black_border=border)), border


def test_signed_and_narrow_labels_after_noise(edt, oracle):
  # planes are not taken for these; the prediction is still "noise"
  lab = noise((20, 33, 132), np.uint32, 3)
  edt.edtsq(lab)
  assert np.array_equal(edt.sdf(lab, black_border=True), oracle.sdf(lab, black_border=True))
  for dtype in (np.uint8, np.uint16):
    small = noise((20, 33, 132), dtype, 4) if dtype == np.uint16 else \
        np.random.default_rng(4).integers(0, 256, (20, 33, 132)).astype(np.uint8)
    assert np.array_equal(twice(edt.edtsq, small), oracle.edtsq(small)), dtype


def test_structured_right_after_noise(edt, oracle):
  edt.edtsq(noise((24, 40, 128), np.uint32, 5))
  lab = blocky((24, 40, 128), np.uint32, 6)
  assert np.array_equal(edt.edtsq(lab, black_border=True), oracle.edtsq(lab, black_border=True))


def test_shapes_in_turn(edt, oracle):
  for shape in [(20, 30, 40), (64, 64, 512), (7, 9, 12), (33, 40, 256), (20, 30, 40)]:
    lab = noise(shape, np.uint32, sum(shape))
    assert np.array_equal(twice(edt.edtsq, lab, black_border=True), oracle.edtsq(lab, black_border=True)), shape


def test_device_resident_and_batch(edt, oracle):
  torch = pytest.importorskip("torch")
  lab = noise((24, 40, 68), np.int32, 8)
  t = torch.from_numpy(lab).cuda()
  got = twice(edt.edt_cuda, t, sqrt=True).cpu().numpy()
  assert np.array_equal(got, oracle.edt(lab.astype(np.uint32)))
  batch = [noise((24, 40, 68), np.uint32, s) for s in range(4)]
  outs = twice(edt.transform_batch, batch, black_border=True)
  for v, o in zip(batch, outs):
    assert np.array_equal(o, oracle.edtsq(v, black_border=True))


def run_ids(rng, n, m):
  """m independent maps of n positions to run ids, with runs of 1 to 4 positions."""
  ends = np.cumsum(rng.integers(1, 5, (m, n)), axis=1)
  starts = np.zeros((m, n), bool)
  rows, cols = np.nonzero(ends < n)
  starts[rows, ends[rows, cols]] = True
  return np.cumsum(starts, axis=1)


def runs_volume(shape, dtype, seed):
  """Noise along x (the last extent), runs of 1 to 4 equal labels along the others, every x its own
  runs; a few background voxels."""
  rng = np.random.default_rng(seed)
  sx = shape[-1]
  base = rng.integers(1, 1 << 20, shape).astype(dtype)
  base[rng.random(shape) < 0.02] = 0
  x = np.arange(sx)
  if len(shape) == 2:
    iy = run_ids(rng, shape[0], sx).T
    return np.ascontiguousarray(base[iy, x[None, :]])
  iz, iy = run_ids(rng, shape[0], sx).T, run_ids(rng, shape[1], sx).T
  return np.ascontiguousarray(base[iz[:, None, :], iy[None, :, :], x[None, None, :]])


def after_noise(edt, dtype, lab, **kw):
  """edtsq of lab right after one of label noise: the run statistic then predicts noise."""
  rng = np.random.default_rng(7)
  edt.edtsq(rng.integers(1, 1 << 20, (4, 9, 512)).astype(dtype))
  return edt.edtsq(lab, **kw)


@pytest.mark.parametrize("sx", SX)
@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_3d_band_and_segment_edges(edt, oracle, dtype, sx):
  for sy in SY:
    for sz in SZ if sy < 134 else SZ[:-1]:
      lab = runs_volume((sz, sy, sx), dtype, sx * 1000 + sy * 10 + sz)
      for border in (False, True):
        got = after_noise(edt, dtype, lab, anisotropy=(1.0, 2.0, 3.0), black_border=border)
        want = oracle.edtsq(lab, anisotropy=(1.0, 2.0, 3.0), black_border=border)
        assert np.array_equal(got, want), ((sz, sy, sx), border, int((got != want).sum()))


@pytest.mark.parametrize("sx", SX)
@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_2d_band_edges(edt, oracle, dtype, sx):
  for sy in SY + (32, 323, 201):
    lab = runs_volume((sy, sx), dtype, sx * 100 + sy)
    for border in (False, True):
      got = after_noise(edt, dtype, lab, anisotropy=(1.5, 1.0), black_border=border)
      want = oracle.edtsq(lab, anisotropy=(1.5, 1.0), black_border=border)
      assert np.array_equal(got, want), ((sy, sx), border, int((got != want).sum()))


def test_planes_beyond_2_31_voxels(edt, oracle):
  """512 x 512 x 8209 four-byte labels (more than 2^31 voxels) on the plane path: every 16th z plane
  is background, so each period of 16 planes and the background plane after it is transformed as
  the oracle transforms that tile on its own; the Y pass reads its plane (the Z pass, on lines of
  more than 4096 voxels, reads the labels).  Compared on the device, tile by tile."""
  import torch
  free, _ = torch.cuda.mem_get_info()
  if free < (40 << 30):
    pytest.skip("needs 40 GB of free device memory, %.1f GB free" % (free / 2**30))
  period, sy, sx = 16, 512, 512
  sz = period * 513 + 1
  tile = runs_volume((period, sy, sx), np.uint32, 41)
  tile[0] = 0
  want_t = oracle.edtsq(tile[np.arange(period + 1) % period], anisotropy=(1.0, 2.0, 3.0))
  want = torch.from_numpy(want_t).cuda()
  lab_t = torch.from_numpy(tile.view(np.int32)).cuda()[torch.arange(sz, device="cuda") % period]
  assert lab_t.numel() > 2**31
  torch.cuda.synchronize()
  edt.edt_cuda(torch.from_numpy(np.random.default_rng(3).integers(1, 1 << 20, (4, 9, 512)).astype(np.int32)).cuda())
  got = edt.edt_cuda(lab_t, anisotropy=(1.0, 2.0, 3.0))
  torch.cuda.synchronize()
  for z0 in range(0, sz - 1, period):
    if not torch.equal(got[z0:z0 + period], want[:period]):
      bad = (got[z0:z0 + period] != want[:period]).nonzero()[0].tolist()
      raise AssertionError("z %d y %d x %d differs" % (z0 + bad[0], bad[1], bad[2]))
  assert torch.equal(got[sz - 1], want[period])
  del lab_t, got
