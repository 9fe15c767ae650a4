"""GPU tests (-m gpu) of the X kernel that writes the run-start planes (first_axis_planes_kernel) at the
edges of its work: bands of W = 8 rows with a halo row, runs of (band, z) items split over one wave
of CTAs, and a ring of label stages.  Every volume has random runs of 1 to 4 equal labels along y and
z (so that a wrong start bit changes the result) and noise along x; each is transformed right after
a noise volume, so that the planes are taken, and compared with the oracle bit for bit.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

WIDE = (np.uint32, np.uint64)
W = 8                                          # rows per band (launch_first_vec)
SY = (1, W - 1, W, W + 1, 3 * W + 5)
SZ = (1, 2, 3, 257)
SX = (4, 128, 132, 508, 512)


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
    for sz in SZ:
      lab = runs_volume((sz, sy, sx), dtype, sx * 1000 + sy * 10 + sz)
      for border in (False, True):
        got = after_noise(edt, dtype, lab, anisotropy=(1.0, 2.0, 3.0), black_border=border)
        want = oracle.edtsq(lab, anisotropy=(1.0, 2.0, 3.0), black_border=border)
        assert np.array_equal(got, want), ((sz, sy, sx), border, int((got != want).sum()))


@pytest.mark.parametrize("sx", SX)
@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_2d_band_edges(edt, oracle, dtype, sx):
  for sy in SY + (4 * W, 40 * W + 3):
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
