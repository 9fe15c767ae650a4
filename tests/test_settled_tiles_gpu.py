"""GPU tests (-m gpu) of settled-tile skipping: on predicted label noise the X pass also writes, per
row and 32-voxel x-segment, whether every voxel of the segment ends it at f <= w2 of the Y / Z pass;
a later pass leaves such voxels as they are, so it skips every tile whose segments are all settled,
and the Y pass sets the Z pass's bits of the rows it settles.  The volumes are label noise with
planted unsettled voxels (x-runs of 3 and 5, at the row ends and across segment edges, with y-runs of
one and of two rows, background triples, a tile with more than 32 unsettled rows), transformed twice
so that the second transform takes the label-noise plan, and compared with the oracle bit for bit.
The plan's `settled` field says whether the skip was armed: on int_hull passes without an epilogue.
"""
import numpy as np
import pytest

from noise_cases import FRESH, WIDE, noise, twice

pytestmark = pytest.mark.gpu


def planted(shape, dtype, seed):
  """Label noise (C order, x last) with unsettled voxels planted into it.  With w_x = 1 a noise voxel
  ends the X pass at f = 1; the middle voxel of an x-run of three at 4, of an x-run of five at 9."""
  lab = noise(shape, dtype, seed)
  rng = np.random.default_rng(seed + 1)
  vol = lab.reshape((-1,) + lab.shape[-2:])       # 2-D: one slice
  nz, sy, sx = vol.shape
  fresh = iter(range(FRESH, FRESH + 10 ** 6))
  # row ends, segment edges, and the first and last voxels of a row whose Z tiles (32 consecutive
  # x of the x-y plane) reach into the next row when sx is not a multiple of 32
  starts = sorted({0, 1, max(sx - 3, 0)} | {x for x in (29, 30, 31, 32, sx - 4) if 0 <= x and x + 3 <= sx})
  per_slice = 8 if sx >= 32 else 2                # narrow rows stay label noise
  for z in range(nz):
    for y in rng.choice(sy, size=min(sy, per_slice), replace=False):
      x0 = int(rng.choice(starts))
      kind = int(rng.integers(0, 5))
      if kind == 0:                                   # x-run of 3, y-run of 1: the Y pass settles it
        vol[z, y, x0:x0 + 3] = next(fresh)
      elif kind in (1, 2):                            # y-run of 3: the middle row reaches the Z pass
        vol[z, y:y + 3, x0:x0 + 3] = next(fresh)      # at f = 4 when w_y = 1
      elif kind == 3 and sx >= 5:                     # x-run of 5: f = 4 and f = 9
        x0 = int(rng.integers(0, sx - 4))
        vol[z, y, x0:x0 + 5] = next(fresh)
      else:                                           # background triple
        vol[z, y, x0:x0 + 3] = 0
    if sx >= 32 and sy >= 4:
      # one Y tile (this z, segment 0) that runs when w_y = 2 (an x-run of five: f = 9 > 4) and holds
      # another row at f = 4 after the Y pass: with w_z = 1 its Z bit must stay clear in the refresh
      ya, yb = rng.choice(sy, size=2, replace=False)
      vol[z, ya, 0:5] = next(fresh)
      vol[z, yb, 1:4] = next(fresh)
  # one tile (z = 0, segment 0) with more than 32 rows left unsettled by the X pass
  if sx >= 32:
    for y in range(min(sy, 40)):
      vol[0, y, 0:3] = next(fresh)
  return lab


def per_slice_2d(oracle, lab, w, border):
  """The X and Y passes of a 3-D transform: the 2-D transform of every z slice."""
  return np.stack([oracle.edtsq(np.ascontiguousarray(sl), anisotropy=w[1:], black_border=border) for sl in lab])


def unsettled_everywhere(shape, dtype, seed):
  """Label noise with one x-run of three in every 32-voxel segment of every row: every segment
  holds a voxel with f = 4, and the volume is still label noise."""
  lab = noise(shape, dtype, seed)
  rng = np.random.default_rng(seed + 1)
  sx = shape[-1]
  rows = lab.reshape(-1, sx)
  fresh = FRESH
  for s0 in range(0, sx, 32):
    x0 = s0 + rng.integers(0, min(32, sx - s0) - 2, rows.shape[0])
    for d in range(3):
      rows[np.arange(rows.shape[0]), x0 + d] = np.arange(fresh, fresh + rows.shape[0])
    fresh += rows.shape[0]
  return lab


# (sz, sy, sx): sx in 4, 36, 132, 500, 512; sy and sz not multiples of 8.  Rows of fewer than 32
# voxels are not label noise without a black border (the row's first voxel starts no run), and in 2-D
# they take no 32-wide TMA tiles: only exactness there
SHAPES_3D = [(19, 45, 4), (23, 37, 36), (13, 70, 132), (9, 41, 500), (7, 67, 512)]
# anisotropy in array order (z, y, x); in parentheses (w_x, w_y, w_z).  Tiles are settled only where
# the noise voxels' f = w_x^2 is at most w2 of the pass.
ANISO = [(1.0, 1.0, 1.0),      # (1, 1, 1)
         (1.0, 2.0, 1.0),      # (1, 2, 1): w_y > w_z, values in (w_z^2, w_y^2] after Y
         (2.0, 1.0, 1.0),      # (1, 1, 2)
         (3.0, 2.0, 1.0),      # (1, 2, 3)
         (1.0, 2.0, 3.0)]      # (3, 2, 1): nothing settled
# where the Z pass must change voxels that the planted volumes bring to it unsettled
Z_CHANGES = [(1.0, 1.0, 1.0), (1.0, 2.0, 1.0)]


@pytest.mark.parametrize("shape", SHAPES_3D, ids=["x".join(map(str, s)) for s in SHAPES_3D])
@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_3d_planted_bit_exact(edt, oracle, shape, dtype):
  lab = planted(shape, dtype, sum(shape))
  for border in (False, True):
    for w in ANISO:
      got = twice(edt.edtsq, lab, anisotropy=w, black_border=border)
      if shape[-1] >= 32:
        assert edt.last_later_launch()["settled"] == 1, (w, border, edt.last_later_launch())
      want = oracle.edtsq(lab, anisotropy=w, black_border=border)
      assert np.array_equal(got, want), (w, border, int((got != want).sum()))
      if w in Z_CHANGES and shape[-1] >= 32:
        assert np.any(want != per_slice_2d(oracle, lab, w, border)), (w, border)   # the case is exercised
    # sqrt in the Z pass's store: the Z pass does not skip
    got = twice(edt.edt, lab, anisotropy=(1.0, 2.0, 3.0), black_border=border)
    assert edt.last_later_launch()["settled"] == 0
    assert np.array_equal(got, oracle.edt(lab, anisotropy=(1.0, 2.0, 3.0), black_border=border)), border


SHAPES_2D = [(45, 4), (37, 36), (70, 132), (41, 500), (67, 512)]


@pytest.mark.parametrize("shape", SHAPES_2D, ids=["x".join(map(str, s)) for s in SHAPES_2D])
@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_2d_planted_bit_exact(edt, oracle, shape, dtype):
  lab = planted(shape, dtype, sum(shape) + 3)
  for border in (False, True):
    for w in ((1.0, 1.0), (2.0, 1.0), (1.0, 3.0)):
      got = twice(edt.edtsq, lab, anisotropy=w, black_border=border)
      if shape[-1] >= 32:
        assert edt.last_later_launch()["settled"] == 1, (w, border)
      want = oracle.edtsq(lab, anisotropy=w, black_border=border)
      assert np.array_equal(got, want), (w, border, int((got != want).sum()))


@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_every_segment_unsettled(edt, oracle, dtype):
  for shape in [(11, 45, 132), (7, 37, 512)]:
    lab = unsettled_everywhere(shape, dtype, sum(shape))
    for border in (False, True):
      got = twice(edt.edtsq, lab, black_border=border)
      assert edt.last_later_launch()["settled"] == 1
      assert np.array_equal(got, oracle.edtsq(lab, black_border=border)), (shape, border)


@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_stack_planted(edt, oracle, dtype):
  for shape in [(9, 37, 36), (5, 41, 500)]:
    vols = [planted(shape, dtype, 100 * b + shape[-1]) for b in range(3)]
    stack = np.ascontiguousarray(np.stack(vols, axis=0))
    for border in (False, True):
      got = twice(edt.edtsq, stack, anisotropy=(1.0, 2.0, 3.0), black_border=border, stacked=True)
      assert edt.last_later_launch()["settled"] == 1
      for b, v in enumerate(vols):
        want = oracle.edtsq(v, anisotropy=(1.0, 2.0, 3.0), black_border=border)
        assert np.array_equal(got[b], want), (shape, border, b)


def test_gates(edt, oracle):
  lab = planted((13, 70, 132), np.uint32, 5)
  # float samples: no integer hull, no skip
  got = twice(edt.edtsq, lab, anisotropy=(1.5, 1.0, 1.0))
  assert edt.last_later_launch()["settled"] == 0
  assert np.array_equal(got, oracle.edtsq(lab, anisotropy=(1.5, 1.0, 1.0)))
  got = twice(edt.edtsq, lab, anisotropy=(1.0, 1.0, 1.5))
  assert edt.last_later_launch()["settled"] == 0
  assert np.array_equal(got, oracle.edtsq(lab, anisotropy=(1.0, 1.0, 1.5)))
  # signed transforms take no planes
  got = twice(edt.sdf, lab, black_border=True)
  assert edt.last_later_launch()["settled"] == 0
  assert np.array_equal(got, oracle.sdf(lab, black_border=True))
  # the same volume again: armed
  got = twice(edt.edtsq, lab)
  assert edt.last_later_launch()["settled"] == 1
  assert np.array_equal(got, oracle.edtsq(lab))
