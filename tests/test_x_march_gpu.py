"""GPU tests (-m gpu) of the plane-writing X pass whose warps march along y (first_axis_planes_kernel): a
CTA owns a band of 8 slices and a y-chunk of rows, stages one row of every slice of the band plus the
halo row of the slice below it per step, and reads each chunk's leading row ya - 1 and trailing row
yb + 1 for their compares only.  In 2-D the warps take independent (image, y-chunk) sequences.  Where
a voxel's y-run is one row long it stores min(f, w_y^2), exactly what the Y pass would leave there.

The volumes are noise_cases.planted_rows: planted x-runs of 3 and 5 whose y-runs are 1, 2 and 3 rows
long on every row that can start or end a y-chunk, across those cuts, at y = 0 and y = sy - 1 and on
the rows y = 0, 7 mod 8, and in 3-D pairs of slices z - 1, z that share a label at one voxel: across
every band's first and last slice, ragged last bands, nz < 8, and bands that cross a volume boundary
in stacks.  Each volume is transformed twice, so that the second transform takes the label-noise plan
with run-start planes, and compared with the oracle bit for bit.

What a wrong build does here:
  * applies the one-row rule at a chunk's last row without its trailing row: the two-row y-runs planted
    on rows yb, yb + 1 keep f = 4 or 9 in the oracle and drop to min(f, w_y^2) at row yb -- every case;
  * applies it to the rows at either end of a y-run: a run that touches y = 0 or y = sy - 1 without
    black_border has no border term next to that row, and f = 4 drops to w_y^2 = 1 where the oracle
    keeps 4;
  * uses w_z^2 (tz) in place of w_y^2: in 2-D tz is 0 and every such voxel drops to 0; in 3-D with
    w_z < w_y the blocks whose z-runs are three long drop from 4 to w_z^2 in their middle;
  * compares a band's first slice with its own row instead of the halo: the z plane says no run starts
    there, so the Z pass joins slice z0 to slice z0 - 1 where the labels differ -- every 3-D case with
    more than one band and the stacks;
  * takes a volume start where there is none (a slice's vz from its band's first slice): the planted
    pairs inside a band that starts a volume are split and keep 4 where the oracle has 2 -- every 3-D
    case and the stacks.  A build that ignores vz = 0 inside a band changes no result: the Z pass starts
    a run at every line's first row whatever its bit says.
"""
import numpy as np
import pytest

from noise_cases import FRESH, WIDE, assert_planes_plan, integral, planted_rows as planted, twice

pytestmark = pytest.mark.gpu

# (sz, sy, sx): nz < 8; ragged last bands (19 = 2 * 8 + 3, 9 = 8 + 1, 10); sy from 1 to 3 chunks, their
# cuts planted; rows of one, two and four 128-voxel blocks
SHAPES_3D = [(5, 201, 36), (19, 140, 132), (9, 134, 512), (7, 21, 36), (10, 45, 132), (5, 23, 512)]
# anisotropy in array order (z, y, x), w_x = 1: (w_z, w_y, w_x)
ANISO_3D = [(1.0, 1.0, 1.0),           # w_z = w_y
            (1.0, 2.0, 1.0),           # w_z < w_y
            (3.0, 2.0, 1.0),           # w_z > w_y
            (0.5, 0.7, 1.0),           # non-integer w_y (no settled-tile skip), w_z < w_y
            (1.0, 0.7, 1.0)]           # non-integer w_y, w_z > w_y


@pytest.mark.parametrize("shape", SHAPES_3D, ids=["x".join(map(str, s)) for s in SHAPES_3D])
@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_3d_chunks_and_bands(edt, oracle, shape, dtype):
  lab = planted(shape, dtype, sum(shape))
  for border in (False, True):
    for w in ANISO_3D:
      got = twice(edt.edtsq, lab, anisotropy=w, black_border=border)
      assert_planes_plan(edt, 1 if integral(w) else 0)
      want = oracle.edtsq(lab, anisotropy=w, black_border=border)
      assert np.array_equal(got, want), (w, border, int((got != want).sum()))
    for w in ((1.0, 2.0, 1.0), (0.5, 0.7, 1.0)):                 # sqrt in the Z pass's store
      got = twice(edt.edt, lab, anisotropy=w, black_border=border)
      assert_planes_plan(edt, 0)
      assert np.array_equal(got, oracle.edt(lab, anisotropy=w, black_border=border)), (w, border)


@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_3d_stack_bands_across_volumes(edt, oracle, dtype):
  """Volumes of 6 slices: bands of 8 slices start and end inside volumes."""
  stack_across_volumes(edt, oracle, dtype, (6, 140, 68), 5)


@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_stack_one_row_runs(edt, oracle, dtype):
  stack_across_volumes(edt, oracle, dtype, (6, 29, 132), 3)


def stack_across_volumes(edt, oracle, dtype, shape, seed, count=3):
  vols = [planted(shape, dtype, 10 * b + seed) for b in range(count)]
  stack = np.ascontiguousarray(np.stack(vols, axis=0))
  # each volume holds its own pairs; one more across every volume boundary, in two volumes and so
  # never one z-run
  flat = stack.reshape((-1,) + shape[1:])
  rng = np.random.default_rng(11)
  for z in range(shape[0], flat.shape[0], shape[0]):
    y, x0 = int(rng.integers(0, shape[1] - 1)), int(rng.integers(0, shape[2] - 3))
    flat[z - 1, y:y + 2, x0:x0 + 3] = FRESH - z
    flat[z, y, x0 + 1] = FRESH - z
  vols = list(stack)
  for border in (False, True):
    for w in ANISO_3D:
      got = twice(edt.edtsq, stack, anisotropy=w, black_border=border, stacked=True)
      assert_planes_plan(edt, 1 if integral(w) else 0)
      for b, v in enumerate(vols):
        want = oracle.edtsq(v, anisotropy=w, black_border=border)
        assert np.array_equal(got[b], want), (w, border, b, int((got[b] != want).sum()))


SHAPES_2D = [(201, 36), (140, 132), (134, 512), (21, 36), (67, 132), (45, 512)]


@pytest.mark.parametrize("shape", SHAPES_2D, ids=["x".join(map(str, s)) for s in SHAPES_2D])
@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_2d_chunks(edt, oracle, shape, dtype):
  lab = planted(shape, dtype, sum(shape) + 1)
  for border in (False, True):
    for w in ((1.0, 1.0), (2.0, 1.0), (0.7, 1.0)):
      got = twice(edt.edtsq, lab, anisotropy=w, black_border=border)
      assert_planes_plan(edt, 1 if integral(w) else 0)
      want = oracle.edtsq(lab, anisotropy=w, black_border=border)
      assert np.array_equal(got, want), (w, border, int((got != want).sum()))
    got = twice(edt.edt, lab, anisotropy=(2.0, 1.0), black_border=border)
    assert_planes_plan(edt, 0)
    assert np.array_equal(got, oracle.edt(lab, anisotropy=(2.0, 1.0), black_border=border)), border


@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_2d_stack_chunks(edt, oracle, dtype):
  """Eleven images: more sequences than one CTA's warps, some CTAs with idle warps."""
  shape, count = (150, 68), 11
  vols = [planted(shape, dtype, 10 * b + 7) for b in range(count)]
  stack = np.ascontiguousarray(np.stack(vols, axis=0))
  for border in (False, True):
    for w in ((1.0, 1.0), (0.7, 1.0)):
      got = twice(edt.edtsq, stack, anisotropy=w, black_border=border, stacked=True)
      assert_planes_plan(edt, 1 if integral(w) else 0)
      for b, v in enumerate(vols):
        want = oracle.edtsq(v, anisotropy=w, black_border=border)
        assert np.array_equal(got[b], want), (w, border, b, int((got[b] != want).sum()))


def test_rows_of_one_line(edt, oracle):
  """sy = 1: the Y pass's lines have one row, and no border term without black_border."""
  lab = planted((5, 1, 132), np.uint32, 9)
  for border in (False, True):
    got = twice(edt.edtsq, lab, anisotropy=(1.0, 2.0, 1.0), black_border=border)
    assert np.array_equal(got, oracle.edtsq(lab, anisotropy=(1.0, 2.0, 1.0), black_border=border)), border
