"""GPU tests (-m gpu) of the plane-writing X pass whose warps march along y (first_axis_planes_kernel): a
CTA owns a band of W = 8 slices and a y-chunk of rows, stages
one row of every slice of the band plus the halo row of the slice below it per step, and reads each
chunk's leading row ya - 1 and trailing row yb + 1 for their compares only.  In 2-D the warps take
independent (image, y-chunk) sequences.

The volumes are label noise with planted x-runs of 3 and 5 (f = 4 and 9 with w_x = 1) whose y-runs are
1, 2 and 3 rows long, on every row that can start or end a y-chunk (the launcher cuts a slice into at
most 3 sy / 200 chunks; every such cut is planted), across those cuts, and at y = 0 and y = sy - 1, on
every slice; and, in 3-D, pairs of slices z - 1, z that share a label at one voxel whose values differ
(f = 4 against 1), for every z: across every band's first and last slice, ragged last bands, nz < W,
and bands that cross a volume boundary in stacks.  Each volume is transformed twice, so that the second
transform takes the label-noise plan with run-start planes, and compared with the oracle bit for bit.

What a wrong build does here:
  * applies the one-row rule at a chunk's last row without its trailing row: the two-row y-runs planted
    on rows yb, yb + 1 keep f = 4 or 9 in the oracle and drop to min(f, w_y^2) at row yb -- every case;
  * compares a band's first slice with its own row instead of the halo: the z plane says no run starts
    there, so the Z pass joins slice z0 to slice z0 - 1 where the labels differ -- every 3-D case with
    more than one band (all but 5 x 201 x 36) and the stacks;
  * takes a volume start where there is none (a slice's vz from its band's first slice): the planted
    pairs inside a band that starts a volume are split and keep 4 where the oracle has 2 -- every 3-D
    case and the stacks.  A build that ignores vz = 0 inside a band changes no result: the Z pass starts
    a run at every line's first row whatever its bit says.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

WIDE = (np.uint32, np.uint64)
FRESH = 1 << 21                        # planted labels: above every noise label


def noise(shape, dtype, seed, background=0.02):
  rng = np.random.default_rng(seed)
  lab = rng.integers(1, 1 << 20, shape).astype(dtype)
  lab[rng.random(shape) < background] = 0
  return lab


# (x extent, y rows relative to the target row) of the planted blocks
KINDS = [(3, (0,)),                    # x-run of 3, y-run of 1: f = 4
         (5, (0,)),                    # x-run of 5, y-run of 1: f = 4 and 9
         (3, (0, 1)),                  # y-run of 2 starting at the target row
         (3, (-1, 0)),                 # y-run of 2 ending at the target row
         (3, (-1, 0, 1)),              # y-run of 3 around the target row: its middle keeps f = 4
         (5, (0, 1))]


def chunk_starts(sy):
  """Every row that starts a y-chunk for some chunk count the launcher may pick (1 .. 3 sy / 200)."""
  starts = set()
  for n in range(2, sy * 3 // 200 + 1):
    starts |= {k * sy // n for k in range(1, n)}
  return starts


def target_rows(sy):
  rows = {0, 1, sy - 2, sy - 1}
  for ya in chunk_starts(sy):
    rows |= {ya - 2, ya - 1, ya, ya + 1}
  return sorted(y for y in rows if 0 <= y < sy)


def planted(shape, dtype, seed):
  """Label noise (C order, x last) with blocks of the KINDS on every target row of every slice, one per
  66 voxels of the row (at least one), the kinds taking turns over rows, slices and blocks.  With three
  or more axes, also one pair per slice z >= 1: an x-run of 3 with a y-run of 2 on slice z - 1 (f = 4 in
  its middle) and the same label at that middle voxel alone on slice z (f = 1), so that the middle
  leaves the Z pass at 2 where z - 1 and z are one z-run and at 4 where they are not."""
  lab = noise(shape, dtype, seed)
  vol = lab.reshape((-1,) + lab.shape[-2:])
  nz, sy, sx = vol.shape
  fresh = iter(range(FRESH, FRESH + 10 ** 7))
  rows = target_rows(sy)
  blocks = max(1, sx // 66)
  span = sx // blocks
  for z in range(nz):
    for i, y in enumerate(rows):
      for j in range(blocks):
        xn, dys = KINDS[(i + z + j) % len(KINDS)]
        x0 = j * span + (7 * (i + 2 * z)) % max(1, span - xn)
        x0 = min(x0, sx - xn)
        ys = [y + d for d in dys if 0 <= y + d < sy]
        vol[z, ys, x0:x0 + xn] = next(fresh)
  if lab.ndim >= 3 and sy >= 2 and sx >= 3:
    for z in range(1, nz):
      y = (5 * z) % (sy - 1)
      x0 = sx - 3 - (z % max(1, sx - 3))
      label = next(fresh)
      vol[z - 1, y:y + 2, x0:x0 + 3] = label
      vol[z, y, x0 + 1] = label
  return lab


def twice(fn, labels, **kw):
  # leaves the run statistic of this volume behind (a black border makes narrow rows noise too)
  fn(labels, **dict(kw, black_border=True))
  return fn(labels, **kw)


def assert_planes_plan(edt, settled):
  info = edt.last_later_launch()
  assert info["kernel"] == "tile" and info["ctas"] == 2 and info["tx"] == 32 and info["tma"] == 1, info
  if settled is not None:
    assert info["settled"] == settled, info


def integral(w):
  return all(float(v).is_integer() for v in w)


# (sz, sy, sx): nz < W; ragged last bands (19 = 2 * 8 + 3, 9 = 8 + 1); sy from 2 to 3
# chunks, their cuts planted; rows of one, two and four 128-voxel blocks
SHAPES_3D = [(5, 201, 36), (19, 140, 132), (9, 134, 512)]
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
    got = twice(edt.edt, lab, anisotropy=(1.0, 2.0, 1.0), black_border=border)
    assert_planes_plan(edt, 0)
    assert np.array_equal(got, oracle.edt(lab, anisotropy=(1.0, 2.0, 1.0), black_border=border)), border


@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_3d_stack_bands_across_volumes(edt, oracle, dtype):
  """Volumes of 6 slices: bands of 8 slices start and end inside volumes."""
  shape, count = (6, 140, 68), 3
  vols = [planted(shape, dtype, 10 * b + 5) for b in range(count)]
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


SHAPES_2D = [(201, 36), (140, 132), (134, 512)]


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
