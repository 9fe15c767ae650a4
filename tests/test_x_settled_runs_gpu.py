"""GPU tests (-m gpu) of the y-runs of one row that the plane-writing X pass settles: on predicted label
noise the X pass compares every row with rows y - 1 and y + 1 and stores min(f, w_y^2) where the
voxel's y-run is one row long, which is exactly what the Y pass would leave there.  The volumes are
label noise with planted x-runs of 3 and 5 (f = 4 and 9 with w_x = 1) whose y-runs are 1, 2 and 3 rows
long, on the first and last rows of the X pass's 8-row bands (y = 0, 7 mod 8) and at y = 0 and
y = sy - 1, and x-y-z blocks whose z-runs are 3 long; each is transformed twice so that the second
transform takes the label-noise plan, and compared with the oracle bit for bit.

What a wrong build does here:
  * applied to the rows at either end of a y-run (every row of a two-row run): a run that touches
    y = 0 or y = sy - 1 without black_border has no border term next to that row, and f = 4 drops to
    w_y^2 = 1 (with w_y = 1) where the oracle keeps 4;
  * applied to a band's last row (y = 7 mod 8) without seeing row y + 1: the middle row of the
    three-row runs planted on rows 6, 7, 8 keeps f = 4 in the oracle and drops to 1;
  * with w_z^2 (tz) in place of w_y^2: in 2-D tz is 0 and every such voxel drops to 0; in 3-D with
    w_z < w_y the blocks whose z-runs are three long drop from 4 to w_z^2 in their middle.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

WIDE = (np.uint32, np.uint64)
FRESH = 1 << 21                        # planted labels: above every noise label
W = 8                                  # rows per band of the X pass


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
         (5, (-1, 0, 1))]


def target_rows(sy):
  """The band edges (y = 0 and 7 mod 8, their neighbours) and the line's first and last rows."""
  rows = {0, 1, sy - 2, sy - 1}
  for y0 in range(0, sy, W):
    rows |= {y0, y0 + W - 1}
  return sorted(y for y in rows if 0 <= y < sy)


def planted(shape, dtype, seed):
  """Label noise (C order, x last) with blocks of the KINDS planted on every target row of every slice:
  one per 66 voxels of the row (at least one), the kinds taking turns over rows, slices and blocks, at
  x offsets that differ between neighbouring target rows.  Sparse enough that the volume is still label
  noise along x (at least 9 runs per 10 voxels).  In 3-D, also x-runs of 3 on one row through three
  slices."""
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
  if nz >= 3:                          # x-runs of 3 with z-runs of 3, y-runs of 1, at the row ends
    for z in range(1, nz - 1, 3):
      for y, x0 in ((sy // 2, sx - 3), (W - 1, 0)):
        if y < sy:
          vol[z - 1:z + 2, y, x0:x0 + 3] = next(fresh)
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


# (sz, sy, sx): sy ragged (bands cut short) and long enough for several bands
SHAPES_3D = [(7, 21, 36), (10, 45, 132), (5, 23, 512)]
# anisotropy in array order (z, y, x), w_x = 1: (w_z, w_y, w_x)
ANISO_3D = [(1.0, 1.0, 1.0),           # w_z = w_y
            (1.0, 2.0, 1.0),           # w_z < w_y
            (3.0, 2.0, 1.0),           # w_z > w_y
            (0.5, 0.7, 1.0),           # non-integer w_y (no settled-tile skip), w_z < w_y
            (1.0, 0.7, 1.0)]           # non-integer w_y, w_z > w_y


def integral(w):
  return all(float(v).is_integer() for v in w)


@pytest.mark.parametrize("shape", SHAPES_3D, ids=["x".join(map(str, s)) for s in SHAPES_3D])
@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_3d_one_row_runs_bit_exact(edt, oracle, shape, dtype):
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


SHAPES_2D = [(21, 36), (67, 132), (45, 512)]


@pytest.mark.parametrize("shape", SHAPES_2D, ids=["x".join(map(str, s)) for s in SHAPES_2D])
@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_2d_one_row_runs_bit_exact(edt, oracle, shape, dtype):
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
def test_stack_one_row_runs(edt, oracle, dtype):
  shape = (6, 29, 132)
  vols = [planted(shape, dtype, 10 * b + 3) for b in range(3)]
  stack = np.ascontiguousarray(np.stack(vols, axis=0))
  for border in (False, True):
    for w in ((1.0, 2.0, 1.0), (1.0, 0.7, 1.0)):
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
