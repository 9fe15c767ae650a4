"""Shared cases of the label-noise tests: on predicted label noise with labels of 4 or 8 bytes the X
pass writes run-start and settled planes (first_axis_planes_kernel), and the later passes read them
instead of the labels and skip the tiles the X pass settled.  The prediction comes from the previous
transform on the device, so a case transforms its volume twice and checks the second result.
"""
import numpy as np

WIDE = (np.uint32, np.uint64)
FRESH = 1 << 21                        # planted labels: above every noise label
BAND = 8                               # slices per band of the plane-writing X pass (kPlaneWarps)

# (x extent, y rows relative to the target row) of planted blocks: x-runs of 3 and 5 (f = 4 and 9 with
# w_x = 1) whose y-runs are 1, 2 and 3 rows long
KINDS = [(3, (0,)),                    # x-run of 3, y-run of 1: f = 4
         (5, (0,)),                    # x-run of 5, y-run of 1: f = 4 and 9
         (3, (0, 1)),                  # y-run of 2 starting at the target row
         (3, (-1, 0)),                 # y-run of 2 ending at the target row
         (3, (-1, 0, 1)),              # y-run of 3 around the target row: its middle keeps f = 4
         (5, (-1, 0, 1)),
         (5, (0, 1))]


def noise(shape, dtype, seed, background=0.02):
  """Label noise: almost every voxel differs from its neighbours, a few are background."""
  rng = np.random.default_rng(seed)
  lab = rng.integers(1, 1 << 20, shape).astype(dtype)
  lab[rng.random(shape) < background] = 0
  return lab


def twice(fn, labels, **kw):
  """fn(labels, **kw) right after fn on the same labels, which leaves the run statistic of this volume
  behind.  Under that first call's black border the row's first voxel counts as a run start, so that
  narrow rows (sx = 4) are label noise too."""
  fn(labels, **dict(kw, black_border=True))
  return fn(labels, **kw)


def integral(w):
  return all(float(v).is_integer() for v in w)


def chunk_starts(sy):
  """Every row that starts a y-chunk of the plane-writing X pass for some chunk count it may pick:
  launch_first_vec cuts a slice of sy rows into n <= 3 sy / 200 chunks, chunk k starting at k sy / n."""
  starts = set()
  for n in range(2, sy * 3 // 200 + 1):
    starts |= {k * sy // n for k in range(1, n)}
  return starts


def target_rows(sy):
  """The rows where a y-run meets an edge of the X pass's work: the line's first and last rows, every
  y-chunk cut and the rows around it; and every row y = 0, 7 mod 8."""
  rows = {0, 1, sy - 2, sy - 1}
  for ya in chunk_starts(sy):
    rows |= {ya - 2, ya - 1, ya, ya + 1}
  for y0 in range(0, sy, 8):
    rows |= {y0, y0 + 7}
  return sorted(y for y in rows if 0 <= y < sy)


def planted_rows(shape, dtype, seed):
  """Label noise (C order, x last) with blocks of the KINDS on every target row of every slice, one per
  66 voxels of the row (at least one), the kinds taking turns over rows, slices and blocks.  Sparse
  enough that the volume is still label noise along x.  With three or more axes, also one pair per
  slice z >= 1: an x-run of 3 with a y-run of 2 on slice z - 1 (f = 4 in its middle) and the same label
  at that middle voxel alone on slice z (f = 1), so that the middle leaves the Z pass at 2 where z - 1
  and z are one z-run and at 4 where they are not; and x-runs of 3 on one row through three slices."""
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
  if lab.ndim >= 3:                    # x-runs of 3 with z-runs of 3, y-runs of 1, at the row ends
    for z in range(1, nz - 1, 3):
      for y, x0 in ((sy // 2, sx - 3), (7, 0)):
        if y < sy:
          vol[z - 1:z + 2, y, x0:x0 + 3] = next(fresh)
  return lab


def assert_planes_plan(edt, settled):
  """The last later pass took the label-noise tile kernel, and skipped settled tiles or not."""
  info = edt.last_later_launch()
  assert info["kernel"] == "tile" and info["ctas"] == 2 and info["tx"] == 32 and info["tma"] == 1, info
  assert info["settled"] == settled, info
