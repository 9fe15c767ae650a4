"""GPU tests (-m gpu) of the grouped settled check: with `settled` armed, each CTA of the label-noise
later-pass kernel owns a group of consecutive tiles, reads the group's settled words once and runs
only the tiles that are not settled.  The volumes are label noise with unsettled voxels planted
group by group: at a group's first and last tile, in every tile of a group, in one tile, and in none;
with row lengths of 32, 48, 96 and 512 (Z tiles of 32 lines reach into the next row when the row
length is not a multiple of 32), partial last groups and stacks whose groups cross from one volume
into the next.  Each volume is transformed twice, so that the second transform takes the label-noise
plan, and compared with the oracle bit for bit.  The same cases run again with the group size forced
through EDTB200_SETTLED_GROUP, read once per process: to 1, to 7 (which divides no tile count here)
and to 16.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from noise_cases import FRESH, WIDE, twice

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
# (sz, sy, sx) in array order; Y tiles sz * ceil(sx / 32), Z tiles ceil(sx * sy / 32)
SHAPES = [(20, 33, 32), (12, 40, 48), (10, 37, 96), (6, 24, 512)]
STACK = (3, 5, 21, 48)                 # 3 volumes: 32 Z tiles each, the last one half full
# array order (w_z, w_y, w_x): with w_z = 2 the Z pass takes voxels at f <= 4 as settled, so the Y
# pass's refresh settles the Z tiles of x-runs of five (f = 9 after X, 2 after Y)
ANISO = [(1.0, 1.0, 1.0), (2.0, 1.0, 1.0)]


def pattern(group_index, group, rng):
  """The tiles (offsets in the group) to leave unsettled: none, the first and the last, all, one."""
  kind = group_index % 4
  if kind == 0:
    return []
  if kind == 1:
    return sorted({0, group - 1})
  if kind == 2:
    return list(range(group))
  return [int(rng.integers(0, group))]


def planted(shape, dtype, seed, group):
  """Label noise (C order, x last) of one volume, or of a stack (leading axis), with planted voxels.
  Z tiles: a 3x3x3 cube around one line of the tile (its centre line ends the Y pass at f = 4).  Y
  tiles (z, x-segment): an x-run of three inside the segment (f = 4 after X), and in every fourth
  such tile an x-run of five, whose middle voxel only the Y pass settles for the Z pass."""
  rng = np.random.default_rng(seed)
  lab = rng.integers(1, 1 << 20, shape).astype(dtype)
  vols = lab.reshape((-1,) + shape[-3:])
  nv = vols.shape[0]
  sz, sy, sx = shape[-3:]
  fresh = iter(range(FRESH, FRESH + 10 ** 7))
  # Z pass: outer = volume, 32 lines (y * sx + x) per tile
  tpo = (sx * sy + 31) // 32
  for g0 in range(0, nv * tpo, group):
    for k in pattern(g0 // group, group, rng):
      t = g0 + k
      if t >= nv * tpo:
        continue
      v, j0 = divmod(t, tpo)
      for j in range(j0 * 32 + 5, min(j0 * 32 + 32, sx * sy)):
        y, x = divmod(j, sx)
        if 1 <= y < sy - 1 and 1 <= x < sx - 1:
          z = int(rng.integers(0, sz - 2))
          vols[v, z:z + 3, y - 1:y + 2, x - 1:x + 2] = next(fresh)
          break
  # Y pass: outer = z of every volume, one tile per 32-voxel x-segment
  tpo = (sx + 31) // 32
  for g0 in range(0, nv * sz * tpo, group):
    for k in pattern(g0 // group + 1, group, rng):
      t = g0 + k
      if t >= nv * sz * tpo:
        continue
      vz, seg = divmod(t, tpo)
      v, z = divmod(vz, sz)
      y = int(rng.integers(0, sy))
      width = 5 if t % 4 == 0 else 3
      x0 = seg * 32 + 10
      if x0 + width <= sx:
        vols[v, z, y, x0:x0 + width] = next(fresh)
  return lab


def run_cases(edt, oracle, group):
  """Every case, with unsettled tiles planted for groups of `group` tiles."""
  for dtype in WIDE:
    for shape in SHAPES:
      lab = planted(shape, dtype, sum(shape) + group, group)
      for w in ANISO:
        got = twice(edt.edtsq, lab, anisotropy=w)
        assert edt.last_later_launch()["settled"] == 1, (shape, w, edt.last_later_launch())
        want = oracle.edtsq(lab, anisotropy=w)
        assert np.array_equal(got, want), (dtype.__name__, shape, w, group, int((got != want).sum()))
    stack = planted(STACK, dtype, 7 + group, group)
    for w in ANISO:
      got = twice(edt.edtsq, stack, anisotropy=w, stacked=True)
      assert edt.last_later_launch()["settled"] == 1
      for b in range(STACK[0]):
        want = oracle.edtsq(np.ascontiguousarray(stack[b]), anisotropy=w)
        assert np.array_equal(got[b], want), (dtype.__name__, "stack", b, w, group)


def test_groups_bit_exact(edt, oracle):
  run_cases(edt, oracle, 16)


@pytest.mark.parametrize("group", [1, 7, 16])
def test_forced_group_bit_exact(group, tmp_path):
  script = ("import sys; sys.path[:0] = [%r, %r]; import edt_b200, test_settled_groups_gpu as t; "
            "from oracle import oracle; t.run_cases(edt_b200, oracle, %d)") % (ROOT, HERE, group)
  proc = subprocess.run([sys.executable, "-c", script], env=dict(os.environ, EDTB200_SETTLED_GROUP=str(group)),
                        cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
  assert proc.returncode == 0, proc.stderr[-3000:]
