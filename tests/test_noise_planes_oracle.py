"""CPU tests of the restatement of the label-noise X pass's planes (tests/noise_planes_cases.py) against
identities that need no GPU: later passes that find their runs in the restated run-start planes equal
the oracle's, which finds them in the labels; the oracle's later passes leave every segment the
restated settled planes mark as it is; and hand-built cases whose bits are known by hand.
"""
import numpy as np
import pytest

import noise_planes_cases as npc

WIDE = (np.uint32, np.int32, np.uint64, np.int64)


def runs_along(rng, shape, axis, dtype):
  """Noise along x, runs of 1 to 4 equal labels along `axis` (1: y, 0: z of the slice stack)."""
  lab = npc.noise(shape, dtype, rng)
  n = shape[axis]
  for _ in range(n):
    at = int(rng.integers(1, n)) if n > 1 else 0
    if at:
      src = [slice(None)] * 3
      dst = [slice(None)] * 3
      src[axis], dst[axis] = at - 1, at
      keep = rng.random(shape[:axis] + shape[axis + 1:]) < 0.5
      lab[tuple(dst)] = np.where(keep, lab[tuple(src)], lab[tuple(dst)])
  return lab


CASES = [((2, 5, 9, 36), 3), ((1, 3, 7, 132), 3), ((3, 3, 4, 64), 3), ((4, 11, 508), 2), ((1, 1, 40), 2),
         ((2, 1, 1, 8), 3)]


@pytest.mark.parametrize("shape,ndim", CASES, ids=["x".join(map(str, c[0])) for c in CASES])
@pytest.mark.parametrize("border", (0, 1))
def test_runs_from_the_planes_give_the_oracle_later_passes(oracle, shape, ndim, border):
  rng = np.random.default_rng(sum(shape) + border)
  lab = runs_along(rng, shape, 1, np.uint32) if len(shape) == 3 else runs_along(
    rng, (shape[0] * shape[1],) + shape[2:], 1, np.uint32).reshape(shape)
  w = (1.0, 2.0, 3.0)
  x = npc.restate(oracle, lab, ndim, w, border)
  vol, depth = npc.slices(lab, ndim)
  n, sy, sx = vol.shape
  want = oracle.pass_later(vol, x["f"].copy(), 1, w[1], border, border)
  got = oracle.pass_later(npc.runs_from_plane(x["y"], n, sy, sx), x["f"].copy(), 1, w[1], border, border)
  assert np.array_equal(got, want)
  if ndim == 3:
    bits = np.unpackbits(x["z"].view(np.uint8), axis=1, bitorder="little")[:, :sx].astype(bool).reshape(n, sy, sx)
    for v in range(0, n, depth):
      part = slice(v, v + depth)
      ids = np.cumsum(bits[part], axis=0).astype(np.uint32) + 1
      want = oracle.pass_later(vol[part], x["f"][part].copy(), 2, w[2], border, border)
      got = oracle.pass_later(ids, x["f"][part].copy(), 2, w[2], border, border)
      assert np.array_equal(got, want), v


@pytest.mark.parametrize("shape,ndim", CASES, ids=["x".join(map(str, c[0])) for c in CASES])
@pytest.mark.parametrize("w", [(1.0, 1.0, 1.0), (1.0, 2.0, 0.5), (1.33355, 1.33355, 2.5), (2.0, 1.0, 1.0)])
def test_settled_segments_are_left_alone(oracle, shape, ndim, w):
  rng = np.random.default_rng(len(shape) * 100 + sum(shape))
  for kind in ("noise", "all", "none", "some"):
    for border in (0, 1):
      lab = npc.noise(shape, np.uint32, rng) if kind == "noise" else npc.settled_pattern(shape, np.uint32, rng, kind)
      x = npc.restate(oracle, lab, ndim, w, border)
      vol, depth = npc.slices(lab, ndim)
      n, sy, sx = vol.shape
      after_y = oracle.pass_later(vol, x["f"].copy(), 1, w[1], border, border)
      checks = [("settled_y", after_y)]
      if ndim == 3:
        after_z = x["f"].copy()
        for v in range(0, n, depth):
          after_z[v:v + depth] = oracle.pass_later(vol[v:v + depth], x["f"][v:v + depth].copy(), 2, w[2], border,
                                                   border)
        checks.append(("settled_z", after_z))
      for name, after in checks:
        words = x[name].reshape(n, sy)
        for s in range(npc.wpr(sx)):
          on = (words >> np.uint32(s)) & 1 == 1
          seg = slice(s * npc.SEG, (s + 1) * npc.SEG)
          assert np.array_equal(after[:, :, seg][on], x["f"][:, :, seg][on]), (kind, border, name, s)
        assert np.all(x[name] & npc.PAD_BITS == npc.PAD_BITS), name


def test_single_row_volume():
  """sy = 1: every voxel starts a y-run, and no line of one row takes min(f, ty)."""
  class Oracle:                            # an X pass whose answer is known: every neighbour differs
    @staticmethod
    def pass_first(vol, wx, border):
      return np.full(vol.shape, np.float32(wx) * np.float32(wx), np.float32)
  row = np.arange(1, 9, dtype=np.uint32)
  lab = np.stack([row, row]).reshape(1, 2, 1, 8)
  lab[0, 1, 0, 3] = 99
  x = npc.restate(Oracle, lab, 3, (1.0, 2.0, 0.5), 0)
  assert x["y"].tolist() == [[0xff], [0xff]]
  assert x["z"].tolist() == [[0xff], [0x8]]
  assert x["settled_y"].tolist() == [0xffffffff, 0xffffffff]        # f = 1 <= 4
  assert x["settled_z"].tolist() == [0xfffffffe, 0xfffffffe]        # f = 1 > 0.25
  assert np.all(x["f"] == 1.0)


@pytest.mark.parametrize("sx,last,settled", [(36, 0xf, 0xfffffffc), (132, 0xf, 0xffffffe0), (508, 0x0fffffff, 0xffff0000)])
def test_partial_last_word(oracle, sx, last, settled):
  """Rows 0 and 1 one y-run, row 2 another: padding bits 0, every real segment of rows 0 and 1
  unsettled (f = 1 > ty = 0.25), row 2 settled by its one-row run."""
  lab = np.arange(1, 3 * sx + 1, dtype=np.uint64).reshape(1, 3, sx)
  lab[0, 1] = lab[0, 0]
  x = npc.restate(oracle, lab, 2, (1.0, 0.5), 0)
  full = npc.wpr(sx) - 1
  assert x["y"][0].tolist() == [0xffffffff] * full + [last]
  assert x["y"][1].tolist() == [0] * (full + 1)
  assert x["y"][2].tolist() == [0xffffffff] * full + [last]
  assert x["settled_y"].tolist() == [settled, settled, 0xffffffff]
  assert np.all(x["f"][0, :2] == 1.0) and np.all(x["f"][0, 2] == 0.25)
  assert "z" not in x


def test_stack_depth_not_dividing_the_band():
  """Three volumes of three identical slices: the z bits are set on slices 0, 3 and 6 only."""
  class Oracle:
    @staticmethod
    def pass_first(vol, wx, border):
      return np.ones(vol.shape, np.float32)
  lab = np.broadcast_to(np.arange(1, 4 * 40 + 1, dtype=np.int32).reshape(4, 40), (3, 3, 4, 40)).copy()
  x = npc.restate(Oracle, lab, 3, (1.0, 1.0, 1.0), 0)
  z = x["z"].reshape(9, 4, 2)
  for s in range(9):
    want = [0xffffffff, 0xff] if s % 3 == 0 else [0, 0]
    assert np.all(z[s] == want), s
  assert len(npc.slices(lab, 3)[0]) == 9 and npc.slices(lab, 3)[1] == 3


def test_refresh_rule():
  """refresh_settled's rule on a hand-built slice: a tile that ran with 1 to 32 clear rows sets
  exactly the rows now <= tz; one with 33 clear rows, or one that did not run, sets none."""
  sy, sx = 40, 64
  f = np.zeros((3, sy, sx), np.float32)
  f[:, 5, 3] = 2.0                                  # row 5 of segment 0 stays above tz = 1
  settled_y = np.full((3, sy), 0xffffffff, np.uint32)
  settled_y[0, 7] &= ~np.uint32(1)                  # slice 0: tile 0 runs, tile 1 does not
  settled_y[1, 0] &= ~np.uint32(3)                  # slice 1: both tiles run
  settled_z = np.full((3, sy), 0xffffffff, np.uint32)
  settled_z[0, :10] &= ~np.uint32(3)                # slice 0: 10 rows clear in both segments
  settled_z[1, :33] &= ~np.uint32(1)                # slice 1: 33 rows clear in segment 0, 1 in segment 1
  settled_z[1, 20] &= ~np.uint32(2)
  settled_z[2, 4] &= ~np.uint32(1)                  # slice 2: no tile runs
  got = npc.refresh(settled_z.reshape(-1), settled_y.reshape(-1), f, np.float32(1.0)).reshape(3, sy)
  want = settled_z.copy()
  want[0, :10] |= np.uint32(1)
  want[0, 5] &= ~np.uint32(1)
  want[1, 20] |= np.uint32(2)
  assert np.array_equal(got, want)


def test_buffer_layout():
  """[y plane | settled_y | z plane | settled_z], as take_run_planes allocates it."""
  assert npc.layout(36, 5, 10, 3) == [("y", 0, 20), ("settled_y", 20, 10), ("z", 30, 20), ("settled_z", 50, 10)]
  assert npc.layout(512, 5, 10, 2) == [("y", 0, 160), ("settled_y", 160, 10)]
  assert npc.buffer_words(4, 1, 7, 3) == 28
