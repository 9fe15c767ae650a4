"""CPU tests of the skeleton's restatement (skeleton_cases.py): the simple-voxel predicate against an
independent invariants check, the guarantees on multi-label 2-D and 3-D volumes (per-label topology, thinness,
skeleton within the labels, even shifts), the worked examples, and each planted defect caught."""
import itertools

import numpy as np
import pytest

import skeleton_cases as skc


def _by_invariants(block):
  """Removing the centre of the 3x3(x3) block (padded by background) keeps the label's components, its
  complement's components and its Euler characteristic."""
  centre = (1,) * block.ndim
  without = block.copy()
  without[centre] = False
  return skc.invariants(block) == skc.invariants(without)


def _code(block):
  nd = block.ndim
  b = block if nd == 3 else np.stack([np.zeros_like(block), block, np.zeros_like(block)])
  return sum(1 << j for j, (dz, dy, dx) in enumerate(skc.OFFSETS) if b[1 + dz, 1 + dy, 1 + dx])


def test_the_2d_predicate_on_every_neighbourhood():
  for bits in range(256):
    block = np.zeros((3, 3), bool)
    block[1, 1] = True
    for n, (y, x) in enumerate(p for p in itertools.product(range(3), repeat=2) if p != (1, 1)):
      block[y, x] = bool(bits >> n & 1)
    assert skc.simple(_code(block), 2) == _by_invariants(block), block.astype(int)


def test_the_3d_predicate_on_random_neighbourhoods():
  rng = np.random.default_rng(3)
  seen = {True: 0, False: 0}
  for n in range(3000):
    block = rng.random((3, 3, 3)) < rng.uniform(0.2, 0.8)
    block[1, 1, 1] = True
    want = _by_invariants(block)
    assert skc.simple(_code(block), 3) == want, block.astype(int)
    seen[want] += 1
  assert min(seen.values()) > 300


def _volumes():
  rng = np.random.default_rng(17)
  for kind in skc.KINDS:
    yield skc.seeded(rng, kind, (9, 12, 14), np.uint16), (1.0, 1.0, 1.0)
    yield skc.seeded(rng, kind, (10, 13, 11), np.uint8), (3.0, 1.0, 1.0)
    yield skc.seeded(rng, kind, (24, 31), np.int32), (1.0, 1.0)
    yield skc.seeded(rng, kind, (21, 26), np.uint8), (0.7, 1.9)
  yield skc.balls(rng, (8, 20, 20), 4, 6.0, np.uint8), (4.0, 4.0, 40.0)
  yield skc.voronoi(rng, (7, 18, 22), 5, np.uint16), (4.0, 4.0, 40.0)


@pytest.mark.parametrize("border", [False, True])
def test_the_guarantees_on_multi_label_volumes(border):
  for labels, w in _volumes():
    skel = skc.restate(labels, w, border)
    assert not (skel & (labels == 0)).any()
    assert skc.topology_kept(labels, skel) == [], (labels.shape, w)
    assert skc.not_thin(labels, skel) == 0, (labels.shape, w)


def test_an_even_shift_shifts_the_skeleton():
  rng = np.random.default_rng(5)
  for nd, w in ((2, (1.0, 2.0)), (3, (1.0, 1.0, 3.0))):
    labels = skc.seeded(rng, "balls", (9, 11, 12)[:nd] if nd == 3 else (17, 19), np.uint8)
    pad = [(2, 0)] + [(0, 4)] * (nd - 1)
    want = np.pad(skc.restate(np.pad(labels, 1), w, True), pad)
    assert np.array_equal(skc.restate(np.pad(np.pad(labels, 1), pad), w, True), want)


def test_the_worked_examples():
  line = np.zeros((5, 7, 9), np.uint8)
  line[2, 3, 1:8] = 1
  assert np.array_equal(skc.restate(line), line != 0)
  dot = np.zeros((3, 3, 3), np.uint8)
  dot[1, 1, 1] = 7
  assert np.array_equal(skc.restate(dot), dot != 0)
  cube = np.zeros((5, 5, 5), np.uint8)
  cube[1:4, 1:4, 1:4] = 1
  assert np.argwhere(skc.restate(cube)).tolist() == [[2, 2, 2]]
  zz, yy, xx = np.indices((13, 13, 13))
  r2 = (zz - 6) ** 2 + (yy - 6) ** 2 + (xx - 6) ** 2
  shell = (r2 <= 25) & (r2 >= 9)
  skel = skc.restate(shell)
  assert skc.invariants(skel) == (1, 2, 2) and skel.sum() < shell.sum()
  box = np.zeros((6, 8, 14), np.uint8)
  box[1:5, 1:7, 1:13] = 1
  assert np.argwhere(skc.restate(box)).tolist() == [[3, 4, x] for x in range(4, 11)]
  yy, xx = np.indices((15, 15))
  assert np.argwhere(skc.restate((yy - 7) ** 2 + (xx - 7) ** 2 <= 36)).tolist() == [[7, 7]]


def test_one_label_volumes_thin_in_the_final_round():
  stats = {}
  full = np.ones((5, 6, 7), np.uint8)
  r = np.full(full.shape, np.inf, np.float32)
  skel = skc.thin(full, r, 1.0, stats=stats)
  assert stats["rounds"] == 1 and skc.invariants(skel) == skc.invariants(full) and skc.not_thin(full, skel) == 0


# ---- the planted defects ------------------------------------------------------------------------------

@pytest.mark.parametrize("defect", ["parallel", "background26"])
def test_defects_that_break_the_invariants(defect):
  broken = 0
  for labels, w in _volumes():
    skel = skc.restate(labels, w, True, defect=defect)
    broken += len(skc.topology_kept(labels, skel))
  assert broken > 0


def test_no_endpoints_breaks_the_straight_line():
  line = np.zeros((5, 9), np.uint8)
  line[2, 1:8] = 1
  assert np.array_equal(skc.restate(line), line != 0)
  assert not np.array_equal(skc.restate(line, defect="no_endpoints"), line != 0)


def test_step_endpoints_breaks_the_cube():
  cube = np.zeros((5, 5, 5), np.uint8)
  cube[1:4, 1:4, 1:4] = 1
  assert skc.restate(cube, defect="step_endpoints").sum() == 9


def test_voxel_order_changes_a_pinned_anisotropic_case():
  box = np.zeros((8, 14, 14), np.uint8)
  box[1:7, 1:13, 1:13] = 1
  w = (4.0, 4.0, 40.0)
  assert not np.array_equal(skc.restate(box, w, True), skc.restate(box, w, True, defect="voxel_order"))
