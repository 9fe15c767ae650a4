"""CPU tests of the geodesic_distance restatement (geodesic_cases.py): closed-form answers on straight lines,
diagonals and L-shapes, +inf and -1 where no seed is reachable, and agreement with an independent heapq
Dijkstra over (D, S) pairs on random multi-label volumes, mazes and corridors through tile corners."""
import math

import numpy as np
import pytest

import geodesic_cases as gc


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("w", [(1.0, 1.0), (1.0, 0.5), (1.33355, 1.0), (4.0, 40.0)])
def test_straight_lines_are_steps_times_the_weight(order, w):
  lab = np.zeros((3, 12), np.uint8)
  lab[1, 1:11] = 1
  lab = np.asfortranarray(lab) if order == "F" else lab
  seeds = np.zeros(lab.shape, bool)
  seeds[1, 1] = True
  dist, S = gc.restate(lab, seeds, w, order)
  want = np.array([k * w[1] for k in range(10)])          # axis 1 is the line's axis
  # each step adds the float32 weight in double, in order: the sum of k equal doubles
  acc, exact = 0.0, []
  for k in range(10):
    exact.append(acc)
    acc += gc.weight(w[1])
  assert np.array_equal(dist[1, 1:11], np.float32(exact))
  assert np.allclose(dist[1, 1:11], want, rtol=1e-6)
  assert np.isinf(dist[0]).all() and np.isinf(dist[2]).all() and np.isinf(dist[1, [0, 11]]).all()
  planes = gc.index_planes(S, lab.shape, order)
  assert (planes[0][1, 1:11] == 1).all() and (planes[1][1, 1:11] == 1).all()
  assert (planes[:, 0] == -1).all()


@pytest.mark.parametrize("w", [(1.0, 1.0), (1.0, 2.0), (1.7, 0.3)])
def test_diagonals_are_steps_times_the_diagonal_length(w):
  n = 9
  lab = np.eye(n, dtype=np.uint8)
  seeds = np.zeros((n, n), bool)
  seeds[0, 0] = True
  dist, _ = gc.restate(lab, seeds, w)
  wx, wy = gc.weight(w[1]), gc.weight(w[0])
  step = math.sqrt(wx * wx + wy * wy)                    # x (the last axis) first
  acc = 0.0
  for k in range(n):
    assert dist[k, k] == np.float32(acc)
    acc += step
  assert np.isinf(dist[lab == 0]).all()


def test_the_l_shape_is_longer_than_the_straight_line():
  lab = np.zeros((5, 5), np.uint8)
  lab[0, :] = 1
  lab[:, 4] = 1
  seeds = np.zeros((5, 5), bool)
  seeds[0, 0] = True
  dist, S = gc.restate(lab, seeds)
  assert dist[4, 4] == np.float32(6 + np.sqrt(2)) and dist[4, 4] > np.sqrt(32)
  assert dist[0, 3] == 3 and dist[1, 4] == np.float32(3 + np.sqrt(2))
  assert (S[lab != 0] == 0).all() and (S[lab == 0] == -1).all()


def test_unreachable_voxels_are_inf_and_minus_one():
  lab = np.zeros((4, 10), np.uint16)
  lab[:, :4] = 1
  lab[:, 6:] = 1               # the same label, cut by background: a component with no seed
  lab[0, 5] = 2
  seeds = np.zeros(lab.shape, np.int32)
  seeds[1, 1] = 7
  seeds[3, 4] = 1              # on background: ignored
  dist, S = gc.restate(lab, seeds)
  assert np.isfinite(dist[:, :4]).all()
  assert np.isinf(dist[:, 4:]).all() and (S[:, 4:] == -1).all()
  planes = gc.index_planes(S, lab.shape)
  assert (planes[:, :, 4:] == -1).all() and (planes[0][:, :4] == 1).all() and (planes[1][:, :4] == 1).all()


def test_ties_go_to_the_least_x_fastest_index():
  lab = np.ones((1, 5), np.uint8)
  seeds = np.zeros((1, 5), bool)
  seeds[0, 0] = seeds[0, 4] = True
  _, S = gc.restate(lab, seeds)
  assert S.tolist() == [[0, 0, 0, 4, 4]]         # the middle voxel ties: the least index wins
  lab = np.ones((3, 3), np.uint8)
  seeds = np.zeros((3, 3), bool)
  seeds[0, 2] = seeds[2, 0] = True                # C order: x-fastest indices 2 and 6
  _, S = gc.restate(lab, seeds)
  assert S[1, 1] == 2
  _, S = gc.restate(np.asfortranarray(lab), np.asfortranarray(seeds), order="F")
  assert S[1, 1] == 2                             # F order: (0, 2) is x-fastest index 0 + 3 * 2 = 6; (2, 0) is 2


CASES = [((13, 17), (1.0, 1.33355)), ((6, 7, 9), (1.7, 1.0, 3.1)), ((6, 7, 5), (1.33355, 1.0, 2.0 ** -26)),
         ((5, 6, 7), (4.0, 4.0, 40.0)), ((70,), (0.7,)), ((9, 10, 11), (1.0, 1.0, 1.0))]


@pytest.mark.parametrize("order", ["C", "F"])
@pytest.mark.parametrize("shape,w", CASES)
def test_the_restatement_equals_a_heapq_dijkstra_over_pairs(shape, w, order):
  rng = np.random.default_rng(sum(shape))
  for _ in range(3):
    lab = gc.random_labels(rng, shape)
    seeds = gc.random_seeds(rng, shape, 0.03, np.uint8)
    if order == "F":
      lab, seeds = np.asfortranarray(lab), np.asfortranarray(seeds)
    dist, S = gc.restate(lab, seeds, w, order)
    D2, S2 = gc.dijkstra_pairs(lab, seeds, w, order)
    assert np.array_equal(dist, D2.astype(np.float32))
    assert np.array_equal(S, S2)


@pytest.mark.parametrize("nd,cross", [(1, "corner"), (2, "corner"), (3, "corner"), (3, "edge")])
def test_corridors_through_tile_corners_and_edges(nd, cross):
  lab = gc.corridor_through_corner(nd, cross=cross)
  seeds = np.zeros(lab.shape, bool)
  first = tuple(np.argwhere(lab)[np.argwhere(lab)[:, 0].argmin()])
  seeds[first] = True
  lab_c, seeds_c = np.ascontiguousarray(lab.T), np.ascontiguousarray(seeds.T)   # x last
  dist, S = gc.restate(lab_c, seeds_c)
  assert np.isfinite(dist[lab_c != 0]).all() and np.isinf(dist[lab_c == 0]).all()
  D2, S2 = gc.dijkstra_pairs(lab_c, seeds_c)
  assert np.array_equal(dist, D2.astype(np.float32)) and np.array_equal(S, S2)


def test_mazes_agree_with_the_pairs():
  for lab in (gc.spiral(20), gc.serpentine((12, 13, 2)).T.copy()):
    seeds = np.zeros(lab.shape, bool)
    seeds[(0,) * lab.ndim] = True
    dist, S = gc.restate(lab, seeds)
    D2, S2 = gc.dijkstra_pairs(lab, seeds)
    assert np.array_equal(dist, D2.astype(np.float32)) and np.array_equal(S, S2)
    assert np.isfinite(dist[lab != 0]).all()
    assert dist.max() > 2 * max(lab.shape)         # the path winds



@pytest.mark.parametrize("name,lab,seeds", gc.seeded_at_tile_borders(), ids=[c[0] for c in gc.seeded_at_tile_borders()])
def test_seeds_on_tile_borders_reach_both_sides(name, lab, seeds):
  dist, S = gc.restate(lab, seeds)
  D2, S2 = gc.dijkstra_pairs(lab, seeds)
  assert np.array_equal(dist, D2.astype(np.float32)) and np.array_equal(S, S2)
  seed_index = np.flatnonzero(seeds.T.reshape(-1, order="F"))[0]          # x-fastest
  assert np.isfinite(dist[lab != 0]).all() and (S[lab != 0] == seed_index).all()
  # steps from the seed, each of length 1 along the runs and sqrt(ndim) along the diagonals
  step = math.sqrt(lab.ndim) if name.startswith("diagonal") else 1.0
  at = np.argwhere(seeds)[0]
  for p in np.argwhere(lab != 0):
    acc = 0.0
    for _ in range(int(np.abs(p - at).max())):
      acc += step
    assert dist[tuple(p)] == np.float32(acc), (name, p)
