"""The CPU restatement of geodesic_distance and the volumes it is tested on.

restate() builds the graph exactly as include/edt_b200.h defines it -- same-label 26- (2-D: 8-, 1-D: 2-)
neighbours, label 0 and the volume's outside uncrossable, step lengths formed from the float32 weights in
Python double with the squares summed in the order x, y, z -- and takes D from scipy.sparse.csgraph.dijkstra(min_only=True).  S is
the least fixed point of S[v] = min(S[v], S[u]) over the tight edges (D[v] == D[u] + w in double), from the
seed's own x-fastest linear index on the seeds: the least seed with a tight path to v.  Arrays are in array
axes; `order` says which axis is x (the last of a C-ordered array, the first of an F-ordered one).
"""
import heapq
import itertools
import math

import numpy as np
import scipy.sparse
import scipy.sparse.csgraph

# the tiles of the GPU passes, in x-fastest axes
TILE = {1: (256,), 2: (16, 16), 3: (8, 8, 8)}


def weight(w):
  """A weight as the C ABI takes it: rounded to float32, then promoted to double."""
  return float(np.float32(w))


def step_length(delta, w_xfirst):
  """sqrt of the squares of (delta_k * w_k) summed in double in the order x, y, z (delta and w x first), each
  weight rounded to float32 first."""
  s = 0.0
  for d, w in zip(delta, w_xfirst):
    if d:
      s += weight(w) * weight(w)
  return math.sqrt(s)


def _xfirst(arr, order):
  """The array with x as its first axis (a view)."""
  return arr if order == "F" else arr.T


def edges(labels, w, order="C"):
  """(a, b, length): every undirected graph edge once, voxels as x-fastest linear indices."""
  lab = _xfirst(np.asarray(labels), order)
  wx = list(w) if order == "F" else list(w)[::-1]
  nd, shape = lab.ndim, lab.shape
  flat = np.arange(lab.size).reshape(shape, order="F")        # x-fastest linear index
  A, B, L = [], [], []
  for delta in itertools.product((-1, 0, 1), repeat=nd):
    if delta <= (0,) * nd:                                     # one of each +/- pair, and not 0
      continue
    src = tuple(slice(max(0, -d), s - max(0, d)) for d, s in zip(delta, shape))
    dst = tuple(slice(max(0, d), s - max(0, -d)) for d, s in zip(delta, shape))
    la, lb = lab[src], lab[dst]
    m = (la == lb) & (la != 0)
    A.append(flat[src][m])
    B.append(flat[dst][m])
    L.append(np.full(int(m.sum()), step_length(delta, wx)))
  if not A:
    return np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0)
  return np.concatenate(A), np.concatenate(B), np.concatenate(L)


def seed_mask(labels, seeds):
  return (np.asarray(seeds) != 0) & (np.asarray(labels) != 0)


def restate(labels, seeds, w=None, order="C"):
  """(dist float32, S int64 x-fastest linear seed index or -1), both in array axes, for ONE volume."""
  labels = np.asarray(labels)
  if w is None:
    w = (1.0,) * labels.ndim
  n = labels.size
  a, b, length = edges(labels, w, order)
  src = np.flatnonzero(_xfirst(seed_mask(labels, seeds), order).reshape(-1, order="F"))
  D = np.full(n, np.inf)
  if src.size:
    g = scipy.sparse.coo_matrix((length, (a, b)), shape=(n, n)).tocsr()
    D = scipy.sparse.csgraph.dijkstra(g, directed=False, indices=src, min_only=True)
  S = tight_indices(D, src, a, b, length)
  dist = D.astype(np.float32)
  shape_x = _xfirst(labels, order).shape
  back = lambda x: _from_xfirst(x.reshape(shape_x, order="F"), order)
  return back(dist), back(S)


def _from_xfirst(x, order):
  return np.asfortranarray(x) if order == "F" else np.ascontiguousarray(x.T)


def tight_indices(D, src, a, b, length):
  """The least fixed point of S over the tight edges: S = own index on the seeds, -1 (none) elsewhere."""
  big = np.iinfo(np.int64).max
  S = np.full(D.size, big, np.int64)
  S[src] = src
  # the tight edges, directed from the nearer end: D[v] == D[u] + w with D[v] finite
  u = np.concatenate([a, b])
  v = np.concatenate([b, a])
  w = np.concatenate([length, length])
  t = np.isfinite(D[v]) & (D[u] + w == D[v])
  u, v = u[t], v[t]
  # relax the out-edges of the voxels whose S went down, until none does (CSR by source)
  order = np.argsort(u, kind="stable")
  u, v = u[order], v[order]
  indptr = np.searchsorted(u, np.arange(D.size + 1))
  frontier = np.asarray(src, np.int64)
  while frontier.size:
    starts, counts = indptr[frontier], indptr[frontier + 1] - indptr[frontier]
    e = np.repeat(starts - np.concatenate([[0], np.cumsum(counts)[:-1]]), counts) + np.arange(int(counts.sum()))
    eu, ev = u[e], v[e]
    old = S[ev]
    np.minimum.at(S, ev, S[eu])
    frontier = np.unique(ev[S[ev] < old])
  S[S == big] = -1
  return S


def dijkstra_pairs(labels, seeds, w=None, order="C"):
  """An independent check: heapq Dijkstra over (D, S) pairs in lexicographic order, on a dict of
  neighbours built voxel by voxel.  Returns (D float64, S) in array axes."""
  labels = np.asarray(labels)
  if w is None:
    w = (1.0,) * labels.ndim
  lab = _xfirst(labels, order)
  wx = list(w) if order == "F" else list(w)[::-1]
  shape = lab.shape
  nd = lab.ndim
  strides = [int(np.prod(shape[:k])) for k in range(nd)]
  flat_lab = lab.reshape(-1, order="F")
  seeds_x = _xfirst(seed_mask(labels, seeds), order).reshape(-1, order="F")
  D = np.full(lab.size, np.inf)
  S = np.full(lab.size, -1, np.int64)
  heap = []
  for i in np.flatnonzero(seeds_x):
    D[i], S[i] = 0.0, i
    heap.append((0.0, int(i), int(i)))
  heapq.heapify(heap)
  done = np.zeros(lab.size, bool)
  deltas = [d for d in itertools.product((-1, 0, 1), repeat=nd) if any(d)]
  lengths = [step_length(d, wx) for d in deltas]
  while heap:
    d, s, i = heapq.heappop(heap)
    if done[i] or (d, s) != (D[i], S[i]):
      continue
    done[i] = True
    coord = [(i // strides[k]) % shape[k] for k in range(nd)]
    for delta, ln in zip(deltas, lengths):
      c = [coord[k] + delta[k] for k in range(nd)]
      if any(x < 0 or x >= shape[k] for k, x in enumerate(c)):
        continue
      j = sum(x * st for x, st in zip(c, strides))
      if flat_lab[j] != flat_lab[i]:
        continue
      nd_ = d + ln
      if (nd_, s) < (D[j], S[j] if S[j] >= 0 else np.iinfo(np.int64).max):
        D[j], S[j] = nd_, s
        heapq.heappush(heap, (nd_, s, j))
  back = lambda x: _from_xfirst(x.reshape(shape, order="F"), order)
  return back(D), back(S)


def index_planes(S, shape, order="C"):
  """S (x-fastest linear indices within the volume, -1 none) as int32 coordinate planes in array axes."""
  S = np.asarray(S)
  shape_x = tuple(shape) if order == "F" else tuple(shape)[::-1]
  planes = np.full((len(shape),) + tuple(shape), -1, np.int32)
  ok = S >= 0
  coords_x = np.unravel_index(S[ok], shape_x, order="F")
  coords = coords_x if order == "F" else coords_x[::-1]
  for k in range(len(shape)):
    planes[k][ok] = coords[k]
  return planes


# ---- case builders ------------------------------------------------------------------------------------

def random_labels(rng, shape, nlabels=3, block=3, dtype=np.uint16):
  """Blocky random labels 0..nlabels: blocks of `block` voxels with a few single-voxel flips."""
  coarse = rng.integers(0, nlabels + 1, tuple(-(-s // block) for s in shape))
  lab = coarse
  for ax, s in enumerate(shape):
    lab = np.repeat(lab, block, axis=ax).take(np.arange(s), axis=ax)
  flip = rng.random(shape) < 0.05
  lab = np.where(flip, rng.integers(0, nlabels + 1, shape), lab)
  return lab.astype(dtype)


def random_seeds(rng, shape, p=0.01, dtype=np.bool_):
  """Random seeds (some on background, which are ignored), at least one."""
  s = rng.random(shape) < p
  s.reshape(-1)[rng.integers(0, s.size)] = True
  return s.astype(dtype)


def corridor_through_corner(nd, tile=None, cross="corner"):
  """A one-voxel-thick corridor (x-fastest axes; transpose for C order) that crosses from one tile into the
  next only through a tile `corner` (3-D) or `edge`: it runs along the tile's last x row, steps diagonally
  into the neighbour tile and goes on; its two ends are the seed and the far voxel."""
  tile = tile or TILE[nd]
  shape = tuple(2 * t + 3 for t in tile)
  lab = np.zeros(shape, np.uint8)
  if nd == 1:
    lab[1:-1] = 1
    return lab
  c = [t - 1 for t in tile]                      # the tile's last voxel on every axis
  path = []
  for x in range(0, c[0] + 1):                   # along x inside tile (0, 0, 0) at the other coordinates' last
    path.append([x] + c[1:])
  step = [1] * nd if cross == "corner" else [1, 1] + [0] * (nd - 2)
  at = [c[k] + step[k] for k in range(nd)]
  path.append(at)
  for x in range(at[0] + 1, shape[0] - 1):
    path.append([x] + at[1:])
  for p in path:
    lab[tuple(p)] = 1
  return lab


def serpentine(shape, period=4):
  """A serpentine maze of label 1 in x-fastest axes: walls of label 0 across every `period`-th y row,
  open at alternate ends, extruded along z."""
  lab = np.ones(shape, np.uint8)
  sx, sy = shape[0], shape[1]
  for k, y in enumerate(range(period - 1, sy - 1, period)):
    lab[:, y] = 0
    gap = sx - 1 if k % 2 == 0 else 0
    lab[gap, y] = 1
  return lab


def spiral(n):
  """A square spiral corridor of label 1 in an n x n image (x-fastest): walls of 0 one voxel thick."""
  lab = np.zeros((n, n), np.uint8)
  x, y, d = 0, 0, 0
  dirs = [(1, 0), (0, 1), (-1, 0), (0, -1)]
  lo = [0, 0]
  hi = [n - 1, n - 1]
  lab[0, 0] = 1
  while True:
    dx, dy = dirs[d]
    moved = False
    while True:
      nx, ny = x + dx, y + dy
      if not (0 <= nx < n and 0 <= ny < n):
        break
      ax, ay = nx + dx, ny + dy
      if 0 <= ax < n and 0 <= ay < n and lab[ax, ay]:
        break
      # keep a wall between this arm and the arm beside it
      side = [(nx + dy, ny + dx), (nx - dy, ny - dx)]
      if any(0 <= a < n and 0 <= b < n and lab[a, b] and (a, b) != (x, y) for a, b in side):
        break
      x, y = nx, ny
      lab[x, y] = 1
      moved = True
    if not moved:
      break
    d = (d + 1) % 4
  return lab


def seeded_at_tile_borders():
  """(name, labels, seeds) in C order: thin structures whose one seed sits on a tile's face, edge or corner,
  where the seed is the structure's only contact with the tiles beyond it -- a 1-D run seeded at x = 255 and
  256, a 3-D x-corridor one voxel thick seeded at x = 7 and 8, and 2-D and 3-D diagonals seeded at a tile
  corner and just past it."""
  cases = []
  for n, x in ((300, 255), (512, 255), (512, 256)):
    lab = np.ones(n, np.uint8)
    seeds = np.zeros(n, bool)
    seeds[x] = True
    cases.append(("run%d_at_%d" % (n, x), lab, seeds))
  for x in (7, 8):
    lab = np.zeros((8, 8, 20), np.uint16)                # (z, y, x)
    lab[3, 3, :] = 2
    seeds = np.zeros(lab.shape, bool)
    seeds[3, 3, x] = True
    cases.append(("x_corridor_at_%d" % x, lab, seeds))
  for nd, n, at in ((2, 40, (15, 16)), (3, 20, (7, 8))):
    for c in at:
      lab = np.zeros((n,) * nd, np.uint8)
      lab[(np.arange(n),) * nd] = 1
      seeds = np.zeros(lab.shape, bool)
      seeds[(c,) * nd] = True
      cases.append(("diagonal%dd_at_%d" % (nd, c), lab, seeds))
  return cases
