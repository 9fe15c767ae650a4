"""The CPU restatement of watershed and the volumes it is tested on.

restate() follows the definition in include/edt_b200.h step by step: the graph of same-label neighbours under
`connectivity` (label 0 and the volume's outside uncrossable), altitudes as float32 with NaN read as +inf and
-0.0 as +0.0, the level L by a heapq minimax Dijkstra (it only compares float32 values, so it is exact), and
W by a breadth-first search over the tight edges for each distinct marker value in ascending order (read as
unsigned integers of the markers' width), never entering a seed, where the first visit wins.  flood() relaxes
the same equations with numpy, frontier by frontier, for volumes too large for heapq; brute() is a third
restatement for tiny volumes: L per marker from the connected components of every threshold set, and W from
tight-path reachability.  tiled() models the GPU's tile rounds, so that a defect of its worklists can be
planted.  Arrays are in array axes; `order` says which axis is x (the last of a C-ordered array, the first of
an F-ordered one).
"""
import heapq
import itertools
from collections import deque

import numpy as np
import scipy.sparse
import scipy.sparse.csgraph

# the tiles of the GPU passes, in x-fastest axes
TILE = {1: (256,), 2: (16, 16), 3: (8, 8, 8)}
# the defects a restatement can plant, each one a way the GPU could go wrong
DEFECTS = ("seeds_overwritten", "non_tight", "connectivity_plus_one", "nan_as_minus_inf")


def altitude(image, defect=None):
  """The image as float32, NaN as +inf (defect nan_as_minus_inf: as -inf) and -0.0 as +0.0."""
  f = np.array(image, dtype=np.float32, copy=True)
  f[np.isnan(f)] = -np.inf if defect == "nan_as_minus_inf" else np.inf
  f[f == 0] = 0.0
  return f


def unsigned(markers):
  """The markers as unsigned integers of their width (bool as uint8)."""
  m = np.asarray(markers)
  if m.dtype == np.bool_:
    return m.view(np.uint8)
  return m.view(np.dtype("u%d" % m.dtype.itemsize))


def out_dtype(markers):
  m = np.asarray(markers)
  return np.uint8 if m.dtype == np.bool_ else m.dtype


def offsets(nd, connectivity):
  """The neighbour offsets (x first) with between 1 and `connectivity` non-zero components."""
  return [d for d in itertools.product((-1, 0, 1), repeat=nd) if 0 < sum(map(bool, d)) <= connectivity]


class Graph:
  """One volume in x-fastest axes, padded by one voxel of label 0 on every side: flat (F-order) label,
  altitude, seed and marker arrays, and the flat offsets of the neighbours."""

  def __init__(self, image, markers, labels, connectivity, order, defect=None):
    image = np.asarray(image)
    xf = (lambda a: a) if order == "F" else (lambda a: np.asarray(a).T)
    self.shape_x = xf(image).shape
    nd = len(self.shape_x)
    lab = np.ones(self.shape_x, np.uint64) if labels is None else unsigned(xf(labels)).astype(np.uint64)
    pad = lambda a, v: np.pad(a, 1, constant_values=v).reshape(-1, order="F")
    self.lab = pad(lab, 0)
    self.f = pad(altitude(xf(image), defect), np.inf)
    self.m = pad(unsigned(xf(markers)).astype(np.uint64), 0)
    self.seed = (self.m != 0) & (self.lab != 0)
    self.inside = pad(np.ones(self.shape_x, bool), False)
    padded = tuple(s + 2 for s in self.shape_x)
    strides = [int(np.prod(padded[:k])) for k in range(nd)]
    conn = connectivity + 1 if defect == "connectivity_plus_one" else connectivity
    self.off = [sum(d * s for d, s in zip(delta, strides)) for delta in offsets(nd, min(conn, nd))]
    self.order = order
    self.padded = padded

  def neighbours(self, i):
    for o in self.off:
      j = i + o
      if self.lab[j] == self.lab[i] and self.lab[i] != 0:
        yield j

  def back(self, flat):
    """A padded flat array in the caller's array axes, without the padding."""
    x = flat.reshape(self.padded, order="F")[tuple(slice(1, -1) for _ in self.padded)]
    return np.asfortranarray(x) if self.order == "F" else np.ascontiguousarray(x.T)


def levels(g):
  """L by a minimax Dijkstra over (level, voxel) pairs."""
  L = np.full(g.lab.size, np.inf, np.float32)
  heap = []
  for i in np.flatnonzero(g.seed):
    L[i] = g.f[i]
    heap.append((float(L[i]), int(i)))
  heapq.heapify(heap)
  done = np.zeros(g.lab.size, bool)
  while heap:
    lv, i = heapq.heappop(heap)
    if done[i] or lv != L[i]:
      continue
    done[i] = True
    for j in g.neighbours(i):
      c = max(g.f[j], L[i])
      if c < L[j]:
        L[j] = c
        heapq.heappush(heap, (float(c), int(j)))
  return L


def tight(g, L, u, v, defect=None):
  """Whether the edge u -> v is tight (defect non_tight: every edge; seeds_overwritten: into seeds too)."""
  if g.seed[v] and defect != "seeds_overwritten":
    return False
  return defect == "non_tight" or L[v] == max(g.f[v], L[u])


def labels_of(g, L, defect=None):
  """W (marker values, 0 none) by a BFS over the tight edges per marker value in ascending order."""
  W = np.zeros(g.lab.size, np.uint64)
  W[g.seed] = g.m[g.seed]
  if defect in ("seeds_overwritten", "non_tight"):
    return relax_labels(g, L, W, defect)
  claimed = g.seed.copy()
  for m in np.unique(g.m[g.seed]):
    q = deque(int(i) for i in np.flatnonzero(g.seed & (g.m == m)))
    while q:
      u = q.popleft()
      for v in g.neighbours(u):
        if not claimed[v] and tight(g, L, u, v):
          claimed[v] = True
          W[v] = m
          q.append(v)
  return W


def relax_labels(g, L, W, defect):
  """W by min over the (defective) tight edges until nothing changes, for the planted defects that let a
  value reach a voxel the BFS above never enters."""
  none = np.iinfo(np.uint64).max
  cur = np.where(W == 0, none, W)
  cur[~g.inside | (g.lab == 0)] = none
  changed = True
  while changed:
    changed = False
    for v in np.flatnonzero(g.lab != 0):
      best = cur[v]
      for u in g.neighbours(v):
        if tight(g, L, u, v, defect) and cur[u] < best:
          best = cur[u]
      if best < cur[v]:
        cur[v] = best
        changed = True
  return np.where(cur == none, 0, cur).astype(np.uint64)


def restate(image, markers, labels=None, connectivity=1, order="C", defect=None):
  """(W in the markers' dtype, bool as uint8; L float32), both in array axes, for ONE volume."""
  g = Graph(image, markers, labels, connectivity, order, defect)
  L = levels(g)
  W = labels_of(g, L, defect)
  return g.back(W).astype(out_dtype(markers)), g.back(L)


def flood(image, markers, labels=None, connectivity=1, order="C"):
  """restate() by numpy frontiers: L and then W relaxed by np.minimum.at over the voxels that changed,
  until none does.  The same equations, for volumes too large for heapq."""
  g = Graph(image, markers, labels, connectivity, order)
  lab, f = g.lab, g.f
  L = np.full(lab.size, np.inf, np.float32)
  L[g.seed] = f[g.seed]
  frontier = np.flatnonzero(g.seed)
  while frontier.size:
    nxt = []
    for o in g.off:
      j = frontier + o
      ok = (lab[j] == lab[frontier]) & (lab[j] != 0)
      u, j = frontier[ok], j[ok]
      c = np.maximum(f[j], L[u])
      low = c < L[j]
      j, c = j[low], c[low]
      np.minimum.at(L, j, c)
      nxt.append(j)
    frontier = np.unique(np.concatenate(nxt)) if nxt else frontier[:0]
  none = np.iinfo(np.uint64).max
  W = np.full(lab.size, none, np.uint64)
  W[g.seed] = g.m[g.seed] - 1
  frontier = np.flatnonzero(g.seed)
  while frontier.size:
    nxt = []
    for o in g.off:
      j = frontier + o
      ok = (lab[j] == lab[frontier]) & (lab[j] != 0) & ~g.seed[j]
      u, j = frontier[ok], j[ok]
      ok = (L[j] == np.maximum(f[j], L[u])) & (W[u] < W[j])
      u, j = u[ok], j[ok]
      np.minimum.at(W, j, W[u])
      nxt.append(j)
    frontier = np.unique(np.concatenate(nxt)) if nxt else frontier[:0]
  W = W + np.uint64(1)                  # none wraps to 0
  return g.back(W).astype(out_dtype(markers)), g.back(L)


def brute(image, markers, labels=None, connectivity=1, order="C"):
  """A third restatement for tiny volumes.  L per marker value m: the least threshold t (over the
  altitudes and +inf) at which v shares a connected component of {f <= t} with a seed of m; L = min over m.
  W: the least m from whose seeds v is reachable over tight edges into non-seeds."""
  g = Graph(image, markers, labels, connectivity, order)
  n = g.lab.size
  a, b = [], []
  for i in np.flatnonzero(g.lab != 0):
    for j in g.neighbours(i):
      a.append(i)
      b.append(j)
  a, b = np.array(a, np.int64), np.array(b, np.int64)
  values = np.unique(np.concatenate([g.f[g.lab != 0], [np.inf]]))
  L = np.full(n, np.inf, np.float32)
  per_marker = {}
  for m in np.unique(g.m[g.seed]):
    seeds = np.flatnonzero(g.seed & (g.m == m))
    Lm = np.full(n, np.inf, np.float32)
    for t in values[::-1]:                 # from the top: every lower threshold that still connects wins
      keep = (g.f[a] <= t) & (g.f[b] <= t)
      adj = scipy.sparse.coo_matrix((np.ones(int(keep.sum())), (a[keep], b[keep])), shape=(n, n))
      _, comp = scipy.sparse.csgraph.connected_components(adj, directed=False)
      ok = np.zeros(n, bool)
      live = seeds[g.f[seeds] <= t]
      ok[np.isin(comp, comp[live])] = True
      ok &= (g.f <= t) & (g.lab != 0)
      Lm[ok] = t
    per_marker[m] = Lm
    L = np.minimum(L, Lm)
  W = np.zeros(n, np.uint64)
  W[g.seed] = g.m[g.seed]
  t = ~g.seed[b] & (L[b] == np.maximum(g.f[b], L[a]))
  for m in sorted(per_marker, reverse=True):           # the least m is written last
    seeds = np.flatnonzero(g.seed & (g.m == m))
    # node n: a source joined to every seed of m
    src = np.concatenate([a[t], np.full(seeds.size, n)])
    dst = np.concatenate([b[t], seeds])
    adj = scipy.sparse.coo_matrix((np.ones(src.size), (src, dst)), shape=(n + 1, n + 1)).tocsr()
    reached = scipy.sparse.csgraph.breadth_first_order(adj, n, directed=True, return_predecessors=False)
    hit = np.zeros(n + 1, bool)
    hit[reached] = True
    hit = hit[:n] & ~g.seed
    W[hit] = m
  return g.back(W).astype(out_dtype(markers)), g.back(L)


def tiled(image, markers, labels=None, connectivity=1, order="C", defect=None):
  """The GPU's rounds, modelled: tiles of TILE[nd] relaxed to their own fixed point from a worklist, each
  queueing the neighbour tiles that a changed voxel on its face, edge or corner touches through the
  connectivity; in round 1 the seeds count as changed.  defect round1_no_corner: round 1 does not queue
  across tile corners and edges for the seeds.  Returns (W, L) as restate() does."""
  g = Graph(image, markers, labels, connectivity, order)
  nd = len(g.shape_x)
  tile = TILE[nd]
  ntile = tuple(-(-s // t) for s, t in zip(g.shape_x, tile))
  coord = lambda i: [(i // int(np.prod(g.padded[:k]))) % g.padded[k] - 1 for k in range(nd)]
  members = {}
  for i in np.flatnonzero(g.inside):
    members.setdefault(tuple(c // t for c, t in zip(coord(i), tile)), []).append(int(i))
  allowed = [d for d in itertools.product((-1, 0, 1), repeat=nd) if 0 < sum(map(bool, d)) <= connectivity]

  def rounds(value, update, unset):
    queue = sorted({tuple(c // t for c, t in zip(coord(i), tile)) for i in np.flatnonzero(g.seed)})
    r = 1
    while queue:
      nxt = set()
      for t in queue:
        before = {i: value[i] for i in members[t]}
        while any([update(i) for i in members[t]]):
          pass
        for i in members[t]:
          changed = value[i] != before[i]
          if not changed and not (r == 1 and value[i] != unset):
            continue
          c = coord(i)
          e = [-1 if c[k] % tile[k] == 0 else 1 if c[k] % tile[k] == tile[k] - 1 else 0 for k in range(nd)]
          for d in allowed:
            if any(d[k] and d[k] != e[k] for k in range(nd)):
              continue
            if defect == "round1_no_corner" and r == 1 and not changed and sum(map(bool, d)) > 1:
              continue
            n = tuple(t[k] + d[k] for k in range(nd))
            if all(0 <= n[k] < ntile[k] for k in range(nd)):
              nxt.add(n)
      queue = sorted(nxt)
      r += 1

  L = np.full(g.lab.size, np.inf, np.float32)
  L[g.seed] = g.f[g.seed]

  def lower_level(i):
    if g.lab[i] == 0:
      return False
    best = min([L[i]] + [max(g.f[i], L[u]) for u in g.neighbours(i)])
    if best < L[i]:
      L[i] = best
      return True
    return False

  rounds(L, lower_level, np.float32(np.inf))
  none = np.iinfo(np.uint64).max
  W = np.full(g.lab.size, none, np.uint64)
  W[g.seed] = g.m[g.seed] - 1

  def lower_label(i):
    if g.lab[i] == 0 or g.seed[i]:
      return False
    best = min([W[i]] + [W[u] for u in g.neighbours(i) if L[i] == max(g.f[i], L[u])])
    if best < W[i]:
      W[i] = best
      return True
    return False

  rounds(W, lower_label, none)
  W = W + np.uint64(1)
  return g.back(W).astype(out_dtype(markers)), g.back(L)


# ---- case builders ------------------------------------------------------------------------------------

def random_case(rng, shape, nlabels=2, p=0.03, levels=None, block=3):
  """(image float32, markers uint16, labels uint8): blocky labels, a random image (quantised to `levels`
  values when given, so that plateaus and ties are common) and sparse markers with repeated values."""
  coarse = rng.integers(0, nlabels + 1, tuple(-(-s // block) for s in shape))
  lab = coarse
  for ax, s in enumerate(shape):
    lab = np.repeat(lab, block, axis=ax).take(np.arange(s), axis=ax)
  lab = np.where(rng.random(shape) < 0.05, rng.integers(0, nlabels + 1, shape), lab).astype(np.uint8)
  img = rng.random(shape).astype(np.float32)
  if levels:
    img = np.floor(img * levels).astype(np.float32)
  mk = np.where(rng.random(shape) < p, rng.integers(1, 6, shape), 0).astype(np.uint16)
  mk.reshape(-1)[rng.integers(0, mk.size)] = 3
  return img, mk, lab


def balls(shape, centres, radii):
  """(mask uint8, markers int32): the union of balls (array axes), markers 1, 2, ... at their centres."""
  mask = np.zeros(shape, bool)
  markers = np.zeros(shape, np.int32)
  for k, (c, r) in enumerate(zip(centres, radii)):
    box = tuple(slice(max(0, ci - r), min(s, ci + r + 1)) for ci, s in zip(c, shape))
    grid = np.ogrid[box]
    mask[box] |= sum((g - ci) ** 2 for g, ci in zip(grid, c)) <= r * r
    markers[tuple(c)] = k + 1
  return mask.astype(np.uint8), markers


def minus_edt(mask):
  """-edt(mask) by scipy, as float32."""
  import scipy.ndimage
  return -scipy.ndimage.distance_transform_edt(mask).astype(np.float32)


def seeded_at_tile_borders():
  """(name, image, markers, labels) in C order: thin structures whose one seed sits on a tile's face, edge
  or corner, where the seed is the structure's only contact with the tiles beyond it -- a 1-D run seeded at
  x = 255 and 256, a 3-D x-corridor seeded at x = 7 and 8, and 2-D and 3-D diagonals (connectivity ndim)
  seeded at a tile corner and just past it."""
  cases = []
  for n, x in ((300, 255), (512, 256)):
    mk = np.zeros(n, np.uint8)
    mk[x] = 4
    cases.append(("run%d_at_%d" % (n, x), np.arange(n, dtype=np.float32) % 7, mk, np.ones(n, np.uint8), 1))
  for x in (7, 8):
    lab = np.zeros((8, 8, 20), np.uint16)
    lab[3, 3, :] = 2
    mk = np.zeros(lab.shape, np.uint8)
    mk[3, 3, x] = 9
    img = np.cos(np.arange(lab.size, dtype=np.float32)).reshape(lab.shape)
    cases.append(("x_corridor_at_%d" % x, img, mk, lab, 1))
  for nd, n, at in ((2, 40, (15, 16)), (3, 20, (7, 8))):
    for c in at:
      lab = np.zeros((n,) * nd, np.uint8)
      lab[(np.arange(n),) * nd] = 1
      mk = np.zeros(lab.shape, np.uint8)
      mk[(c,) * nd] = 5
      img = np.sin(np.arange(lab.size, dtype=np.float32)).reshape(lab.shape)
      cases.append(("diagonal%dd_at_%d" % (nd, c), img, mk, lab, nd))
  return cases


def serpentine(shape, period=4):
  """A serpentine maze of label 1 in x-fastest axes: walls of label 0 across every `period`-th y row,
  open at alternate ends, extruded along z."""
  lab = np.ones(shape, np.uint8)
  sx, sy = shape[0], shape[1]
  for k, y in enumerate(range(period - 1, sy - 1, period)):
    lab[:, y] = 0
    lab[sx - 1 if k % 2 == 0 else 0, y] = 1
  return lab
