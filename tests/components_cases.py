"""The CPU restatements of connected_components and extended_maxima, and the volumes they are tested on.

Every restatement works on one C-ordered volume, where memory order is numpy's flat order; an F-ordered
volume is restated as its transpose and transposed back (restate_cc / restate_em take `order`).

Connected components, three ways:
  cc_scipy    scipy.ndimage.label of each distinct key's mask, renumbered by least memory index;
  cc_bfs      a plain breadth-first search from every unnumbered node in memory order;
  cc_csgraph  scipy.sparse.csgraph.connected_components over the joined edges, renumbered by least index.
A key is a tuple of arrays that must all be equal for two neighbours to be joined: (labels,) for
connected_components, (labels, R) for the plateaus of extended_maxima.

R, the reconstruction by dilation of m under f, three ways:
  r_relax     numpy sweeps of R = max(R, min(f, R[u])) over every joined offset until nothing changes;
  r_flood     a priority flood (heapq): the highest pending value first, exact because it only compares;
  r_brute     (tiny volumes) R[v] = the largest threshold t with v in a component of {f >= t} that
              holds a u with m[u] >= t.

Each restatement can plant a defect, each one a way the GPU could go wrong (DEFECTS).
"""
import heapq
import itertools
from collections import deque

import numpy as np
import scipy.ndimage
import scipy.sparse
import scipy.sparse.csgraph

DEFECTS = ("connectivity_plus_one", "connectivity_minus_one", "numbered_backwards", "ge_in_marking",
           "negative_zero_apart", "nan_as_plus_inf")


def offsets(nd, connectivity):
  """Neighbour offsets (array axes) with between 1 and `connectivity` non-zero components."""
  return [d for d in itertools.product((-1, 0, 1), repeat=nd) if 0 < sum(map(bool, d)) <= connectivity]


def _conn(nd, connectivity, defect):
  if defect == "connectivity_plus_one":
    return min(nd, connectivity + 1) if connectivity < nd else connectivity
  if defect == "connectivity_minus_one":
    return max(1, connectivity - 1)
  return connectivity


def _shifted(a, d, fill):
  """b[p] = a[p + d] where p + d is inside the volume, else `fill`."""
  b = np.full_like(a, fill)
  src = tuple(slice(max(0, k), a.shape[i] - max(0, -k)) for i, k in enumerate(d))
  dst = tuple(slice(max(0, -k), a.shape[i] - max(0, k)) for i, k in enumerate(d))
  b[dst] = a[src]
  return b


def _same(a, b, defect=None):
  """Keys equal as the definition compares them (floats by value, NaN never occurs); defect
  negative_zero_apart compares float keys by their bits, so that -0.0 != +0.0."""
  if defect == "negative_zero_apart" and a.dtype.kind == "f":
    return a.view(np.uint32) == b.view(np.uint32)
  return a == b


def _renumber(comp, nodes):
  """comp: a component id per voxel (any ids) -> 1..n in increasing order of each component's least flat
  index, 0 off the nodes."""
  flat = comp.reshape(-1)
  idx = np.flatnonzero(nodes.reshape(-1))
  out = np.zeros(comp.size, np.int64)
  if idx.size:
    ids, first = np.unique(flat[idx], return_index=True)      # idx is increasing: first = least index
    rank = np.empty(ids.size, np.int64)
    rank[np.argsort(idx[first], kind="stable")] = np.arange(1, ids.size + 1)
    out[idx] = rank[np.searchsorted(ids, flat[idx])]
  return out.reshape(comp.shape)


def _backwards(out, nodes, defect):
  if defect != "numbered_backwards" or not out.any():
    return out
  n = out.max()
  return np.where(nodes & (out > 0), n + 1 - out, 0)


def cc_scipy(nodes, keys, connectivity, defect=None):
  nd = nodes.ndim
  structure = scipy.ndimage.generate_binary_structure(nd, _conn(nd, connectivity, defect))
  comp = np.zeros(nodes.shape, np.int64)
  combined = np.stack([k.astype(np.float64) if k.dtype.kind == "f" else k.astype(np.int64).astype(np.float64)
                       for k in keys], -1) if keys else None
  rows = combined[nodes] if keys else np.zeros((int(nodes.sum()), 0))
  if defect == "negative_zero_apart":
    rows = np.where(np.signbit(rows) & (rows == 0), -1e300, rows)
  if rows.shape[1] == 1:                           # one key: a plain unique, much faster than by rows
    _, inv = np.unique(rows[:, 0], return_inverse=True)
  else:
    _, inv = np.unique(rows, axis=0, return_inverse=True)
  kid = np.full(nodes.shape, -1, np.int64)
  kid[nodes] = inv.reshape(-1)
  base = 0
  for k in range(int(inv.max()) + 1 if inv.size else 0):
    lab, n = scipy.ndimage.label(kid == k, structure)
    comp[lab > 0] = lab[lab > 0] + base
    base += n
  return _backwards(_renumber(comp, nodes), nodes, defect)


def _joined_edges(nodes, keys, connectivity, defect):
  """(u, v) flat index pairs of every joined edge, each once (d forward)."""
  nd = nodes.ndim
  flat = np.arange(nodes.size).reshape(nodes.shape)
  us, vs = [], []
  for d in offsets(nd, _conn(nd, connectivity, defect)):
    if d <= tuple([0] * nd):
      continue
    ok = nodes & _shifted(nodes, d, False)
    for k in keys:
      ok &= _same(k, _shifted(k, d, k.dtype.type(0)), defect)
    us.append(flat[ok])
    vs.append(_shifted(flat, d, -1)[ok])
  return (np.concatenate(us) if us else np.zeros(0, np.int64)), (np.concatenate(vs) if vs else np.zeros(0, np.int64))


def cc_csgraph(nodes, keys, connectivity, defect=None):
  u, v = _joined_edges(nodes, keys, connectivity, defect)
  g = scipy.sparse.coo_matrix((np.ones(u.size, np.int8), (u, v)), shape=(nodes.size, nodes.size))
  _, comp = scipy.sparse.csgraph.connected_components(g, directed=False)
  return _backwards(_renumber(comp.reshape(nodes.shape), nodes), nodes, defect)


def cc_bfs(nodes, keys, connectivity, defect=None):
  nd = nodes.ndim
  offs = offsets(nd, _conn(nd, connectivity, defect))
  out = np.zeros(nodes.shape, np.int64)
  n = 0
  for start in zip(*np.nonzero(nodes)):            # memory order
    if out[start]:
      continue
    n += 1
    out[start] = n
    queue = deque([start])
    while queue:
      p = queue.popleft()
      for d in offs:
        q = tuple(a + b for a, b in zip(p, d))
        if any(c < 0 or c >= s for c, s in zip(q, nodes.shape)) or not nodes[q] or out[q]:
          continue
        if all(_same(np.asarray(k[p]), np.asarray(k[q]), defect) for k in keys):
          out[q] = n
          queue.append(q)
  return _backwards(out, nodes, defect)


CC = {"scipy": cc_scipy, "bfs": cc_bfs, "csgraph": cc_csgraph}


def _c_order(a, order):
  a = np.asarray(a)
  return a.T if order == "F" else a


def _nodes_keys(labels, shape):
  if labels is None:
    return np.ones(shape, bool), ()
  lab = np.asarray(labels)
  lab = lab.view(np.uint8) if lab.dtype == np.bool_ else lab
  return lab != 0, (lab,)


def restate_cc(labels, connectivity=1, order="C", how="csgraph", defect=None):
  """connected_components of one volume (array axes, `order` the array's memory order) as int64."""
  lab = _c_order(labels, order)
  nodes, keys = _nodes_keys(lab, lab.shape)
  out = CC[how](nodes, keys, connectivity, defect)
  return out.T if order == "F" else out


# ---- extended maxima --------------------------------------------------------------------------------------

def image_f(image, defect=None):
  """f: the image as float32, NaN as -inf (defect nan_as_plus_inf: as +inf), -0.0 as +0.0 (defect
  negative_zero_apart: kept)."""
  f = np.array(image, dtype=np.float32, copy=True)
  f[np.isnan(f)] = np.inf if defect == "nan_as_plus_inf" else -np.inf
  if defect != "negative_zero_apart":
    f[f == 0] = 0.0
  return f


def start_m(f, h, defect=None):
  m = (f.astype(np.float64) - np.float64(h)).astype(np.float32)
  if defect != "negative_zero_apart":
    m[m == 0] = 0.0
  return m


def _joined(nodes, keys, d):
  ok = nodes & _shifted(nodes, d, False)
  for k in keys:
    ok &= k == _shifted(k, d, k.dtype.type(0))
  return ok


def r_relax(f, m, nodes, keys, connectivity):
  R = np.where(nodes, m, -np.inf).astype(np.float32)
  offs = [(d, _joined(nodes, keys, d)) for d in offsets(f.ndim, connectivity)]
  while True:
    before = R.copy()
    for d, ok in offs:
      cand = np.minimum(f, _shifted(R, d, np.float32(-np.inf)))
      R = np.where(ok & (cand > R), cand, R)
    if np.array_equal(R.view(np.uint32), before.view(np.uint32)):
      return R


def r_flood(f, m, nodes, keys, connectivity):
  R = np.where(nodes, m, -np.inf).astype(np.float32)
  offs = offsets(f.ndim, connectivity)
  heap = [(-float(R[p]), p) for p in zip(*np.nonzero(nodes))]
  heapq.heapify(heap)
  while heap:
    negv, p = heapq.heappop(heap)
    if -negv < R[p]:
      continue
    for d in offs:
      q = tuple(a + b for a, b in zip(p, d))
      if any(c < 0 or c >= s for c, s in zip(q, f.shape)) or not nodes[q]:
        continue
      if any(k[p] != k[q] for k in keys):
        continue
      cand = min(f[q], R[p])
      if cand > R[q]:
        R[q] = cand
        heapq.heappush(heap, (-float(cand), q))
  return R


def r_brute(f, m, nodes, keys, connectivity):
  """R[v] = the largest threshold t (a value of m or f) for which v shares a component of {f >= t} (joined
  nodes) with some u whose m[u] >= t: the largest min(m[u], the lowest f on a path from u to v)."""
  R = np.where(nodes, m, -np.inf).astype(np.float32)
  structure = scipy.ndimage.generate_binary_structure(f.ndim, connectivity)
  groups = [nodes]
  if keys:
    groups = [nodes & (keys[0] == k) for k in np.unique(keys[0][nodes])]
  for g in groups:
    for t in np.unique(np.concatenate([m[g], f[g]])):
      lab, _ = scipy.ndimage.label(g & (f >= t), structure)
      hit = np.unique(lab[g & (f >= t) & (m >= t)])
      R = np.where(np.isin(lab, hit[hit > 0]), np.maximum(R, t), R)
  return R


RECON = {"relax": r_relax, "flood": r_flood, "brute": r_brute}


def maxima(R, nodes, keys, connectivity, how="csgraph", defect=None):
  """The maximum plateaus of R, numbered."""
  plateaus = CC[how](nodes, keys + (R,), connectivity, defect if defect != "numbered_backwards" else None)
  drop = nodes & (R == -np.inf)
  for d in offsets(R.ndim, connectivity):
    nb = _shifted(R, d, np.float32(-np.inf))
    ok = nodes & _shifted(nodes, d, False)
    for k in keys:
      ok &= k == _shifted(k, d, k.dtype.type(0))
    drop |= ok & ((nb >= R) & ~_same(nb, R, defect) if defect != "ge_in_marking" else (nb >= R))
  dropped = np.unique(plateaus[drop])
  keep = nodes & ~np.isin(plateaus, dropped)
  return _backwards(_renumber(plateaus, keep), keep, defect)


def restate_em(image, h=0.0, labels=None, connectivity=1, order="C", recon="relax", how="csgraph", defect=None):
  """extended_maxima of one volume (array axes, `order` the memory order) as int64."""
  img = _c_order(image, order)
  lab = None if labels is None else _c_order(labels, order)
  nodes, keys = _nodes_keys(lab, img.shape)
  f = image_f(img, defect)
  m = start_m(f, h, defect)
  R = f.copy() if h == 0 and recon == "relax" else RECON[recon](f, m, nodes, keys, _conn(f.ndim, connectivity, defect))
  out = maxima(R, nodes, keys, _conn(f.ndim, connectivity, defect), how, defect)
  return out.T if order == "F" else out


def out_dtype(shape, stacked=False):
  vol = int(np.prod(shape[1:] if stacked else shape))
  return np.int32 if vol < (1 << 31) else np.int64


# ---- volumes ----------------------------------------------------------------------------------------------

def random_labels(rng, shape, nlabels=3, block=3, p=0.08):
  """Blocky labels in 0..nlabels with a sprinkle of noise, uint8."""
  coarse = rng.integers(0, nlabels + 1, tuple(-(-s // block) for s in shape))
  lab = coarse
  for ax, s in enumerate(shape):
    lab = np.repeat(lab, block, axis=ax).take(np.arange(s), axis=ax)
  return np.where(rng.random(shape) < p, rng.integers(0, nlabels + 1, shape), lab).astype(np.uint8)


def random_image(rng, shape, levels=None):
  img = rng.random(shape).astype(np.float32)
  if levels:
    img = np.floor(img * levels).astype(np.float32)
  return img


def crossing_tiles():
  """(name, labels, connectivity) in C order: structures of label 1 whose only link is one edge across a GPU
  tile's face, edge or corner (tiles of 16x8x8 in x-fastest axes, 32x32 in 2-D, 1024 in 1-D), so that they
  are one component exactly when the border pass joins that edge."""
  cases = []
  run = np.zeros(2100, np.uint8)
  run[1000:1050] = 1
  cases.append(("run_across_1024", run, 1))
  for nd, n, at in ((2, 70, 31), (3, 40, 7)):
    for axis in range(nd):                             # a straight line across every tile face of one axis
      lab = np.zeros((n,) * nd, np.uint8)
      lab[tuple(slice(None) if k == axis else at for k in range(nd))] = 1
      cases.append(("%dd_line_axis%d" % (nd, axis), lab, 1))
    lab = np.zeros((n,) * nd, np.uint8)                # a diagonal through tile corners
    lab[(np.arange(n),) * nd] = 1
    cases.append(("%dd_diagonal" % nd, lab, nd))
  # 3-D: two bars meeting only across a tile edge of x = 15|16, y = 7|8 (connectivity 2) and a corner of
  # x = 15|16, y = 7|8, z = 7|8 (connectivity 3)
  for conn, d in ((2, (0, 1, 1)), (3, (1, 1, 1))):
    lab = np.zeros((16, 16, 32), np.uint16)
    lab[7, 7, :16] = 5
    lab[7 + d[0], 7 + d[1], 16:] = 5
    cases.append(("3d_meet_c%d" % conn, lab, conn))
  return cases
