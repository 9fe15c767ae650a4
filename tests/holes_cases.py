"""Restatements of fill_holes and dust (include/edt_b200.h), each built two independent ways, the defects they
can plant, and the volumes the tests run them on.

fill_holes:
  "scipy"  scipy.ndimage.label of the background, OPEN from the labels found on the faces, the bordering labels
           of each component from scipy.ndimage.binary_dilation of each label's mask;
  "flood"  plain numpy: components by least-index propagation over shifted copies, OPEN by a flood from the
           faces, the bordering labels by a scan over every neighbour offset.
dust:
  "scipy"  scipy.ndimage.label of each label's mask and np.bincount;
  "cc"     components_cases.restate_cc (a breadth-first search) and np.bincount.

Volumes are C-ordered numpy arrays here; an F-ordered array is restated as its transpose (x-fastest in both),
which is the same thing because the definitions do not depend on the order of the axes.

Planted defects (DEFECTS): the restatement computes what a kernel with that fault would."""
import numpy as np
import scipy.ndimage as ndi

import components_cases as cc

DEFECTS = ("diagonal_claims_ignored", "one_face_missed", "first_claim_wins", "max_size_off_by_one",
           "threshold_off_by_one", "stack_faces_shared")


def structure(nd, connectivity):
  return ndi.generate_binary_structure(nd, connectivity)


def _faces(shape, defect=None, stack_pos=None):
  """The voxels on a face of the volume.  one_face_missed: the high face of the last (fastest) axis is not
  one.  stack_faces_shared with stack_pos = (i, n): the faces of the slowest axis count only at the stack's
  ends (volume 0's low face, volume n-1's high face)."""
  face = np.zeros(shape, bool)
  for ax in range(len(shape)):
    lo = [slice(None)] * len(shape)
    hi = [slice(None)] * len(shape)
    lo[ax], hi[ax] = 0, -1
    shared = defect == "stack_faces_shared" and stack_pos is not None and ax == 0
    if not (shared and stack_pos[0] > 0):
      face[tuple(lo)] = True
    if not (defect == "one_face_missed" and ax == len(shape) - 1) and not (shared and stack_pos[0] < stack_pos[1] - 1):
      face[tuple(hi)] = True
  return face


def _shift(a, d, fill):
  """b[p] = a[p + d], `fill` outside."""
  out = np.full(a.shape, fill, a.dtype)
  src = tuple(slice(max(k, 0), a.shape[i] + min(k, 0)) for i, k in enumerate(d))
  dst = tuple(slice(max(-k, 0), a.shape[i] + min(-k, 0)) for i, k in enumerate(d))
  out[dst] = a[src]
  return out


def _decide(labels, comp, n, is_open, sizes, bordering, max_size, defect):
  """The result from per-component facts: comp (0: not background), is_open[c], sizes[c], bordering[c] the
  sorted distinct bordering labels (first_claim_wins: in the order claimed)."""
  out = labels.copy()
  fill = np.zeros(n + 1, labels.dtype)
  ok = np.zeros(n + 1, bool)
  for c in range(1, n + 1):
    labs = bordering[c]
    if is_open[c] or len(labs) == 0 or (len(labs) > 1 and defect != "first_claim_wins"):
      continue
    if max_size is not None and not (sizes[c] < max_size if defect == "max_size_off_by_one" else sizes[c] <= max_size):
      continue
    ok[c], fill[c] = True, labs[0]
  hole = ok[comp] & (comp > 0)
  out[hole] = fill[comp][hole]
  return out, int(hole.sum())


def _bits(labels):
  """The labels as unsigned integers of their width (bool as uint8): what the definitions compare."""
  return labels.view(np.uint8) if labels.dtype == np.bool_ else labels.view(np.dtype("u%d" % labels.itemsize))


def fill_scipy(labels, connectivity=1, max_size=None, defect=None, stack_pos=None):
  lab = _bits(labels)
  st = structure(lab.ndim, connectivity)
  bg = lab == 0
  comp, n = ndi.label(bg, st)
  is_open = np.zeros(n + 1, bool)
  is_open[np.unique(comp[_faces(lab.shape, defect, stack_pos) & bg])] = True
  is_open[0] = False
  sizes = np.bincount(comp.ravel(), minlength=n + 1)
  claim_st = structure(lab.ndim, 1) if defect == "diagonal_claims_ignored" else st
  bordering = [[] for _ in range(n + 1)]
  for L in np.unique(lab[~bg]):
    touched = np.unique(comp[ndi.binary_dilation(lab == L, claim_st) & bg])
    for c in touched[touched > 0]:
      bordering[c].append(L)
  if defect == "first_claim_wins":          # the label of the first bordering voxel in memory order wins
    first = {}
    for d in cc.offsets(lab.ndim, connectivity):
      nb = _shift(lab, d, 0)
      for idx in np.flatnonzero(bg & (nb != 0)):
        c = comp.flat[idx]
        if c not in first or idx < first[c][0]:
          first[c] = (idx, nb.flat[idx])
    bordering = [[first[c][1]] if c in first else [] for c in range(n + 1)]
  out, filled = _decide(lab, comp, n, is_open, sizes, bordering, max_size, defect)
  return out.view(labels.dtype), filled


def fill_flood(labels, connectivity=1, max_size=None, defect=None, stack_pos=None):
  lab = _bits(labels)
  nd = lab.ndim
  offs = cc.offsets(nd, connectivity)
  bg = lab == 0
  big = np.iinfo(np.int64).max
  # components: every background voxel takes the least index of its component
  idx = np.where(bg, np.arange(lab.size).reshape(lab.shape), big)
  while True:
    nxt = idx
    for d in offs:
      nxt = np.minimum(nxt, np.where(bg, _shift(idx, d, big), big))
    if np.array_equal(nxt, idx):
      break
    idx = nxt
  # open: flood from the faces through the background
  reach = bg & _faces(lab.shape, defect, stack_pos)
  while True:
    nxt = reach.copy()
    for d in offs:
      nxt |= bg & _shift(reach, d, False)
    if np.array_equal(nxt, reach):
      break
    reach = nxt
  roots = np.unique(idx[bg])
  comp = np.zeros(lab.shape, np.int64)
  comp[bg] = np.searchsorted(roots, idx[bg]) + 1
  n = roots.size
  is_open = np.zeros(n + 1, bool)
  is_open[np.unique(comp[reach])] = True
  is_open[0] = False
  sizes = np.bincount(comp.ravel(), minlength=n + 1)
  scan = cc.offsets(nd, 1) if defect == "diagonal_claims_ignored" else offs
  pairs = set()
  first = {}
  for d in scan:
    nb = _shift(lab, d, 0)
    hit = bg & (nb != 0)
    for i, c, L in zip(np.flatnonzero(hit), comp[hit], nb[hit]):
      pairs.add((int(c), L))
      if int(c) not in first or i < first[int(c)][0]:
        first[int(c)] = (i, L)
  bordering = [[] for _ in range(n + 1)]
  for c, L in sorted(pairs):
    bordering[c].append(L)
  if defect == "first_claim_wins":
    bordering = [[first[c][1]] if c in first else [] for c in range(n + 1)]
  out, filled = _decide(lab, comp, n, is_open, sizes, bordering, max_size, defect)
  return out.view(labels.dtype), filled


FILL = {"scipy": fill_scipy, "flood": fill_flood}


def restate_fill(labels, connectivity=1, max_size=None, order="C", how="scipy", defect=None, stacked=False):
  """(result, filled) of fill_holes, in the input's memory order; for a stack, filled is an int64 array."""
  a = np.asarray(labels)
  if order == "F":
    out, filled = restate_fill(np.ascontiguousarray(a.T), connectivity, max_size, "C", how, defect, stacked)
    return np.asfortranarray(out.T), filled
  if stacked:
    n = a.shape[0]
    res = [FILL[how](a[i], connectivity, max_size, defect, (i, n)) for i in range(n)]
    return (np.stack([r[0] for r in res]) if n else a.copy()), np.array([r[1] for r in res], np.int64)
  return FILL[how](a, connectivity, max_size, defect)


def dust_scipy(labels, threshold, connectivity=1, invert=False, defect=None):
  lab = _bits(labels)
  keep = np.zeros(lab.shape, bool)
  for L in np.unique(lab[lab != 0]):
    comp, _ = ndi.label(lab == L, structure(lab.ndim, connectivity))
    sizes = np.bincount(comp.ravel())
    big = sizes > threshold if defect == "threshold_off_by_one" else sizes >= threshold
    keep |= (comp > 0) & (big[comp] != invert)
  return np.where(keep, lab, 0).astype(lab.dtype).view(labels.dtype)


def dust_cc(labels, threshold, connectivity=1, invert=False, defect=None):
  lab = _bits(labels)
  comp = cc.restate_cc(lab, connectivity, "C", "bfs")
  sizes = np.bincount(comp.ravel())
  big = sizes > threshold if defect == "threshold_off_by_one" else sizes >= threshold
  keep = (comp > 0) & (big[comp] != invert)
  return np.where(keep, lab, 0).astype(lab.dtype).view(labels.dtype)


DUST = {"scipy": dust_scipy, "cc": dust_cc}


def restate_dust(labels, threshold, connectivity=1, invert=False, order="C", how="scipy", defect=None, stacked=False):
  a = np.asarray(labels)
  if order == "F":
    return np.asfortranarray(restate_dust(np.ascontiguousarray(a.T), threshold, connectivity, invert, "C", how,
                                          defect, stacked).T)
  if stacked:
    return np.stack([DUST[how](v, threshold, connectivity, invert, defect) for v in a]) if a.shape[0] else a.copy()
  return DUST[how](a, threshold, connectivity, invert, defect)


# ---- volumes ------------------------------------------------------------------------------------------------

def random_mask(rng, shape, p=0.55):
  return rng.random(shape) < p


def random_labels(rng, shape, nlabels=3, p=0.6):
  """Labels 1..nlabels on about a fraction p of the voxels: many holes, gaps and specks."""
  lab = rng.integers(1, nlabels + 1, shape)
  return np.where(rng.random(shape) < p, lab, 0).astype(np.uint8)


def cell_with_nucleus(nd=2):
  """A cell (label 1, a square shell) around a nucleus (label 2) with a background gap between them, and a
  cavity in the nucleus.  Returns (labels, want) for every connectivity: the gap borders both labels and stays
  0, the cavity becomes 2."""
  n = 15
  r = np.abs(np.indices((n,) * nd) - n // 2).max(0)
  lab = np.zeros((n,) * nd, np.uint8)
  lab[(r >= 5) & (r <= 6)] = 1                             # the cell's wall
  lab[r <= 2] = 2                                          # the nucleus, inside a gap of radius 3..4
  lab[r == 0] = 0                                          # a cavity in the nucleus
  want = lab.copy()
  want[r == 0] = 2
  return lab, want


def diagonal_touch():
  """A single background voxel walled by label 1 on its faces, with label 2 at one diagonal: filled with 1 at
  connectivity 1, left 0 (MIXED) at connectivity 2."""
  lab = np.zeros((5, 5), np.uint8)
  lab[1:4, 1:4] = 1
  lab[2, 2] = 0
  lab[1, 1] = 2
  return lab


def sized_hole(size):
  """A 1-row background run of `size` voxels inside label 3 (3-D), the only hole."""
  lab = np.full((3, 3, size + 2), 3, np.uint16)
  lab[1, 1, 1:size + 1] = 0
  return lab


def stacked_slabs():
  """A stack of two 3-D volumes: in volume 0 a closed cavity of label 1; in volume 1 a pocket of label 1 that
  is open only through its low face of the slowest axis, the face it shares in memory with volume 0."""
  a = np.ones((2, 6, 6, 6), np.uint8)
  a[0, 2:4, 2:4, 2:4] = 0
  a[1, 0:3, 2:4, 2:4] = 0
  return a


def crossing_holes():
  """(name, labels, connectivity): the structures of components_cases.crossing_tiles, whose only link is one
  edge across a GPU tile's face, edge or corner (tiles of 16x8x8 in x-fastest axes, 32x32 in 2-D, 1024 in
  1-D), made background inside walls of label 1.  "closed": its voxels on the volume's faces are walled, so the
  rest is one hole and is filled.  "open": its last voxel in memory order is joined to the high x face, so the
  whole structure is open and nothing is filled -- unless a link across the tiles is lost."""
  cases = []
  for name, lab, conn in cc.crossing_tiles():
    s = lab != 0
    face = _faces(lab.shape)
    closed = np.where(s & ~face, 0, 1).astype(np.uint8)
    opened = closed.copy()
    p = np.unravel_index(np.flatnonzero(s)[-1], s.shape)
    opened[tuple(p[:-1]) + (slice(p[-1], None),)] = 0
    cases.append(("closed_" + name, closed, conn))
    cases.append(("open_" + name, opened, conn))
  return cases
