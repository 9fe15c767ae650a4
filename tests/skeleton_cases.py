"""The skeleton (edt_b200.skeletonize, edtb200_skeletonize in include/edt_b200.h) restated on the CPU:

  restate   the definition as written: R = medial_axis_cases.edtsq (the CPU oracle's edtsq, per volume for
            stacks); each volume turned x-fastest (its transpose when F-ordered) and thinned on its own:
            round t admits the labelled voxels still present with R <= theta_t = (t h)^2 (double), a final
            round admits the rest (R = +inf too); each cycle takes the end-point snapshot, then runs the
            steps k = 0 .. 2^ndim - 1, each deleting at once the admitted subfield-k voxels that are simple
            and were not end points at the start of the cycle; a round ends after a cycle that deletes
            nothing.  The steps are vectorised per subfield, the predicate is memoised by the 3x3x3 code.
  simple    the predicate on a neighbour code: bit j is the j-th of the 26 neighbours in (dz, dy, dx)
            order, the centre left out; 2-D codes use the 8 bits of the plane dz = 0.

`defect` plants one mistake each, so that the tests can show their checks notice it: "parallel" (all
subfields in one step), "no_endpoints", "step_endpoints" (the end-point test at the start of each step),
"background26" (the complement counted with 26-connectivity) and "voxel_order" (rounds by voxel layers --
the edtsq with unit weights -- instead of by R).

Also the checks the tests make: per-label topology invariants (components, complement components, Euler
characteristic) and thinness, and the volumes the tests run on, from morphology_cases.py.
"""
import numpy as np

import medial_axis_cases as mac
import morphology_cases as mc

KINDS = mc.KINDS
seeded = mc.seeded
voronoi = mc.voronoi
balls = mc.balls

OFFSETS = [(dz, dy, dx) for dz in (-1, 0, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1) if (dz, dy, dx) != (0, 0, 0)]


def _bits(pred):
  return sum(1 << j for j, o in enumerate(OFFSETS) if pred(o))


def _adjacency(pred):
  return [sum(1 << b for b, q in enumerate(OFFSETS) if q != o and pred(tuple(abs(u - v) for u, v in zip(o, q))))
          for o in OFFSETS]


ADJ26 = _adjacency(lambda d: max(d) <= 1)
ADJ6 = _adjacency(lambda d: sum(d) == 1)
N18 = _bits(lambda o: sum(map(abs, o)) <= 2)
SIX = _bits(lambda o: sum(map(abs, o)) == 1)
PLANE = _bits(lambda o: o[0] == 0)
PLANE4 = SIX & PLANE
ALL = (1 << 26) - 1


def _flood(region, start, adj):
  seen = frontier = start
  while frontier:
    nxt = 0
    while frontier:
      low = frontier & -frontier
      nxt |= adj[low.bit_length() - 1]
      frontier ^= low
    frontier = nxt & region & ~seen
    seen |= frontier
  return seen


def simple(code, nd=3, defect=None):
  """The simple-voxel predicate on one neighbour code (see the module's docstring)."""
  fg = int(code)
  if nd == 2:
    fg &= PLANE
  if not fg or _flood(fg, fg & -fg, ADJ26) != fg:
    return False
  if defect == "background26":
    region, seeds, adj = (ALL if nd == 3 else PLANE), None, ADJ26
  else:
    region, seeds, adj = (N18, SIX, ADJ6) if nd == 3 else (PLANE, PLANE4, ADJ6)
  bg = region & ~fg
  seeds = bg if seeds is None else seeds & bg
  if not seeds:
    return False
  return (seeds & ~_flood(bg, seeds & -seeds, adj)) == 0


_MEMO = {}


def simple_codes(codes, nd=3, defect=None):
  """simple() of every code of an int array, memoised by code."""
  memo = _MEMO.setdefault((nd, defect == "background26"), {})
  uniq, inv = np.unique(codes, return_inverse=True)
  out = np.array([memo[c] if c in memo else memo.setdefault(c, simple(c, nd, defect)) for c in uniq.tolist()],
                 bool)
  return out[inv.reshape(-1)] if uniq.size else np.zeros(0, bool)


def theta(t, h):
  """theta_t = (t h)^2 in double; t = +inf (the final round) gives +inf."""
  th = np.asarray(t, np.float64) * np.float64(h)
  return th * th


def round_of(r, h):
  """The least t >= 1 with theta_t >= R, per voxel; +inf for R = +inf (the final round)."""
  R = np.asarray(r, np.float64)
  fin = np.isfinite(R)
  t = np.where(fin, np.maximum(np.ceil(np.sqrt(np.where(fin, R, 0.0)) / h), 1.0), np.inf)
  while True:
    down = fin & (t > 1) & (theta(t - 1, h) >= R)
    if not down.any():
      break
    t = np.where(down, t - 1, t)
  while True:
    up = fin & (theta(t, h) < R)
    if not up.any():
      break
    t = np.where(up, t + 1, t)
  return t


def _codes(present, lab, at, offs):
  """The neighbour codes of the flat indices `at` of the padded volume: bit j set where neighbour j is
  present with the same label."""
  code = np.zeros(at.size, np.int64)
  own = lab[at]
  for j, o in enumerate(offs):
    n = at + o
    code |= (present[n] & (lab[n] == own)).astype(np.int64) << j
  return code


def thin(lab, r, h, defect=None, stats=None):
  """The skeleton of one x-fastest (C-ordered, (z, y, x) or (y, x)) volume, given its R and h."""
  nd = lab.ndim
  shape = lab.shape
  if nd == 2:
    lab, r = lab[None], r[None]
  L = np.pad(lab, 1).reshape(-1)
  P = np.pad(lab != 0, 1).reshape(-1)
  pz, py, px = (s + 2 for s in lab.shape)
  offs = [dz * py * px + dy * px + dx for dz, dy, dx in OFFSETS]
  zz, yy, xx = np.indices(lab.shape)
  flat = ((zz + 1) * py + (yy + 1)) * px + (xx + 1)
  on = lab != 0
  idx = flat[on]
  par = ((xx & 1) | (yy & 1) << 1 | (zz & 1) << 2)[on]
  parity = np.zeros(P.size, np.int8)
  parity[idx] = par
  keys = round_of(r[on], h)
  nsteps = 8 if nd == 3 else 4
  cand = np.zeros(0, np.int64)
  rounds = cycles = 0
  for t in np.unique(keys):                      # ascending, the final round (+inf) last
    cand = np.concatenate([cand, idx[keys == t]])
    rounds += 1
    while True:
      cand = cand[P[cand]]
      ends = np.zeros(cand.size, bool) if defect == "no_endpoints" else (
        np.bitwise_count(_codes(P, L, cand, offs)) == 1)
      changed = False
      groups = [np.ones(cand.size, bool)] if defect == "parallel" else [parity[cand] == k for k in range(nsteps)]
      for g in groups:
        if defect == "step_endpoints":
          ends = np.bitwise_count(_codes(P, L, cand, offs)) == 1
        sel = cand[g & ~ends & P[cand]]
        if sel.size:
          gone = sel[simple_codes(_codes(P, L, sel, offs), nd, defect)]
          if gone.size:
            P[gone] = False
            changed = True
      cycles += 1
      if not changed:
        break
  if stats is not None:
    stats.update(rounds=rounds, cycles=cycles)
  return P.reshape(lab.shape[0] + 2, py, px)[1:-1, 1:-1, 1:-1].reshape(shape)


def restate(labels, anisotropy=None, black_border=False, order="C", stacked=False, defect=None, r=None):
  """The skeleton of `labels` by the definition (order: the memory order the call sees); r: its R when the
  caller has it."""
  labels = np.asarray(labels)
  vnd = labels.ndim - (1 if stacked else 0)
  w = (1.0,) * vnd if anisotropy is None else tuple(np.atleast_1d(np.asarray(anisotropy, np.float64)))
  if defect == "voxel_order":
    r, h = mac.edtsq(labels, None, black_border, order, stacked), 1.0
  else:
    h = float(np.min(np.float32(w)))
    if r is None:
      r = mac.edtsq(labels, anisotropy, black_border, order, stacked)
  vols, axis = mac._volumes(labels, order, stacked)
  rvols, _ = mac._volumes(r, order, stacked)
  out = []
  for v, rv in zip(vols, rvols):
    if order == "F":
      out.append(thin(np.ascontiguousarray(v.T), np.ascontiguousarray(rv.T), h, defect).T)
    else:
      out.append(thin(np.ascontiguousarray(v), np.ascontiguousarray(rv), h, defect))
  return out[0] if axis is None else np.stack(out, axis=axis)


# ---- the checks ---------------------------------------------------------------------------------------

def euler(mask):
  """The Euler characteristic of the union of the closed voxels (pixels) of `mask`: the alternating count
  of the cells of its cubical complex.  A cell spans some axes from its lower corner; it belongs where a
  voxel it bounds is set, i.e. the voxel at the corner or the one below it along each axis it does not
  span."""
  import itertools
  m = np.pad(np.asarray(mask, bool), 1)
  total = 0
  for span in itertools.product((0, 1), repeat=m.ndim):
    cells = m
    for a, spans in enumerate(span):
      if not spans:
        cells = cells | np.roll(cells, 1, axis=a)
    total += (-1) ** sum(span) * int(cells.sum())
  return total


def invariants(mask):
  """(components, complement components, Euler characteristic) of one label's mask: 26- (2-D: 8-)
  connected voxels, a 6- (2-D: 4-) connected complement that includes everything outside."""
  from scipy import ndimage
  m = np.asarray(mask, bool)
  nd = m.ndim
  fg = ndimage.label(m, structure=np.ones((3,) * nd, bool))[1]
  bg = ndimage.label(~np.pad(m, 1), structure=ndimage.generate_binary_structure(nd, 1))[1]
  return fg, bg, euler(m)


def label_boxes(labels):
  """{label: slices of its bounding box grown by one voxel} for every non-zero label."""
  from scipy import ndimage
  labels = np.asarray(labels)
  keys = np.unique(labels[labels != 0])
  out = {}
  for k in keys.tolist():
    where = np.nonzero(labels == k)
    out[k] = tuple(slice(max(int(a.min()) - 1, 0), int(a.max()) + 2) for a in where)
  return out


def topology_kept(labels, skeleton):
  """The labels whose invariants the skeleton changes (empty when every label keeps them)."""
  labels = np.asarray(labels)
  bad = []
  for k, box in label_boxes(labels).items():
    if invariants(labels[box] == k) != invariants(skeleton[box] & (labels[box] == k)):
      bad.append(k)
  return bad


def not_thin(labels, skeleton):
  """The skeleton voxels that are simple and not end points (none when the skeleton is thin)."""
  labels = np.asarray(labels)
  nd = labels.ndim
  lab = np.where(skeleton, labels, 0)
  if nd == 2:
    lab = lab[None]
  L = np.pad(lab, 1).reshape(-1)
  P = L != 0
  pz, py, px = (s + 2 for s in lab.shape)
  offs = [dz * py * px + dy * px + dx for dz, dy, dx in OFFSETS]
  at = np.flatnonzero(P)
  codes = _codes(P, L, at, offs)
  bad = simple_codes(codes, nd) & (np.bitwise_count(codes) != 1)
  return int(bad.sum())
