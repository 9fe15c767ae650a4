"""nearest_labels (edt_b200.nearest_labels, include/edt_b200.h) restated in numpy, twice.

per_pass    the definition the GPU equals bit for bit: one pass per axis in the order x, y, z (x the last
            numpy axis of a C-ordered array, the first of an F-ordered one), each walking its window
            d = 1, 2, ... R and keeping per voxel the k least (value, label) pairs with distinct labels.
            The X pass starts from the voxel itself at 0 (a non-zero label) and offers each labelled voxel
            d samples away at fl32(w2 d^2); every later pass starts from its own list and offers the entries
            of the rows d away, each v as fl32(fl64(w2 d^2) + fl64(v)), formed as
            parabolic_cases.line_pass forms its candidates.  A label keeps its least value, ties go to the
            smaller label read as an unsigned integer, pairs above B are dropped, and the walk stops once
            fl32(w2 d^2) exceeds the k-th value.
per_label   independent of the separability argument: every label's D_M = parabolic_cases.erode of its
            indicator (0 on M, +inf elsewhere), the cut at B, then the k least (D_M, M) pairs.

`defect` plants one mistake in per_pass so that the tests can show they notice it:
  "tie_order"          ties broken by the larger label;
  "no_dedup"           a label may occupy two slots;
  "keep_k_minus_1"     one slot is lost between passes;
  "early_exit_on_tie"  the walk stops when fl32(w2 d^2) equals the k-th value.

The label families (`volume`) are those the GPU tests run.
"""
import numpy as np

import parabolic_cases as pc

INF = np.float32(np.inf)
FLT_MAX = float(np.finfo(np.float32).max)
DEFECTS = ("tie_order", "no_dedup", "keep_k_minus_1", "early_exit_on_tie")
RADIUS_LIMIT = 256


def w2_of(w):
  with np.errstate(over="ignore"):
    return np.float64(np.float32(w) * np.float32(w))


def bound_of(max_distance):
  """B: the largest float32 whose float64 is at most max_distance^2."""
  L = float(max_distance) * float(max_distance)
  if L >= FLT_MAX:
    return np.float32(FLT_MAX)
  b = np.float32(L)
  if float(b) > L:
    b = np.nextafter(b, np.float32(-np.inf))
  return b


def radius_of(w, B):
  """R: the largest r with float64(w2) r^2 < nextafterf(B, +inf), capped at 2^62 (edtb200_bounded_plan)."""
  w2 = float(w2_of(w))
  above = float(np.nextafter(np.float32(B), np.float32(np.inf)))
  lo, hi = 0, 1 << 62
  while lo < hi:
    mid = lo + (hi - lo + 1) // 2
    if w2 * float(mid) * float(mid) < above:
      lo = mid
    else:
      hi = mid - 1
  return lo


def unsigned(labels):
  """The labels as uint64, read as unsigned integers of their own width (bool as one byte)."""
  a = np.asarray(labels)
  if a.dtype == np.bool_:
    a = a.view(np.uint8)
  elif a.dtype.kind == "i":
    a = a.view(np.dtype("u%d" % a.dtype.itemsize))
  return a.astype(np.uint64)


def _back(lab64, dtype):
  """uint64 labels back to `dtype`, bit for bit."""
  dtype = np.dtype(dtype)
  u = lab64.astype(np.dtype("u%d" % dtype.itemsize))
  return u.view(dtype)


def _pass_axes(nd, order, stacked):
  axes = list(range(nd))
  if stacked:
    axes = axes[1:] if order == "C" else axes[:-1]
  return axes, (list(reversed(axes)) if order == "C" else axes)


def _weights(axes, anisotropy):
  w = (1.0,) * len(axes) if anisotropy is None else tuple(float(a) for a in np.atleast_1d(np.asarray(anisotropy, np.float64)))
  assert len(w) == len(axes)
  return dict(zip(axes, w))


def select(vals, labs, k, defect=None):
  """The k least (value, label) pairs with distinct labels along axis 0 of candidates vals (float32, +inf:
  none) and labs (uint64), sorted; empty slots are (+inf, 0)."""
  labs = np.where(np.isinf(vals), np.uint64(0), labs)
  if defect != "no_dedup":
    o = np.lexsort((vals, labs), axis=0)               # by label, then value: each label's least comes first
    vals = np.take_along_axis(vals, o, 0)
    labs = np.take_along_axis(labs, o, 0)
    dup = np.zeros(vals.shape, bool)
    dup[1:] = labs[1:] == labs[:-1]
    vals = np.where(dup, INF, vals)
    labs = np.where(dup, np.uint64(0), labs)
  key = ~labs if defect == "tie_order" else labs
  o = np.lexsort((key, vals), axis=0)[:k]
  v = np.take_along_axis(vals, o, 0)
  lab = np.take_along_axis(labs, o, 0)
  if v.shape[0] < k:
    pad = (k - v.shape[0],) + v.shape[1:]
    v = np.concatenate([v, np.full(pad, INF)])
    lab = np.concatenate([lab, np.zeros(pad, np.uint64)])
  return v, np.where(np.isinf(v), np.uint64(0), lab)


def _shift(a, s, fill):
  """out[..., i] = a[..., i - s] along the last axis, `fill` where i - s is outside."""
  out = np.full_like(a, fill)
  n = a.shape[-1]
  if abs(s) < n:
    if s >= 0:
      out[..., s:] = a[..., :n - s]
    else:
      out[..., :n + s] = a[..., -s:]
  return out


def _line_pass(V, L, lab, w, B, k, defect):
  """One pass along the last axis.  First pass: lab (M, n) uint64, V = L = None.  Later: V, L (k, M, n)."""
  w2 = w2_of(w)
  n = (lab if V is None else V).shape[-1]
  if V is None:
    V = np.full((k,) + lab.shape, INF)
    L = np.zeros((k,) + lab.shape, np.uint64)
    V[0] = np.where(lab != 0, np.float32(0), INF)
    L[0] = lab
  V0, L0 = V, L                                          # the pass reads its input, never its own output
  R = min(radius_of(w, B), n - 1) if np.isfinite(w2) else 0
  for d in range(1, R + 1):
    wall64 = w2 * np.float64(d * d)
    wall = np.float32(wall64)
    kth = V[k - 1]
    stop = (wall >= kth) if defect == "early_exit_on_tie" else (wall > kth)
    stop = stop | (wall > B)
    if stop.all():
      break
    cv, cl = [], []
    for s in (d, -d):
      if lab is not None:
        nb = _shift(lab, s, np.uint64(0))
        cv.append(np.where(nb != 0, wall, INF)[None])
        cl.append(nb[None])
      else:
        sv = _shift(V0, s, INF)
        with np.errstate(over="ignore"):
          cv.append((wall64 + sv.astype(np.float64)).astype(np.float32))
        cl.append(_shift(L0, s, np.uint64(0)))
    cv = np.concatenate(cv)
    cv = np.where(cv > B, INF, cv)
    nv, nl = select(np.concatenate([V, cv]), np.concatenate([L, np.concatenate(cl)]), k, defect)
    V = np.where(stop, V, nv)
    L = np.where(stop, L, nl)
  return V, L


def per_pass(labels, max_distance, anisotropy=None, k=2, order="C", stacked=False, squared=True, defect=None):
  """(distances float32, nearest in labels' dtype), each of shape (k,) + labels.shape."""
  labels = np.asarray(labels)
  raw = unsigned(labels)
  axes, passes = _pass_axes(raw.ndim, order, stacked)
  weight = _weights(axes, anisotropy)
  B = bound_of(max_distance)
  V = L = None
  for m, axis in enumerate(passes):
    if V is None:
      moved = np.moveaxis(raw, axis, -1)
      shape = moved.shape
      v, lab = _line_pass(None, None, moved.reshape(-1, shape[-1]), weight[axis], B, k, defect)
    else:
      mv, ml = np.moveaxis(V, axis + 1, -1), np.moveaxis(L, axis + 1, -1)
      shape = mv.shape[1:]
      v, lab = _line_pass(mv.reshape(k, -1, shape[-1]), ml.reshape(k, -1, shape[-1]), None, weight[axis], B, k, defect)
    V = np.moveaxis(v.reshape((k,) + shape), -1, axis + 1)
    L = np.moveaxis(lab.reshape((k,) + shape), -1, axis + 1)
    if defect == "keep_k_minus_1" and m < len(passes) - 1:
      V = V.copy()
      L = L.copy()
      V[k - 1] = INF
      L[k - 1] = 0
  V = np.ascontiguousarray(V)
  return (V if squared else np.sqrt(V)), _back(np.ascontiguousarray(L), labels.dtype)


def per_label_values(labels, anisotropy=None, order="C", stacked=False):
  """(ids uint64, D float32 of shape (len(ids),) + labels.shape): every non-zero label's D_M."""
  raw = unsigned(labels)
  ids = np.unique(raw[raw != 0])
  D = np.stack([pc.erode(np.where(raw == m, np.float32(0), INF), anisotropy, order, stacked=stacked) for m in ids]) \
      if len(ids) else np.zeros((0,) + raw.shape, np.float32)
  return ids, D


def per_label(labels, max_distance, anisotropy=None, k=2, order="C", stacked=False, squared=True):
  labels = np.asarray(labels)
  ids, D = per_label_values(labels, anisotropy, order, stacked)
  B = bound_of(max_distance)
  D = np.where(D > B, INF, D)
  lab = np.broadcast_to(ids.reshape((-1,) + (1,) * labels.ndim), D.shape)
  V, L = select(D, lab, k)
  return (V if squared else np.sqrt(V)), _back(L, labels.dtype)


def brute_sqdist(labels, anisotropy):
  """(ids, S float64): the exact squared distance from every voxel to the nearest voxel of each label
  (weights along the array's axes), by brute force over every pair; small volumes only."""
  raw = unsigned(labels)
  w = np.asarray(anisotropy, np.float64)
  pts = np.indices(raw.shape).reshape(raw.ndim, -1).T * w
  ids = np.unique(raw[raw != 0])
  out = []
  for m in ids:
    sites = pts[(raw == m).reshape(-1)]
    out.append((((pts[:, None, :] - sites[None, :, :]) ** 2).sum(-1)).min(1).reshape(raw.shape))
  return ids, np.array(out)


def same_bits(a, b):
  a, b = np.asarray(a), np.asarray(b)
  return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(
      np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


# ---- label families ---------------------------------------------------------------------------------------

FAMILIES = ("dense", "seeds", "blocks", "lattice", "few")


def _random_labels(count, dtype, rng):
  """`count` distinct non-zero labels of dtype spread over its whole unsigned range (so that the signed
  dtypes hold negative labels, whose unsigned order differs)."""
  dtype = np.dtype(dtype)
  if dtype == np.bool_:
    return np.ones(min(count, 1), np.bool_)
  u = np.dtype("u%d" % dtype.itemsize)
  top = min(np.iinfo(u).max, (1 << 62))
  vals = np.unique(rng.integers(1, top, size=count * 2, dtype=np.uint64, endpoint=True).astype(u))
  vals = vals[vals != 0]
  rng.shuffle(vals)
  return vals[:count].view(dtype)


def volume(family, shape, dtype, rng):
  """A label volume of `shape` and `dtype`."""
  size = int(np.prod(shape))
  if family == "dense":                       # label-dense noise: many distinct labels in every window
    ids = _random_labels(12, dtype, rng)
    pick = rng.integers(0, len(ids) + 1, size)
    out = np.where(pick < len(ids), ids[np.minimum(pick, len(ids) - 1)], np.zeros(1, ids.dtype))
  elif family == "seeds":                     # sparse seeds on background
    ids = _random_labels(40, dtype, rng)
    out = np.zeros(size, ids.dtype)
    at = rng.random(size) < 0.04
    out[at] = ids[rng.integers(0, len(ids), int(at.sum()))]
  elif family == "blocks":                    # blocks of 4 with some background
    ids = _random_labels(30, dtype, rng)
    coarse = [max(1, (s + 3) // 4) for s in shape]
    c = rng.integers(0, len(ids) + 2, int(np.prod(coarse)))
    c = np.where(c < len(ids), ids[np.minimum(c, len(ids) - 1)], np.zeros(1, ids.dtype)).reshape(coarse)
    for a, s in enumerate(shape):
      c = np.repeat(c, 4, axis=a).take(np.arange(s), axis=a)
    out = c.reshape(-1)
  elif family == "lattice":                   # single voxels on a lattice of spacing 3: equidistant labels
    ids = _random_labels(25, dtype, rng)
    grid = np.zeros(shape, bool)
    grid[tuple(slice(int(rng.integers(0, 3)), None, 3) for _ in shape)] = True
    out = np.zeros(size, ids.dtype)
    g = grid.reshape(-1)
    out[g] = ids[rng.integers(0, len(ids), int(g.sum()))]
  elif family == "few":                       # fewer labels than k
    ids = _random_labels(2, dtype, rng)
    out = np.zeros(size, ids.dtype)
    out[rng.integers(0, size, 3)] = ids[rng.integers(0, len(ids), 3)]
  else:
    raise ValueError(family)
  return out.reshape(shape).astype(dtype, copy=False)
