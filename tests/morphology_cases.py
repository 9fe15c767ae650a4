"""The spherical morphology (edt_b200.spherical_erode / _open / _dilate / _close, include/edt_b200.h) restated
twice on the CPU:

  threshold   the definitions, on the CPU oracle's edtsq / sdfsq (oracle/oracle.py): a voxel is "within r"
              when (double)d2 <= r * r for the float32 squared distance d2 the transform computes
  per_label   scipy.ndimage's binary_erosion / binary_dilation per label, with the ball
              B = {v : sum_j (w_j v_j)^2 <= r^2} built in float64

The two agree wherever the arithmetic is exact (integer and dyadic weights); the library must equal the
threshold restatement bit for bit everywhere.  `defect` plants one mistake in either restatement, so that
the tests can show their comparison notices it: "lt" (< in place of <=), "border" (black_border mapped the
wrong way) and "open_border" (opening's second transform given a black border).

Also seeded volumes: Voronoi cells, balls, 1-voxel bridges and specks, several labels touching.
"""
import numpy as np
from scipy import ndimage

OPS = ("erode", "open", "dilate", "close")


def _weights(arr, anisotropy):
  if anisotropy is None:
    return (1.0,) * arr.ndim
  if np.ndim(anisotropy) == 0:
    return (float(anisotropy),)
  return tuple(float(a) for a in anisotropy)


def _raw(arr):
  """The labels' bits as unsigned integers (bool as uint8)."""
  return arr.view(np.uint8) if arr.dtype == np.bool_ else arr.view(np.dtype("u%d" % arr.itemsize))


def _keep(arr, keep):
  """arr where keep, all-zero bits elsewhere; every kept value keeps its bits."""
  raw = _raw(arr)
  return np.where(keep, raw, raw.dtype.type(0)).view(arr.dtype)


def _nonzero(arr):
  return arr != 0                            # floats by value: -0.0 is zero, NaN is not


def _within(d2, r, defect):
  d2 = np.abs(d2).astype(np.float64)
  return d2 < r * r if defect == "lt" else d2 <= r * r


def threshold(op, arr, r, anisotropy=None, black_border=False, defect=None):
  """The definitions on the CPU oracle's transforms."""
  from oracle import oracle
  arr = np.asarray(arr)
  w = _weights(arr, anisotropy)
  bb = bool(black_border) != (defect == "border")
  nz = _nonzero(arr)
  if op in ("erode", "open"):
    keep = nz & ~_within(oracle.edtsq(arr, w, bb), r, defect)
    if op == "open":
      mask = np.where(keep, 0, 1).astype(np.uint8)           # 0 on the erosion E: its edtsq is d2(p, E)
      keep = nz & _within(oracle.edtsq(mask, w, defect == "open_border"), r, defect)
    return _keep(arr, keep)
  dil = nz | _within(oracle.sdfsq(arr, w), r, defect)
  if op == "dilate":
    return dil
  return dil & ~_within(oracle.edtsq(dil.astype(np.uint8), w, bb), r, defect)


def ball(r, w, strict=False):
  """B as a boolean structuring element, centred, in float64 (strict: < r^2, a planted defect)."""
  ext = [int(np.floor(r / wj)) + 1 for wj in w]
  grids = np.meshgrid(*[np.arange(-e, e + 1, dtype=np.float64) for e in ext], indexing="ij")
  d2 = sum((wj * g) ** 2 for wj, g in zip(w, grids))
  return d2 < r * r if strict else d2 <= r * r


def per_label(op, arr, r, anisotropy=None, black_border=False, defect=None):
  """scipy.ndimage per label: erosion with border_value 0 / 1 for black_border / not, opening as the
  dilation of each label's erosion with border_value 0, dilation and closing of the foreground."""
  arr = np.asarray(arr)
  w = _weights(arr, anisotropy)
  B = ball(r, w, strict=defect == "lt")
  bv = 0 if bool(black_border) != (defect == "border") else 1
  nz = _nonzero(arr)
  if op in ("erode", "open"):
    lab = _raw(arr + 0 if arr.dtype.kind == "f" else arr)  # -0.0 folded onto +0.0
    keep = np.zeros(arr.shape, bool)
    for k in np.unique(lab[nz]):
      e = ndimage.binary_erosion(lab == k, B, border_value=bv)
      if op == "open":
        e = ndimage.binary_dilation(e, B, border_value=1 if defect == "open_border" else 0)
      keep |= e
    return _keep(arr, keep)
  dil = ndimage.binary_dilation(nz, B, border_value=0)
  if op == "dilate":
    return dil
  return ndimage.binary_erosion(dil, B, border_value=bv)


# ---- volumes -------------------------------------------------------------------------------------------

def voronoi(rng, shape, cells, dtype=np.uint32):
  """Every voxel labelled 1..cells by its nearest seed."""
  from scipy.spatial import cKDTree
  pts = rng.uniform(0, 1, (cells, len(shape))) * np.array(shape)
  grid = np.stack(np.meshgrid(*[np.arange(s, dtype=np.float64) for s in shape], indexing="ij"), -1)
  return (cKDTree(pts).query(grid.reshape(-1, len(shape)))[1] + 1).astype(dtype).reshape(shape)


def balls(rng, shape, count, rmax, dtype=np.uint8, labels=None):
  """Background with `count` balls of radius up to rmax, labelled 1.. (or from `labels`); later ones win."""
  out = np.zeros(shape, dtype)
  grids = np.meshgrid(*[np.arange(s, dtype=np.float64) for s in shape], indexing="ij")
  for i in range(count):
    c = rng.uniform(0, 1, len(shape)) * np.array(shape)
    rad = rng.uniform(1.0, rmax)
    inside = sum((g - cj) ** 2 for g, cj in zip(grids, c)) <= rad * rad
    out[inside] = labels[i % len(labels)] if labels is not None else (i % 250) + 1
  return out


def bridges(shape, dtype=np.uint16):
  """Two blocks of label 1 joined by a 1-voxel bridge, a block of label 2 touching one of them, and
  single-voxel specks of 1 and 3 in the background."""
  out = np.zeros(shape, dtype)
  n0 = shape[0]
  rest = tuple(slice(1, max(2, s - 1)) for s in shape[1:])
  out[(slice(1, n0 // 3),) + rest] = 1
  out[(slice(2 * n0 // 3, n0 - 1),) + rest] = 1
  mid = tuple(s // 2 for s in shape[1:])
  out[(slice(n0 // 3, 2 * n0 // 3),) + mid] = 1
  if len(shape) > 1:
    out[(slice(1, n0 // 3), slice(shape[1] - 1, shape[1])) + rest[1:]] = 2
  out[(n0 // 2,) + tuple(0 for _ in shape[1:])] = 3
  out[(n0 // 2,) + tuple(s - 1 for s in shape[1:])] = 1
  return out


def touching(rng, shape, dtype=np.int32):
  """Blocks of several labels that touch each other, with a little background."""
  blocks = [max(1, s // 3) for s in shape]
  small = rng.integers(1, 6, [-(-s // b) for s, b in zip(shape, blocks)])
  out = small
  for axis, b in enumerate(blocks):
    out = np.repeat(out, b, axis=axis)
  out = out[tuple(slice(0, s) for s in shape)].astype(dtype)
  out[rng.random(shape) < 0.03] = 0
  return out


def seeded(rng, kind, shape, dtype):
  if kind == "voronoi":
    return voronoi(rng, shape, 6, dtype)
  if kind == "balls":
    return balls(rng, shape, 5, max(2.0, min(shape) / 3), dtype)
  if kind == "bridges":
    return bridges(shape, dtype)
  return touching(rng, shape, dtype)


KINDS = ("voronoi", "balls", "bridges", "touching")
