"""Local thickness (edt_b200.local_thickness, include/edt_b200.h) restated twice on the CPU:

  threshold   the definition on the CPU oracle's edtsq (oracle/oracle.py), as morphology_cases.threshold
              restates the opening: seeds where (double)D2 > r * r, the edtsq of the mask that is 0 on them
              (no black border), and the largest level whose (double)d2_r <= r * r at a labelled voxel
  brute       seed/voxel pairs enumerated directly: D2 as the least squared distance to another label (and,
              with black_border, to the faces), and p covered at r iff p is labelled and some seed s has
              |p - s|^2_w <= r * r; tiny volumes with integer or dyadic weights, where nothing rounds

`defect` plants one mistake in the threshold restatement, so that the tests can show their comparison
notices it: "lt" (< in place of <=) and "open_border" (the second transform given a black border).
`default_levels` restates the default ladder r_i = (h/2) (2R/h)^(i/n) in float64, h the least float32 weight.
"""
import itertools

import numpy as np

import morphology_cases as mc


def weights(arr, anisotropy):
  return mc._weights(np.asarray(arr), anisotropy)


def least_weight(w):
  """h: the least weight as the C ABI takes it, rounded to float32."""
  return float(min(np.float32(x) for x in w))


def _top(d2, nz):
  """R^2 of one volume: the largest finite D2 over its labelled voxels (None: there is none)."""
  vals = d2[nz & np.isfinite(d2)]
  return float(vals.max()) if vals.size else None


def default_levels(arr, n, anisotropy=None, black_border=False):
  """The n default levels of one volume, descending, in float64."""
  from oracle import oracle
  arr = np.asarray(arr)
  w = weights(arr, anisotropy)
  h = least_weight(w)
  top = _top(oracle.edtsq(arr, w, black_border).astype(np.float64), mc._nonzero(arr))
  R = np.sqrt(top) if top is not None else h / 2
  i = np.arange(n - 1, -1, -1, dtype=np.float64)
  return (h / 2) * np.power(2.0 * R / h, i / n)


def threshold(arr, levels, anisotropy=None, black_border=False, defect=None):
  """The definition at the given levels (any order, repeats allowed) on the CPU oracle."""
  from oracle import oracle
  arr = np.asarray(arr)
  w = weights(arr, anisotropy)
  nz = mc._nonzero(arr)
  d2 = oracle.edtsq(arr, w, black_border).astype(np.float64)
  out = np.zeros(arr.shape, np.float32)
  for r in np.asarray(levels, np.float64).reshape(-1):
    mask = np.where(d2 > r * r, 0, 1).astype(np.uint8)
    mask = np.asfortranarray(mask) if arr.flags.f_contiguous and not arr.flags.c_contiguous else mask
    near = mc._within(oracle.edtsq(mask, w, defect == "open_border"), r, defect)
    out = np.maximum(out, np.where(nz & near, np.float32(r), np.float32(0)))
  return out


def brute(arr, levels, anisotropy=None, black_border=False):
  """Seed/voxel pairs enumerated directly; O(N^2), tiny volumes only."""
  arr = np.asarray(arr)
  w = np.array(weights(arr, anisotropy), np.float64)
  raw = mc._raw(arr + 0 if arr.dtype.kind == "f" else arr).reshape(-1)
  nz = mc._nonzero(arr).reshape(-1)
  pts = np.array(list(itertools.product(*[range(s) for s in arr.shape])), np.float64).reshape(-1, arr.ndim)
  dist2 = (((pts[:, None, :] - pts[None, :, :]) * w) ** 2).sum(-1)           # |p - q|^2_w, all pairs
  other = raw[:, None] != raw[None, :]
  d2 = np.where(other, dist2, np.inf).min(1)
  if black_border:
    shape = np.array(arr.shape, np.float64)
    face = np.minimum(pts + 1, shape - pts) * w                                # the nearest face per axis
    d2 = np.minimum(d2, (face ** 2).min(1))
  d2 = np.where(nz, d2, 0.0)
  out = np.zeros(raw.size, np.float32)
  for r in np.asarray(levels, np.float64).reshape(-1):
    seeds = d2 > r * r
    covered = nz & (np.where(seeds[None, :], dist2, np.inf) <= r * r).any(1)
    out = np.maximum(out, np.where(covered, np.float32(r), np.float32(0)))
  return out.reshape(arr.shape)


# ---- known answers --------------------------------------------------------------------------------------

def run_of_seven():
  """A 1-D run of 7 between background: D2 = 1 4 9 16 9 4 1, R = 4."""
  return np.array([0] + [1] * 7 + [0], np.uint8)


def slab(t, shape=(21, 12)):
  """A slab of thickness t along axis 0, spanning the whole of axis 1 (no faces there without black_border)."""
  out = np.zeros(shape, np.uint16)
  lo = (shape[0] - t) // 2
  out[lo:lo + t] = 7
  return out


def rod_between_balls(shape=(17, 45), radius=6, rod=3):
  """Two discs of `radius` joined along axis 1 by a straight rod `rod` voxels thick; returns the labels and
  the voxel in the middle of the rod."""
  out = np.zeros(shape, np.int32)
  yy, xx = np.meshgrid(np.arange(shape[0]), np.arange(shape[1]), indexing="ij")
  cy = shape[0] // 2
  for cx in (radius + 1, shape[1] - radius - 2):
    out[(yy - cy) ** 2 + (xx - cx) ** 2 <= radius * radius] = 3
  out[cy - rod // 2:cy + rod // 2 + 1, radius + 1:shape[1] - radius - 2] = 3
  return out, (cy, shape[1] // 2)


def thin_line(shape=(9, 15)):
  """A line one voxel thick along axis 1, with background on both sides and at both ends."""
  out = np.zeros(shape, np.uint8)
  out[shape[0] // 2, 2:-2] = 1
  return out


DEFECTS = ("lt", "open_border")
