"""The surface distances and the metrics formed from them, restated on numpy / scipy from their
definitions (include/edt_b200.h, edt_b200.surface_distances):

  S_v(k)     mask ^ binary_erosion(mask) for mask = (v == k), scipy's cross structure, border_value 0
  d_v,k(q)   distance_transform_edt of the complement of S_v(k) with `sampling`, cast to float32;
             +inf everywhere when S_v(k) is empty
  A->B (k)   d_b,k at the voxels of S_a(k); B->A the other way round

Metrics are formed in float64 from the float32 distances, with np.percentile's linear rule.  Both
surfaces empty gives NaN for every metric; one empty gives +inf for the distances and 0 for surface
Dice.  Also used by tools/surface_bench.py as the CPU baseline.
"""
import numpy as np
from scipy import ndimage


def surface(vol, key):
  mask = np.asarray(vol) == key
  if mask.ndim == 0 or not mask.any():
    return np.zeros(mask.shape, bool)
  return mask ^ ndimage.binary_erosion(mask, border_value=0)


def distance_to(surf, anisotropy):
  """float32 distance of every voxel to the nearest voxel of `surf`, +inf when it is empty."""
  if not surf.any():
    return np.full(surf.shape, np.inf, np.float32)
  return ndimage.distance_transform_edt(~surf, sampling=anisotropy).astype(np.float32)


def default_keys(a, b):
  keys = np.union1d(np.unique(a), np.unique(b))
  return keys[keys != 0]


def segments(a, b, keys, anisotropy):
  """[(A->B, B->A) per key] of one volume pair, each a sorted float32 array."""
  out = []
  for k in keys:
    sa, sb = surface(a, k), surface(b, k)
    ab = np.sort(distance_to(sb, anisotropy)[sa]) if sa.any() else np.zeros(0, np.float32)
    ba = np.sort(distance_to(sa, anisotropy)[sb]) if sb.any() else np.zeros(0, np.float32)
    out.append((ab, ba))
  return out


def _rule(ab, ba, one_empty):
  if ab.size == 0 and ba.size == 0:
    return np.nan
  if ab.size == 0 or ba.size == 0:
    return one_empty
  return None


def hausdorff(ab, ba, percentile=None, directed=False):
  r = _rule(ab, ba, np.inf)
  if r is not None:
    return r

  def one(x):
    x = x.astype(np.float64)
    return x.max() if percentile is None else np.percentile(x, percentile, method="linear")
  return one(ab) if directed else max(one(ab), one(ba))


def average(ab, ba, symmetric=False):
  r = _rule(ab, ba, np.inf)
  if r is not None:
    return r
  x = np.concatenate([ab, ba]) if symmetric else ab
  return x.astype(np.float64).mean()


def dice(ab, ba, tolerance):
  r = _rule(ab, ba, 0.0)
  if r is not None:
    return r
  within = (ab.astype(np.float64) <= tolerance).sum() + (ba.astype(np.float64) <= tolerance).sum()
  return within / float(ab.size + ba.size)


def metric(a, b, keys, anisotropy, fn, **kw):
  """fn over the segments of every key of one volume pair: float64 (K,)."""
  return np.array([fn(ab, ba, **kw) for ab, ba in segments(a, b, keys, anisotropy)], np.float64)


def random_pair(rng, shape, nlabels=4, dtype=np.uint16, flips=0.05):
  """A blocky label volume with background, and a copy with a fraction of its voxels relabelled."""
  coarse = tuple(max(1, s // 4) for s in shape)
  small = rng.integers(0, nlabels + 1, coarse)
  a = small
  for ax, s in enumerate(shape):
    a = np.repeat(a, -(-s // coarse[ax]), axis=ax)
  a = a[tuple(slice(0, s) for s in shape)]
  b = a.copy()
  flip = rng.random(shape) < flips
  b[flip] = rng.integers(0, nlabels + 1, int(flip.sum()))
  return a.astype(dtype), b.astype(dtype)
