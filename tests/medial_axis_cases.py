"""The medial axis (edt_b200.medial_axis, edtb200_medial_axis in include/edt_b200.h) restated on the CPU:

  restate   the definition as written: D2 = the CPU oracle's edtsq (oracle/oracle.py, per volume for
            stacks), then (V, q) = parabolic_sites_cases.restate("dilate", D2, ...), then the mark step:
            medial[q(p)] = True for every p with L(p) != 0 (floats by value, so -0.0 is background)
  brute     for integer weights only: q(p) as the lexicographically least (z, y, x) -- the least C-order
            flat index of a C-ordered volume -- among the maximisers of D2(y) - |p - y|^2_w over the whole
            volume, evaluated in int64, with +inf samples maximising before any finite one

`defect` plants one mistake in the mark step so that the tests can show their comparisons notice it:
"background" (the sites of background voxels are marked too) and "greatest" (the greatest instead of the
least tied site, parabolic_sites_cases' "last").

Also the reconstruction (the dilation of D2 on the medial voxels, -inf elsewhere) and the volumes the tests
run on, from morphology_cases.py.
"""
import numpy as np

import morphology_cases as mc
import parabolic_cases as pc
import parabolic_sites_cases as sc

KINDS = mc.KINDS
seeded = mc.seeded
voronoi = mc.voronoi
balls = mc.balls


def _volumes(arr, order, stacked):
  """The volumes of `arr` (one unless stacked) and the axis that indexes them (None: not stacked)."""
  if not stacked:
    return [arr], None
  axis = 0 if order == "C" else arr.ndim - 1
  return [np.take(arr, i, axis=axis) for i in range(arr.shape[axis])], axis


def _per_volume(fn, arr, order, stacked):
  vols, axis = _volumes(arr, order, stacked)
  outs = [fn(np.asfortranarray(v) if order == "F" else np.ascontiguousarray(v)) for v in vols]
  return outs[0] if axis is None else np.stack(outs, axis=axis)


def edtsq(labels, anisotropy=None, black_border=False, order="C", stacked=False):
  """Step 1: the CPU oracle's edtsq, per volume for stacks."""
  from oracle import oracle
  labels = np.asarray(labels)
  vnd = labels.ndim - (1 if stacked else 0)
  w = (1.0,) * vnd if anisotropy is None else tuple(np.atleast_1d(np.asarray(anisotropy, np.float64)))
  return _per_volume(lambda v: oracle.edtsq(v, w if v.ndim > 1 else w[0], black_border), labels, order, stacked)


def mark(labels, indices, order="C", stacked=False, defect=None):
  """Step 3: medial[q(p)] for every p with L(p) != 0 (every p with a site, for the "background" defect)."""
  labels = np.asarray(labels)
  idx = np.asarray(indices).astype(np.int64)
  medial = np.zeros(labels.shape, bool)
  if labels.size == 0:
    return medial
  take = (labels != 0) if defect != "background" else np.ones(labels.shape, bool)
  take &= idx[0] >= 0
  _, axis = _volumes(labels, order, stacked)
  vol_axes = [a for a in range(labels.ndim) if a != axis]
  at = [None] * labels.ndim
  for k, a in enumerate(vol_axes):
    at[a] = idx[k][take]
  if axis is not None:
    at[axis] = np.indices(labels.shape)[axis][take]
  medial[tuple(at)] = True
  return medial


def restate(labels, anisotropy=None, black_border=False, order="C", stacked=False, defect=None, d2=None):
  """(medial, D2, V, indices) by the definition; d2: step 1's result when the caller has it."""
  labels = np.asarray(labels)
  if d2 is None:
    d2 = edtsq(labels, anisotropy, black_border, order, stacked)
  values, idx = sc.restate("dilate", d2, anisotropy, order, defect="last" if defect == "greatest" else None,
                           stacked=stacked)
  return mark(labels, idx, order, stacked, defect), d2, values, idx


def reconstruct(medial, d2, anisotropy=None, order="C", stacked=False):
  """The reverse distance transform: the parabolic dilation of D2 on the medial voxels, -inf elsewhere."""
  return pc.restate("dilate", np.where(medial, d2, -np.inf).astype(np.float32), anisotropy, order, stacked=stacked)


def brute(labels, anisotropy, black_border=False):
  """The medial axis of one C-ordered volume with integer weights, by the lexicographic rule."""
  labels = np.ascontiguousarray(labels)
  d2 = edtsq(labels, anisotropy, black_border)
  w = np.atleast_1d(np.asarray(anisotropy, np.float64))
  assert np.all(w == np.round(w)), "brute force: integer weights only"
  w2 = (w * w).astype(np.int64)
  flat = d2.reshape(-1)
  inf = np.isinf(flat)
  val = np.where(inf, 0, flat).astype(np.int64)
  assert np.all(val < (1 << 24))
  Y = np.indices(labels.shape).reshape(labels.ndim, -1).astype(np.int64)
  medial = np.zeros(flat.size, bool)
  for p in np.flatnonzero(labels.reshape(-1) != 0):
    if inf.any():                               # +inf maximises before every finite value
      medial[np.argmax(inf)] = True
      continue
    cost = sum(w2[a] * (Y[a] - Y[a, p]) ** 2 for a in range(labels.ndim))
    medial[np.argmax(val - cost)] = True        # argmax: the first maximiser, the least flat index
  return medial.reshape(labels.shape)
