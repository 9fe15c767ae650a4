"""Numpy restatement of the feature transform's site contract (edtb200_feature_transform).

A site of voxel p is a position q whose label differs from p's, or with black_border a face
position (one coordinate -1 or n on its axis, the others inside the volume).  Unsigned background
maps to itself; with signed=True background is an ordinary label.  "Nearest" is measured in the
transform's own arithmetic:

    value(p, q) = fl32( w2z (pz-qz)^2 + fl32( w2y (py-qy)^2 + T[|px-qx|] ) )

T[k] = (k sequential float32 adds of wx)^2 in float32, w2 = fl32(w * w), and each fl32(...) a
double-precision sum rounded once to float32; x is the memory-fastest axis.  The returned site
must make value(p, site(p)) equal the transform's squared distance bit for bit.

Arrays here are indexed in ARRAY axis order and `anisotropy` is per array axis, as the public
functions take them; `order` ("C" or "F", by default the labels' own: memory_order) says which
array axis is x.
"""
import numpy as np


def step_table(w, n):
  """T[0..n] for weight w."""
  t = np.zeros(n + 1, np.float32)
  a, w = np.float32(0), np.float32(w)
  for k in range(1, n + 1):
    a = np.float32(a + w)
    t[k] = np.float32(a * a)
  return t


def memory_order(a):
  """"F" when x is array axis 0, as the front door decides it (an F-contiguous array, which
  includes arrays that are both), else "C"."""
  return "F" if np.asarray(a).flags.f_contiguous else "C"


def xyz_axes(nd, order):
  """Array axes of x, y, z (the first nd of them)."""
  return list(range(nd)) if order == "F" else list(reversed(range(nd)))


def _fl32(x):
  return np.asarray(x, np.float64).astype(np.float32)


def values(p, q, shape, anisotropy, order, xp=np):
  """value(p, q) for coordinate arrays p[k], q[k] (array axis k), broadcast together."""
  nd = len(shape)
  axes = xyz_axes(nd, order)
  ax = axes[0]
  table = step_table(anisotropy[ax], shape[ax] + 1)
  dx = abs(q[ax] - p[ax])
  if xp is np:
    v = table[dx]
  else:
    v = xp.as_tensor(table, device=dx.device)[dx]
  for ax in axes[1:]:
    w2 = float(np.float32(np.float32(anisotropy[ax]) * np.float32(anisotropy[ax])))
    d = q[ax] - p[ax]
    if xp is np:
      v = _fl32(w2 * (d.astype(np.float64) ** 2) + v.astype(np.float64))
    else:
      v = (w2 * d.to(xp.float64) ** 2 + v.to(xp.float64)).to(xp.float32)
  return v


def no_site(sites, black_border):
  """Where the site is "none": every coordinate -1, which is a face position only with black_border
  (in 1-D)."""
  none = (np.asarray(sites) == -1).all(axis=0)
  return none & (not black_border)


def site_value(labels, sites, anisotropy, black_border, order=None):
  """value(p, site(p)) for every voxel; sites is (nd,) + shape in scipy's layout.  Where there is
  no site the value is meaningless."""
  shape = labels.shape
  order = order or memory_order(labels)
  p = np.indices(shape)
  sites = np.asarray(sites).astype(np.int64)
  q = np.where(no_site(sites, black_border), p, sites)     # any in-range stand-in
  return values(p, q, shape, anisotropy, order)


def check_sites(labels, sites, sqdist, anisotropy, black_border, signed, order=None):
  """Assert the site contract.  sqdist: the squared distances (|sdfsq| for signed)."""
  labels = np.asarray(labels)
  order = order or memory_order(labels)
  shape = labels.shape
  nd = labels.ndim
  sites = np.asarray(sites).astype(np.int64)
  sqdist = np.asarray(sqdist, np.float32)
  assert sites.shape == (nd,) + shape, (sites.shape, shape)
  none = no_site(sites, black_border)
  inf = ~np.isfinite(sqdist)
  assert np.array_equal(none, inf), "'none' sites %d, infinite distances %d" % (none.sum(), inf.sum())
  p = np.indices(shape)
  bg = labels == 0
  if not signed:
    self_ = (sites == p).all(axis=0)
    assert self_[bg].all(), "unsigned background not mapped to itself"
  live = ~none & ~(bg if not signed else np.zeros_like(bg))
  lo = sites < 0
  hi = sites >= np.array(shape).reshape((nd,) + (1,) * nd)
  out_axes = (lo | hi).sum(axis=0)
  face = live & (out_axes > 0)
  if face.any():
    assert black_border, "face site without black_border at %s" % (tuple(np.argwhere(face)[0]),)
    assert (out_axes[face] == 1).all(), "face site outside on more than one axis"
    at_face = (sites == -1) | (sites == np.array(shape).reshape((nd,) + (1,) * nd))
    assert ((lo | hi) <= at_face)[:, face].all(), "face site beyond the face"
  inside = live & (out_axes == 0)
  q = np.where(inside, sites, p)
  assert (labels[tuple(q)][inside] != labels[inside]).all(), "site of the voxel's own label at %s" % (
    tuple(np.argwhere(inside & (labels[tuple(q)] == labels))[0]),)
  got = site_value(labels, sites, anisotropy, black_border, order)
  bad = live & (got.view(np.uint32) != sqdist.view(np.uint32))
  assert not bad.any(), "site value differs from the distance at %s: %r vs %r (%d voxels)" % (
    tuple(np.argwhere(bad)[0]), float(got[bad][0]), float(sqdist[bad][0]), int(bad.sum()))


def skimage_expand(labels, distance, spacing):
  """skimage.segmentation.expand_labels restated on scipy: (result, scipy's nearest sites)."""
  from scipy import ndimage as ndi
  d, idx = ndi.distance_transform_edt(labels == 0, return_indices=True, sampling=spacing)
  out = np.zeros_like(labels)
  mask = d <= distance
  out[mask] = labels[tuple(i[mask] for i in idx)]
  return out, idx


def check_expand(labels, got, sites, want, want_sites, distance, spacing):
  """Assert an expand_labels result `got`, grown from `sites` (feature_transform(signed=True)),
  against skimage's `want` grown from scipy's `want_sites`.  For spacings whose squared distances
  are exact in float32 (integers below 2^24): labelled voxels keep their label; a background voxel
  takes its own site's label exactly when that site is within `distance`, and is 0 otherwise; and
  where `got` and `want` differ, both grew (or both did not) from two different sites at the same
  exact distance -- a tie."""
  labels, got, sites = np.asarray(labels), np.asarray(got), np.asarray(sites).astype(np.int64)
  shape, nd = labels.shape, labels.ndim
  p = np.indices(shape)
  w = np.array(spacing, np.float64).reshape((nd,) + (1,) * nd)

  def exact(s):
    return ((w * (s - p)) ** 2).sum(0)

  bg = labels == 0
  assert np.array_equal(got[~bg], labels[~bg]), "labelled voxels changed"
  has = (sites >= 0).all(0) & (sites < np.array(shape).reshape((nd,) + (1,) * nd)).all(0)
  q = np.where(has, sites, p)
  grow = bg & has & (exact(q) <= float(distance) ** 2)
  assert np.array_equal(got[grow], labels[tuple(q)][grow]), "a grown voxel does not carry its site's label"
  assert (got[bg & ~grow] == 0).all(), "background grew where its site is beyond `distance`"
  diff = got != want
  assert ((got != 0) == (want != 0))[diff].all(), "grew where skimage did not, or the reverse"
  assert (sites != want_sites).any(0)[diff].all(), "same site, different result"
  assert np.array_equal(exact(q)[diff], exact(np.asarray(want_sites))[diff]), "differs from skimage but not at a tie"


def candidates(shape, black_border):
  """Every in-volume position and (with black_border) every face position: (nd, m) int64."""
  nd = len(shape)
  cand = [np.indices(shape).reshape(nd, -1)]
  if black_border:
    for ax in range(nd):
      other = [s for k, s in enumerate(shape) if k != ax]
      grid = np.indices(other).reshape(nd - 1, -1) if other else np.zeros((0, 1), np.int64)
      for face in (-1, shape[ax]):
        rows = list(grid)
        rows.insert(ax, np.full(grid.shape[1], face))
        cand.append(np.array(rows, np.int64).reshape(nd, -1))
  return np.concatenate(cand, axis=1).astype(np.int64)


def brute_sites(labels, anisotropy, black_border, signed, order=None):
  """(squared distances, sites) by trying every admissible site; volumes of up to about 6^3."""
  labels = np.asarray(labels)
  order = order or memory_order(labels)
  shape = labels.shape
  nd = labels.ndim
  cand = candidates(shape, black_border)
  inside = ((cand >= 0) & (cand < np.array(shape).reshape(nd, 1))).all(axis=0)
  clab = np.zeros(cand.shape[1], labels.dtype)
  clab[inside] = labels[tuple(cand[:, inside])]
  flat = labels.reshape(-1)
  pts = np.indices(shape).reshape(nd, -1)
  dist = np.empty(flat.size, np.float32)
  sites = np.empty((nd, flat.size), np.int64)
  for i in range(flat.size):
    p = pts[:, i]
    if flat[i] == 0 and not signed:
      dist[i], sites[:, i] = 0.0, p
      continue
    ok = ~inside | (clab != flat[i])
    if not ok.any():
      dist[i], sites[:, i] = np.inf, -1
      continue
    v = values(p.reshape(nd, 1), cand[:, ok], shape, anisotropy, order)
    j = int(np.argmin(v))
    dist[i], sites[:, i] = v[j], cand[:, ok][:, j]
  return dist.reshape(shape), sites.reshape((nd,) + shape)
