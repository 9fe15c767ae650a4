"""The per-label views (edtb200_label_stats / edtb200_label_extract, include/edt_b200.h; edt_b200.label_stats_cuda,
each_cuda, each) restated in plain numpy, from the header's words and not from the kernels:

  stats     per distinct non-zero key (the label's raw bits, zero-extended to 64 bits): voxel count, the largest
            distance under the IEEE total order (finite values, +-inf, -0.0 < +0.0; no NaN), the smallest
            x-fastest linear index where it is attained, and the inclusive box x0 y0 z0 x1 y1 z1; keys ascending
            as unsigned integers.  Arrays are C-ordered: the last axis is x, missing axes have extent 1.
  extract   out = (labels == key) ? dt : 0 inside the box, or zeros with `erase`; nothing outside it.
  slot_hash the table's hash (csrc/edt_each.cuh, hash_label) in numpy uint64 arithmetic, and colliding_keys, which
            searches for keys that share one home slot so that tests can build probe chains of a known shape.

`defect` plants one mistake in `stats`, so that the tests can show their volumes are able to notice it:
"last_tie" (argmax takes the last index of a tie), "exclusive_box" (high corner one past the end),
"unsigned_max" (floats ordered by their unsigned bits) and "sign_extend" (signed labels sign-extended).

Also seeded label volumes (many Voronoi cells, key noise, stripes, singletons), distance images that are not
transforms (negative, infinite, plateaus), and case_volumes, the small volumes both the CPU and the GPU tests walk.
"""
import numpy as np

DEFECTS = ("last_tie", "exclusive_box", "unsigned_max", "sign_extend")
FIELDS = ("keys", "count", "max", "argmax", "box")


def raw(arr):
  """The labels' bits as unsigned integers of their own width (bool as uint8)."""
  arr = np.asarray(arr)
  return arr.view(np.uint8) if arr.dtype == np.bool_ else arr.view(np.dtype("u%d" % arr.itemsize))


def keys_of(arr, defect=None):
  """Every voxel's table key: raw bits zero-extended to uint64."""
  arr = np.asarray(arr)
  if defect == "sign_extend" and arr.dtype.kind == "i":
    return arr.astype(np.int64).view(np.uint64)
  return raw(arr).astype(np.uint64)


def dims_of(shape):
  """(sx, sy, sz) of a C-ordered array of `shape` (1-D to 3-D)."""
  return tuple(int(s) for s in shape)[::-1] + (1,) * (3 - len(shape))


def _rank(dt, defect=None):
  """float32 -> int64 whose order is the IEEE total order (negatives mirrored below zero)."""
  bits = np.ascontiguousarray(dt, dtype=np.float32).view(np.uint32).astype(np.int64)
  if defect == "unsigned_max":
    return bits
  return np.where(bits >= 1 << 31, (1 << 31) - 1 - bits, bits)


def stats(labels, dt, defect=None):
  """dict of keys (uint64), count, argmax (int64), max (float32) and box (n x 6 int64), one row per key."""
  labels = np.ascontiguousarray(labels)
  dt = np.ascontiguousarray(dt, dtype=np.float32)
  assert labels.shape == dt.shape and 1 <= labels.ndim <= 3
  sx, sy, sz = dims_of(labels.shape)
  key = keys_of(labels, defect).ravel()
  idx = np.flatnonzero(key)
  order = idx[np.argsort(key[idx], kind="stable")]               # by key, then by linear index
  k = key[order]
  start = np.flatnonzero(np.concatenate([[True], k[1:] != k[:-1]])) if k.size else np.zeros(0, np.int64)
  count = np.diff(np.concatenate([start, [k.size]]))
  flat = dt.ravel()[order]
  rank = _rank(flat, defect)
  if k.size:
    top = np.maximum.reduceat(rank, start)
    at_top = rank == np.repeat(top, count)
    if defect == "last_tie":
      argmax = np.maximum.reduceat(np.where(at_top, order, -1), start)
    else:
      argmax = np.minimum.reduceat(np.where(at_top, order, np.iinfo(np.int64).max), start)
    x, y, z = order % sx, order // sx % sy, order // (sx * sy)
    lo = [np.minimum.reduceat(c, start) for c in (x, y, z)]
    hi = [np.maximum.reduceat(c, start) + (defect == "exclusive_box") for c in (x, y, z)]
    box = np.stack(lo + hi, axis=1).astype(np.int64)
  else:
    argmax, box = np.zeros(0, np.int64), np.zeros((0, 6), np.int64)
  return {"keys": k[start] if k.size else k, "count": count.astype(np.int64), "max": dt.ravel()[argmax],
          "argmax": argmax.astype(np.int64), "box": box}


def table_stats(table):
  """The filled slots of a table edtb200_label_stats wrote (a dict of its five arrays), in the form `stats`
  returns."""
  keys, count, mx, argmax, box = (np.asarray(table[f]) for f in FIELDS)
  keys = keys.view(np.uint64)
  sel = np.flatnonzero(keys)
  sel = sel[np.argsort(keys[sel], kind="stable")]
  return {"keys": keys[sel], "count": np.asarray(count).view(np.int64)[sel],
          "max": np.asarray(mx).view(np.float32)[sel], "argmax": np.asarray(argmax).view(np.int64)[sel],
          "box": np.asarray(box).reshape(-1, 6)[sel].astype(np.int64)}


def mismatch(got, want):
  """Names of the fields in which two results of `stats` differ (max compared by bits); [] when equal."""
  if not np.array_equal(got["keys"], want["keys"]):
    return ["keys"]
  bad = []
  for f in FIELDS[1:]:
    a, b = np.asarray(got[f]), np.asarray(want[f])
    if f == "max":
      a, b = a.astype(np.float32).view(np.uint32), b.astype(np.float32).view(np.uint32)
    if a.shape != b.shape or not np.array_equal(a, b):
      bad.append(f)
  return bad


def extract(labels, dt, key, box=None, erase=False, out=None):
  """A copy of `out` (zeros when None) with the box overwritten as edtb200_label_extract does."""
  labels = np.ascontiguousarray(labels)
  dt = np.ascontiguousarray(dt, dtype=np.float32)
  sx, sy, sz = dims_of(labels.shape)
  res = np.zeros(labels.shape, np.float32) if out is None else np.array(out, dtype=np.float32, order="C")
  if box is None:
    box = (0, 0, 0, sx - 1, sy - 1, sz - 1)
  x0, y0, z0, x1, y1, z1 = (int(b) for b in box)
  sl = (slice(z0, z1 + 1), slice(y0, y1 + 1), slice(x0, x1 + 1))
  k3, d3, r3 = keys_of(labels).reshape(sz, sy, sx), dt.reshape(sz, sy, sx), res.reshape(sz, sy, sx)
  r3[sl] = 0 if erase else np.where(k3[sl] == np.uint64(key), d3[sl], np.float32(0))
  return res


# ---- the table's hash ------------------------------------------------------------------------

def slot_hash(key):
  """hash_label of csrc/edt_each.cuh for one key or an array of keys: uint32."""
  k = np.atleast_1d(np.asarray(key, dtype=np.uint64)).copy()
  k ^= k >> np.uint64(33)
  k *= np.uint64(0xff51afd7ed558ccd)
  k ^= k >> np.uint64(33)
  k *= np.uint64(0xc4ceb9fe1a85ec53)
  k ^= k >> np.uint64(33)
  return (k & np.uint64(0xffffffff)).astype(np.uint32)


def home_slot(key, capacity):
  return (slot_hash(key) & np.uint32(capacity - 1)).astype(np.int64)


def colliding_keys(n, capacity, home, nbytes, seed=0):
  """`n` distinct non-zero keys of `nbytes` bytes whose home slot in a table of `capacity` is `home`."""
  rng = np.random.default_rng(seed)
  if nbytes <= 2:
    pool = np.arange(1, 1 << (8 * nbytes), dtype=np.uint64)
  else:
    pool = np.unique(rng.integers(1, (1 << (8 * nbytes)) - 1, 64 * n * capacity, dtype=np.uint64, endpoint=True))
  hit = pool[home_slot(pool, capacity) == home]
  if hit.size < n:
    raise ValueError("only %d keys of %d bytes have home slot %d of %d" % (hit.size, nbytes, home, capacity))
  return np.sort(rng.choice(hit, n, replace=False))


def random_keys(n, nbytes, seed, signed=False):
  """`n` distinct non-zero keys of `nbytes` bytes; with `signed`, half of them have the top bit set."""
  rng = np.random.default_rng(seed)
  top = (1 << (8 * nbytes)) - 1
  if nbytes <= 2:
    return np.sort(rng.choice(np.arange(1, top + 1, dtype=np.uint64), n, replace=False))
  keys = np.zeros(0, np.uint64)
  while keys.size < n:
    keys = np.unique(np.concatenate([keys, rng.integers(1, top, 2 * n, dtype=np.uint64, endpoint=True)]))
  keys = rng.choice(keys, n, replace=False)
  if signed:
    keys[::2] |= np.uint64(1 << (8 * nbytes - 1))
    keys = np.unique(keys)
  return np.sort(keys)


def as_labels(keys, dtype):
  """uint64 keys -> labels of `dtype` with those raw bits (bool: any non-zero key is True)."""
  dtype = np.dtype(dtype)
  if dtype == np.bool_:
    return np.asarray(keys) != 0
  return np.asarray(keys, dtype=np.uint64).astype(np.dtype("u%d" % dtype.itemsize)).view(dtype)


# ---- label volumes ---------------------------------------------------------------------------

def voronoi_many(shape, nlabels, seed, dtype, key_pool=None, background=0.1):
  """`nlabels` Voronoi cells with keys from `key_pool` (random distinct keys of the dtype when None), a
  fraction `background` of the voxels cleared; every label keeps at least its seed voxel."""
  from scipy.spatial import cKDTree
  rng = np.random.default_rng(seed)
  total = int(np.prod(shape))
  seeds = rng.choice(total, nlabels, replace=False)
  pts = np.stack(np.unravel_index(seeds, shape), axis=1)
  grid = np.stack(np.unravel_index(np.arange(total), shape), axis=1)
  cell = cKDTree(pts).query(grid)[1]
  pool = random_keys(nlabels, np.dtype(dtype).itemsize, seed + 1) if key_pool is None else np.asarray(key_pool, np.uint64)
  assert pool.size >= nlabels
  key = rng.permutation(pool)[:nlabels][cell]
  clear = rng.uniform(size=total) < background
  clear[seeds] = False
  key[clear] = 0
  return as_labels(key, dtype).reshape(shape)


def noise(shape, keys, seed, dtype, background=0.0):
  """Every voxel an independent draw from `keys`; each key appears at least once (when the volume has room)."""
  rng = np.random.default_rng(seed)
  keys = np.asarray(keys, np.uint64)
  total = int(np.prod(shape))
  key = keys[rng.integers(0, keys.size, total)]
  key[rng.uniform(size=total) < background] = 0
  where = rng.permutation(total)[:keys.size]
  key[where] = keys[:where.size]
  return as_labels(key, dtype).reshape(shape)


def stripes(shape, run, nlabels, dtype=np.uint16):
  """Label 1 + (linear index // run) % nlabels: with run = 1 and 32 labels every warp of the kernel (32
  consecutive voxels) holds 32 distinct labels, with run = 16 two, with run a multiple of 32 one."""
  lin = np.arange(int(np.prod(shape)), dtype=np.int64)
  return (1 + lin // run % nlabels).astype(dtype).reshape(shape)


def singletons(shape, keys, seed, dtype, background=0.0):
  """Every foreground voxel its own key (needs at least as many keys as voxels)."""
  rng = np.random.default_rng(seed)
  total = int(np.prod(shape))
  key = rng.permutation(np.asarray(keys, np.uint64))[:total].copy()
  assert key.size == total
  key[rng.uniform(size=total) < background] = 0
  return as_labels(key, dtype).reshape(shape)


# ---- distance images that no transform would produce ---------------------------------------------

DT_KINDS = ("ties", "negative", "signed", "inf", "plateau")


def distances(labels, kind, seed=0):
  """float32 image for `labels`:
  ties      multiples of 1/4 in [0, 4): every label's maximum is attained many times
  negative  the same, minus 5: every maximum is negative (and -0.25 steps apart)
  signed    ties - 2, and the label with the smallest key entirely below zero
  inf       by rank of the key mod 3: all +inf / finite with some +inf / all -inf
  plateau   1/2 everywhere and 2 on the last slice of the first axis; the label with the smallest key is 2
            everywhere, so every other label's first maximum lies in the last slice"""
  rng = np.random.default_rng(seed)
  labels = np.asarray(labels)
  key = keys_of(labels)
  uniq = np.unique(key[key != 0])
  ties = (rng.integers(0, 16, labels.shape) / 4.0).astype(np.float32)
  if kind == "ties":
    return ties
  if kind == "negative":
    return ties - np.float32(5)
  if kind == "signed":
    d = ties - np.float32(2)
    if uniq.size:
      d[key == uniq[0]] = -np.abs(d[key == uniq[0]]) - np.float32(0.25)
    return d
  if kind == "inf":
    rank = np.searchsorted(uniq, key) % 3
    d = ties.copy()
    d[rank == 0] = np.inf
    d[(rank == 1) & (rng.uniform(size=labels.shape) < 0.3)] = np.inf
    d[rank == 2] = -np.inf
    return d
  if kind == "plateau":
    d = np.full(labels.shape, 0.5, np.float32)
    d[-1] = 2.0
    if uniq.size:
      d[key == uniq[0]] = 2.0
    return d
  raise ValueError(kind)


# ---- the volumes both the CPU and the GPU tests walk: name -> (labels, dt kind) ---------------------------

def _bg(lab, frac, seed):
  lab = lab.copy()
  lab[np.random.default_rng(seed).uniform(size=lab.shape) < frac] = 0
  return lab


def case_volumes():
  """Yields (name, labels, dt): every shape of the list with every dt kind once, signed and bool labels,
  background fractions 0, 0.1, 0.97, warps of 1, 2 and 32 labels, and a last voxel alone in its warp."""
  shapes = [(1,), (31,), (33,), (7, 5), (3, 5, 7), (2, 3, 1025), (65, 1, 1), (1, 1, 40), (40, 72, 65)]
  dtypes = [np.uint8, np.int8, np.int16, np.int32, np.int64, np.uint16, np.uint32, np.uint64, np.int8]
  for i, (shape, dtype) in enumerate(zip(shapes, dtypes)):
    total = int(np.prod(shape))
    nbytes = np.dtype(dtype).itemsize
    n = max(1, min(total // 3, 200, (1 << (8 * nbytes)) - 1))
    pool = random_keys(n, nbytes, 40 + i, signed=np.dtype(dtype).kind == "i")
    lab = voronoi_many(shape, min(n, pool.size), 50 + i, dtype, pool, background=(0.0, 0.1, 0.97)[i % 3])
    for j, kind in enumerate(DT_KINDS if total > 40 else DT_KINDS[i % 5:][:2]):
      yield "%s-%s-%s" % ("x".join(map(str, shape)), np.dtype(dtype).name, kind), lab, distances(lab, kind, 60 + i + j)
  for run, n in ((1, 32), (16, 64), (64, 5), (1, 1)):
    lab = stripes((6, 10, 64), run, n)
    for kind in ("ties", "plateau"):
      yield "stripes-run%d-n%d-%s" % (run, n, kind), lab, distances(lab, kind, 70 + run)
  yield "bool", _bg(np.ones((5, 9, 33), np.bool_), 0.4, 80), distances(np.ones((5, 9, 33), np.bool_), "signed", 81)
  last = np.zeros((3, 11, 43), np.int16)                         # 1419 voxels: the last one alone in its warp
  last[-1, -1, -1] = -7
  last[0, 0, :5] = 9
  yield "last-voxel", last, distances(last, "negative", 82)
  for frac in (0.0, 0.1, 0.97):
    lab = _bg(noise((9, 20, 37), random_keys(40, 4, 83, signed=True), 84, np.int32), frac, 85)
    yield "noise-bg%g" % frac, lab, distances(lab, "inf", 86)
