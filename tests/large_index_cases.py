"""Walled tiles: large volumes whose answers are known tile by tile.

A big volume is a lattice of small tiles, each one of K variants drawn from a pool.  Every tile's outer
`t` voxels along each axis are a wall of one label W that no tile uses inside (for the parabolic passes:
the volume's least value for erosion, its greatest for dilation).  Any voxel outside a tile is then
dominated, seen from the tile's interior, by the wall voxel on the segment to it (same other
coordinates, strictly closer along one axis), so each operation gives the tile's interior the result of
the tile computed alone, translated.  tests/test_large_index_oracle.py checks that identity for every
operation on a small lattice; tests/test_large_index_gpu.py then relies on it past 2^31 and 2^32 voxels.

The variant of the tile at lattice coordinate (c_0, c_1, ...) is (c_0 + 3 c_1 + 5 c_2) % K, so that
face neighbours differ whenever K does not divide 1, 2, 3, 4 or 5 (K = 4 or 7 here) and a misaddressed
read lands on different content.  A stack of B volumes is the lattice (B, 1, 1) of tiles without walls.

The pools are drawn on the host with numpy; the lattice is assembled with torch on the pool's device,
one slab of tiles at a time, and compared there the same way.
"""
import numpy as np

COEF = (1, 3, 5)


def wall_label(dtype):
  """W: the largest value of the dtype's unsigned reading (bit 63 / 31 / ... set), never used inside."""
  dtype = np.dtype(dtype)
  return dtype.type(np.iinfo(dtype).max) if dtype.kind == "u" else dtype.type(-1)


def _interior(rng, kind, shape, nlabels):
  """Labels 0..nlabels of one tile's inside."""
  if kind == "voronoi":
    seeds = np.stack([rng.integers(0, s, 6) for s in shape], 1)
    grid = np.ogrid[tuple(slice(0, s) for s in shape)]
    d = np.stack([sum((g - c) ** 2 for g, c in zip(grid, seed)) for seed in seeds])
    lab = rng.integers(0, nlabels + 1, 6)[d.argmin(0)]
  elif kind == "blocks":
    coarse = rng.integers(0, nlabels + 1, tuple(-(-s // 3) for s in shape))
    lab = coarse
    for ax, s in enumerate(shape):
      lab = np.repeat(lab, 3, axis=ax).take(np.arange(s), axis=ax)
  elif kind == "noise":
    lab = rng.integers(0, 3, shape)
  else:                                       # "balls": label 0 around a few balls
    lab = np.zeros(shape, np.int64)
    grid = np.ogrid[tuple(slice(0, s) for s in shape)]
    for i in range(3):
      c = [rng.integers(0, s) for s in shape]
      r2 = rng.integers(1, 1 + max(2, min(shape) // 2) ** 2)
      lab[sum((g - cc) ** 2 for g, cc in zip(grid, c)) <= r2] = 1 + i % nlabels
  return lab


KINDS = ("voronoi", "blocks", "noise", "balls")


def label_pool(rng, K, tile, t, dtype, nlabels=5):
  """(K,) + tile labels of `dtype`: variant k has KINDS[k % 4] content inside a wall of t voxels."""
  inner = tuple(s - 2 * t for s in tile)
  assert min(inner) >= 1, (tile, t)
  pool = np.empty((K,) + tuple(tile), dtype)
  pool[...] = wall_label(dtype)
  core = (slice(None),) + tuple(slice(t, s - t) for s in tile)
  pool[core] = np.stack([_interior(rng, KINDS[k % len(KINDS)], inner, nlabels) for k in range(K)]).astype(dtype)
  return pool


def value_pool(rng, K, tile, t, op, top=40):
  """(K,) + tile float32 samples for parabolic_erode (op "erode") or _dilate: integers 0..top inside, a
  fifth of them +inf (-inf for dilation), and walls of the global least value 0 (greatest `top`)."""
  inner = tuple(s - 2 * t for s in tile)
  vals = rng.integers(0, top + 1, (K,) + inner).astype(np.float32)
  vals[rng.random(vals.shape) < 0.2] = np.inf if op == "erode" else -np.inf
  pool = np.full((K,) + tuple(tile), 0.0 if op == "erode" else float(top), np.float32)
  pool[(slice(None),) + tuple(slice(t, s - t) for s in tile)] = vals
  return pool


def block_pool(rng, K, tile, dtype, flips=8, nlabels=5):
  """(a, b): two (K,) + tile label pools whose surfaces are few voxels -- two to three large boxes of
  labels 1..nlabels on background 0 -- b being a with `flips` voxels of each variant relabelled."""
  a = np.zeros((K,) + tuple(tile), dtype)
  for k in range(K):
    for i in range(2 + k % 2):
      lo = [rng.integers(0, s // 2) for s in tile]
      hi = [l + rng.integers(s // 4, s // 2) for l, s in zip(lo, tile)]
      a[(k,) + tuple(slice(l, h) for l, h in zip(lo, hi))] = 1 + (k + i) % nlabels
  b = a.copy()
  for k in range(K):
    at = tuple(rng.integers(0, s, flips) for s in tile)
    b[(k,) + at] = rng.integers(0, nlabels + 1, flips)
  return a, b


def variant_map(counts, K):
  """int64 array of shape `counts`: the variant of every tile."""
  grid = np.indices(counts)
  return sum(COEF[i] * grid[i] for i in range(len(counts))) % K


def _tiles_view(slab, lead, counts, tile):
  """slab (lead + (tile[0],) + big shape[1:]) as (counts[1:]) + lead + tile, a view."""
  nd = len(tile)
  shp = tuple(slab.shape[:lead]) + (tile[0],)
  for c, s in zip(counts[1:], tile[1:]):
    shp += (c, s)
  v = slab.reshape(shp)
  tile_axes = [lead] + [lead + 2 + 2 * i for i in range(nd - 1)]
  count_axes = [lead + 1 + 2 * i for i in range(nd - 1)]
  return v.permute(*count_axes, *range(lead), *tile_axes)


def assemble(pool, counts, out=None):
  """The lattice of `counts` tiles from pool ((K,) + tile, a torch tensor), on the pool's device."""
  import torch
  K, tile = pool.shape[0], tuple(pool.shape[1:])
  kmap = torch.from_numpy(variant_map(counts, K)).to(pool.device)
  if out is None:
    out = torch.empty(tuple(c * s for c, s in zip(counts, tile)), dtype=pool.dtype, device=pool.device)
  for c0 in range(counts[0]):
    slab = out[c0 * tile[0]:(c0 + 1) * tile[0]]
    _tiles_view(slab, 0, counts, tile).copy_(pool[kmap[c0]])
  return out


def stack(pool, count):
  """count volumes, volume b of variant b % K: the lattice (count, 1, ...) without walls, in one gather."""
  import torch
  return pool[torch.arange(count, device=pool.device) % pool.shape[0]]


def _bits(x):
  import torch
  if x.dtype == torch.bool:
    return x.view(torch.uint8)
  return x.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[x.element_size()])


def tile_mismatches(got, want, counts, t=0, sites=False, kmap=None):
  """{tile coordinate: voxels that differ} between got (lead + big shape) and the per-variant answers
  want ((K,) + lead + tile), bit for bit, over every tile's interior (the tile less `t` voxels on each
  side).  sites: lead is one plane of array coordinates per axis, and want's are translated to each
  tile's origin.  kmap: the variant map to expect (default variant_map(counts, K))."""
  import torch
  K = want.shape[0]
  nd = len(counts)
  lead = got.dim() - nd
  tile = tuple(want.shape[1 + lead:])
  if kmap is None:
    kmap = variant_map(counts, K)
  kmap = torch.from_numpy(np.asarray(kmap)).to(got.device)
  inner = (Ellipsis,) + tuple(slice(t, s - t) for s in tile)
  want_in = want[inner]
  out = {}
  for c0 in range(counts[0]):
    g = _tiles_view(got[(slice(None),) * lead + (slice(c0 * tile[0], (c0 + 1) * tile[0]),)], lead, counts, tile)
    w = want_in[kmap[c0]]                             # counts[1:] + lead + inner tile
    if sites:
      coords = torch.meshgrid(*[torch.arange(c, device=got.device) for c in counts[1:]], indexing="ij")
      origin = torch.stack([torch.full_like(coords[0], c0)] + list(coords)) * torch.tensor(
        tile, device=got.device).view((nd,) + (1,) * (nd - 1))
      w = w + origin.permute(*range(1, nd), 0).reshape(tuple(counts[1:]) + (nd,) + (1,) * nd).to(w.dtype)
    diff = (_bits(g[inner].contiguous()) != _bits(w)).reshape(tuple(counts[1:]) + (-1,)).sum(-1)
    bad = diff.nonzero()
    if bad.numel():
      for idx, n in zip(bad.tolist(), diff[tuple(bad.T)].tolist()):
        out[(c0,) + tuple(idx)] = int(n)
  return out


def assert_tiles(got, want, counts, t=0, sites=False, what=""):
  """AssertionError naming the tiles that differ (first few) and how many voxels, when any do."""
  bad = tile_mismatches(got, want, counts, t, sites)
  if bad:
    first = sorted(bad)[:4]
    K = want.shape[0]
    kmap = variant_map(counts, K)
    raise AssertionError("%s: %d tiles differ in %d voxels; first %s" % (
      what, len(bad), sum(bad.values()), ", ".join("%s (variant %d): %d" % (c, kmap[c], bad[c]) for c in first)))


def stack_mismatches(got, want, lead=0, chunk=1 << 28):
  """{volume: voxels that differ} between a stack's results got (lead + (count,) + volume) and the
  per-variant answers want ((K,) + lead + volume), volume b being variant b % K; bit for bit, about
  `chunk` voxels at a time."""
  import torch
  K = want.shape[0]
  count = got.shape[lead]
  step = max(1, chunk // max(1, want[0].numel()))
  out = {}
  for b0 in range(0, count, step):
    b1 = min(count, b0 + step)
    g = got[(slice(None),) * lead + (slice(b0, b1),)]
    w = want[torch.arange(b0, b1, device=want.device) % K].movedim(0, lead)
    diff = (_bits(g) != _bits(w)).movedim(lead, 0).reshape(b1 - b0, -1).sum(1)
    bad = diff.nonzero().view(-1)
    for b, n in zip(bad.tolist(), diff[bad].tolist()):
      out[b0 + b] = int(n)
  return out


def assert_stack(got, want, lead=0, what=""):
  bad = stack_mismatches(got, want, lead)
  if bad:
    first = sorted(bad)[:4]
    raise AssertionError("%s: %d volumes differ in %d voxels; first %s" % (
      what, len(bad), sum(bad.values()), ", ".join("%d (variant %d): %d" % (b, b % want.shape[0], bad[b]) for b in first)))
