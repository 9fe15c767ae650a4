"""The walled-tile identity (tests/large_index_cases.py) on the CPU, for every operation that
tests/test_large_index_gpu.py checks through it: on a 3 x 3 x 3 lattice of small tiles (6 x 6 lattice in
2-D), the restatement of each operation over the whole lattice equals, inside every tile, the
restatement over the tile alone, translated.  Also: the comparison helper reports swapped variants and a
one-ulp change."""
import numpy as np
import pytest

import feature_cases as fc
import large_index_cases as lc
import medial_axis_cases as mc
import morphology_cases as morph
import nearest_labels_cases as nc
import parabolic_cases as pc
import parabolic_sites_cases as sc

torch = pytest.importorskip("torch")

K = 4
COUNTS3, TILE3 = (3, 3, 3), (6, 7, 8)
COUNTS2, TILE2 = (6, 6), (9, 10)


def lattice(pool, counts):
  return lc.assemble(torch.from_numpy(pool), counts).numpy()


def check(fn, pool, counts, t, what, sites=False):
  """fn(volume) -> array (or lead + shape array) for the lattice and for each variant."""
  big = torch.from_numpy(np.ascontiguousarray(fn(lattice(pool, counts))))
  want = torch.from_numpy(np.stack([np.ascontiguousarray(fn(p)) for p in pool]))
  lc.assert_tiles(big, want, counts, t, sites, what)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint32])
@pytest.mark.parametrize("w", [(1.0, 2.0, 1.0), (1.5, 0.75, 1.25)])
@pytest.mark.parametrize("border", [False, True])
def test_transforms(oracle, dtype, w, border):
  """edtsq / edt / sdfsq / sdf, and their cut at max_distance 2 and 8 (the bounded transforms' rule)."""
  pool = lc.label_pool(np.random.default_rng(1), K, TILE3, 1, dtype)
  for name in ("edtsq", "edt", "sdfsq", "sdf"):
    fn = getattr(oracle, name)
    kw = {} if name == "sdfsq" else {"black_border": border}
    check(lambda v: fn(v, w, **kw), pool, COUNTS3, 1, name)
    for d in (2.0, 8.0):
      def cut(v):
        full, s2 = fn(v, w, **kw), (oracle.sdfsq(v, w) if name.startswith("sdf") else oracle.edtsq(v, w, border))
        keep = np.abs(s2).astype(np.float64) <= d * d
        return np.where(keep, full, np.where(np.signbit(s2), -np.inf, np.inf)).astype(np.float32)
      check(cut, pool, COUNTS3, 1, "%s max_distance %g" % (name, d))


@pytest.mark.parametrize("w", [(1.0, 2.0), (1.25, 0.8)])
def test_feature_sites(w):
  """The translated sites of every tile (by brute force on the tile) satisfy the site contract of the
  whole lattice: another label, and value(p, site) equal to the lattice's squared distance."""
  from oracle import oracle
  pool = lc.label_pool(np.random.default_rng(2), K, TILE2, 1, np.uint8)
  big = lattice(pool, COUNTS2)
  sq = oracle.edtsq(big, w)
  small = [fc.brute_sites(p, w, False, False) for p in pool]
  check(lambda v: oracle.edtsq(v, w), pool, COUNTS2, 1, "edtsq")
  kmap = lc.variant_map(COUNTS2, K)
  for c in np.ndindex(*COUNTS2):
    d, s = small[kmap[c]]
    o = np.array(c) * np.array(TILE2)
    sl = tuple(slice(oo + 1, oo + ts - 1) for oo, ts in zip(o, TILE2))
    sites = s[(slice(None), slice(1, -1), slice(1, -1))] + o.reshape(2, 1, 1)
    p = np.indices(big.shape)[(slice(None),) + sl]
    fg = big[sl] != 0                                          # background maps to itself
    assert (big[tuple(sites)] != big[sl])[fg].all(), c
    got = fc.values(p, sites, big.shape, w, "C")
    assert np.array_equal(got.view(np.uint32), sq[sl].view(np.uint32)), c
    assert np.array_equal(d[1:-1, 1:-1].view(np.uint32), sq[sl].view(np.uint32)), c


def test_expand_labels():
  """skimage's expand_labels at distance 2.5 with walls of 3: the same voxels grow; where the grown
  label differs, both labels lie at the nearest distance within the tile (a tie)."""
  from oracle import oracle
  t, dist, w = 3, 2.5, (1.0, 1.0)
  pool = lc.label_pool(np.random.default_rng(3), K, (12, 13), t, np.uint8)
  counts = (4, 4)
  big = lattice(pool, counts)
  got, _ = fc.skimage_expand(big, dist, w)
  kmap = lc.variant_map(counts, K)
  for c in np.ndindex(*counts):
    p = pool[kmap[c]]
    want, _ = fc.skimage_expand(p, dist, w)
    o = np.array(c) * np.array(p.shape)
    g = got[tuple(slice(oo + t, oo + s - t) for oo, s in zip(o, p.shape))]
    wi = want[t:-t, t:-t]
    assert np.array_equal(g != 0, wi != 0), c
    sq = oracle.edtsq((p == 0).astype(np.uint8), w)            # squared distance to the nearest label
    for y, x in np.argwhere(g != wi):
      near = np.argwhere(p == g[y, x])
      assert ((near - (y + t, x + t)) ** 2).sum(1).min() == sq[y + t, x + t], (c, y, x)


@pytest.mark.parametrize("op,border", [("erode", False), ("erode", True), ("open", False), ("open", True),
                                       ("dilate", False), ("close", False)])
def test_morphology(op, border):
  """Radius 2, walls of 1.  A closing's black border would lie two voxels from the interior, within the
  radius, so the closing (here and on the GPU) runs without it."""
  pool = lc.label_pool(np.random.default_rng(4), K, TILE3, 1, np.uint16)
  kw = {} if op == "dilate" else {"black_border": border}
  check(lambda v: morph.threshold(op, v, 2.0, (1.0, 1.0, 1.5), **kw), pool, COUNTS3, 1, op)


@pytest.mark.parametrize("op", ["erode", "dilate"])
def test_parabolic(op):
  """Values and sites (translated) with the wall at the volume's least (greatest) value."""
  pool = lc.value_pool(np.random.default_rng(5), K, TILE3, 1, op)
  w = (1.0, 2.0, 1.0)
  check(lambda f: pc.restate(op, f, w), pool, COUNTS3, 1, op)
  check(lambda f: sc.restate(op, f, w)[1], pool, COUNTS3, 1, op + " sites", sites=True)


@pytest.mark.parametrize("k", [1, 2])
def test_nearest_labels(k):
  """Walls of 3 and max_distance 2.5: no label beyond a wall is within reach."""
  pool = lc.label_pool(np.random.default_rng(6), K, (10, 11), 3, np.uint32)
  for fn in ("per_pass", "per_label"):
    def run(v):
      d, n = getattr(nc, fn)(v, 2.5, (1.0, 1.0), k=k, squared=False)
      return np.concatenate([d.view(np.uint32), n.view(np.uint32)])
    check(run, pool, (4, 4), 3, "%s k=%d" % (fn, k))


@pytest.mark.parametrize("border", [False, True])
def test_medial_axis(border):
  pool = lc.label_pool(np.random.default_rng(7), K, TILE3, 1, np.uint8)
  w = (1.0, 2.0, 1.0)
  check(lambda v: mc.restate(v, w, border)[0], pool, COUNTS3, 1, "medial_axis")


def test_stack_identity(oracle):
  """A stack is the lattice (B, 1, 1) of its volumes without walls; the stack comparison names the
  volume of a planted one-ulp change."""
  pool = lc.label_pool(np.random.default_rng(8), K, TILE3, 0, np.uint8)
  stack = lc.stack(torch.from_numpy(pool), 10)
  assert torch.equal(stack.reshape(-1, *TILE3[1:]), torch.from_numpy(lattice(pool, (10, 1, 1))))
  w = (1.0, 2.0, 1.0)
  got = torch.from_numpy(np.stack([oracle.edtsq(v, w) for v in stack.numpy()]))
  want = torch.from_numpy(np.stack([oracle.edtsq(p, w) for p in pool]))
  assert lc.stack_mismatches(got, want, chunk=1000) == {}
  got[6, 1, 2, 3] = torch.nextafter(got[6, 1, 2, 3], torch.tensor(np.inf))
  assert lc.stack_mismatches(got, want, chunk=1000) == {6: 1}
  planes = torch.stack([got, got])
  assert lc.stack_mismatches(planes, torch.stack([want, want], 1), lead=1) == {6: 2}


def test_comparison_reports_swaps_and_one_ulp(oracle):
  """The helper names the tiles of two swapped variants and the one voxel moved by one ulp."""
  pool = lc.label_pool(np.random.default_rng(9), K, TILE3, 1, np.uint8)
  w = (1.0, 1.0, 1.0)
  big = torch.from_numpy(oracle.edtsq(lattice(pool, COUNTS3), w))
  want = np.stack([oracle.edtsq(p, w) for p in pool])
  assert lc.tile_mismatches(big, torch.from_numpy(want), COUNTS3, 1) == {}
  kmap = lc.variant_map(COUNTS3, K)
  swapped = np.where(kmap == 1, 2, np.where(kmap == 2, 1, kmap))
  bad = lc.tile_mismatches(big, torch.from_numpy(want), COUNTS3, 1, kmap=swapped)
  assert set(bad) == {tuple(c) for c in np.argwhere((kmap == 1) | (kmap == 2))}
  assert all(n > 0 for n in bad.values())
  moved = want.copy()
  moved[3, 2, 3, 4] = np.nextafter(moved[3, 2, 3, 4], np.float32(np.inf))
  bad = lc.tile_mismatches(big, torch.from_numpy(moved), COUNTS3, 1)
  assert bad == {tuple(c): 1 for c in np.argwhere(kmap == 3)}
  with pytest.raises(AssertionError, match=r"%d tiles differ in %d voxels" % (len(bad), len(bad))):
    lc.assert_tiles(big, torch.from_numpy(moved), COUNTS3, 1, what="edtsq")
  # a voxel in a wall is not compared
  moved = want.copy()
  moved[3, 0, 3, 4] += 1
  assert lc.tile_mismatches(big, torch.from_numpy(moved), COUNTS3, 1) == {}
