#!/usr/bin/env python
"""A few small transforms that touch every kernel variant, for runs under compute-sanitizer:
  compute-sanitizer --tool memcheck  python tools/sanitize_cases.py
  compute-sanitizer --tool racecheck python tools/sanitize_cases.py
Results are still compared with the oracle, so a sanitizer-induced slowdown cannot hide a wrong answer."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
import edt_b200 as edt  # noqa: E402
from oracle import oracle  # noqa: E402

rng = np.random.default_rng(3)
done = 0


def check(name, got, want):
  global done
  assert np.array_equal(got, want, equal_nan=True), name
  done += 1


# vector X pass + TMA tile kernel (sx % 4 == 0), short / long runs, all epilogues
for kind in ("iid", "blocks", "balls"):
  lab = np.asfortranarray(cases.random_volume(rng, (64, 80, 72), kind, np.uint32))
  check("edtsq " + kind, edt.edtsq(lab, anisotropy=(1, 2, 3)), oracle.edtsq(lab, anisotropy=(1, 2, 3)))
  check("sdf " + kind, edt.sdf(lab, anisotropy=(1, 2, 3), black_border=True),
        oracle.sdf(lab, anisotropy=(1, 2, 3), black_border=True))
# generic X pass + plain-load tile kernel (odd sizes), every label width
for dtype in (np.uint8, np.uint16, np.uint64):
  lab = np.asfortranarray(cases.random_volume(rng, (37, 45, 51), "blocks", dtype))
  check("odd " + np.dtype(dtype).name, edt.edt(lab, anisotropy=(0.7, 1.3, 2.9)), oracle.edt(lab, anisotropy=(0.7, 1.3, 2.9)))
# long runs across many chunks (stitching stage), 2-D and 1-D drivers
lab = np.ones((8, 300, 12), dtype=np.uint8, order="F")
lab[3, 150, 5] = 0
check("long runs", edt.edtsq(lab), oracle.edtsq(lab))
img = cases.random_volume(rng, (200, 130), "balls", np.uint16)
check("2-D", edt.edt(img, black_border=True), oracle.edt(img, black_border=True))
row = cases.random_volume(rng, (700,), "blocks", np.uint32)
check("1-D", edt.edtsq(row, anisotropy=2.5), oracle.edtsq(row, anisotropy=2.5))
# lines beyond the tile kernel (n > 4096): thread-per-line kernel
tall = np.asfortranarray(cases.random_volume(rng, (8, 4200, 2), "blocks", np.uint8))
check("n > 4096", edt.edtsq(tall), oracle.edtsq(tall))
# voxel graph
lab, graph, kw = cases.random_graph_case(7)
check("voxel graph", edt.edtsq(lab, voxel_graph=graph, **kw), oracle.edtsq(lab, voxel_graph=graph, **kw))
# the 2-CTA variant of the tile kernel (label noise seen by the previous transform) and the double
# hull tests (non-integer weights) on long varying runs; a Voronoi-like volume on a 512-row axis
lab = np.asfortranarray(cases.random_volume(rng, (64, 80, 72), "iid", np.uint32))
for _ in range(2):
  got = edt.edtsq(lab)
check("noise twice", got, oracle.edtsq(lab))
from scipy.spatial import cKDTree  # noqa: E402
pts = rng.uniform(0, 1, (12, 3)) * np.array([40, 512, 24])
grid = np.stack(np.meshgrid(np.arange(40.0), np.arange(512.0), np.arange(24.0), indexing="ij"), -1).reshape(-1, 3)
vor = np.asfortranarray((cKDTree(pts).query(grid)[1] + 1).astype(np.uint16).reshape(40, 512, 24))
check("voronoi int", edt.edtsq(vor, anisotropy=(1, 1, 2)), oracle.edtsq(vor, anisotropy=(1, 1, 2)))
check("voronoi double", edt.edtsq(vor, anisotropy=(0.7, 1.3, 2.9)), oracle.edtsq(vor, anisotropy=(0.7, 1.3, 2.9)))
# wide variant (lines of 513..1024 rows: decoupled warps, chunk mask) and the constant runs that are
# not stored: solid volume with a black border through every epilogue, blocks, noise, one hole
wide = np.ones((16, 1024, 8), dtype=np.uint8, order="F")
check("wide ones bb", edt.edtsq(wide, anisotropy=(6, 6, 30), black_border=True),
      oracle.edtsq(wide, anisotropy=(6, 6, 30), black_border=True))
check("wide ones sdf", edt.sdf(wide, black_border=True), oracle.sdf(wide, black_border=True))
wide[7, 600, 3] = 0
check("wide hole", edt.edt(wide), oracle.edt(wide))
for kind in ("iid", "blocks"):
  lab = np.asfortranarray(cases.random_volume(rng, (16, 1000, 12), kind, np.uint32))
  check("wide " + kind, edt.edtsq(lab, black_border=(kind == "blocks")), oracle.edtsq(lab, black_border=(kind == "blocks")))
solid = np.ones((48, 96, 40), dtype=np.uint16, order="F")
solid[:, :, 20:] = 2
check("solid edt", edt.edt(solid, anisotropy=(2, 1, 3), black_border=True),
      oracle.edt(solid, anisotropy=(2, 1, 3), black_border=True))
# stacks (stacked=True): one launch per pass over many volumes -- the plane plan on label noise whose
# next volume repeats the last slice, odd-sized volumes (Z pass without TMA), long-line weights, host
# groups and the feature resolver across volumes
noise = rng.integers(1, 1 << 20, (4, 9, 40, 64)).astype(np.uint32)
noise[1:, 0] = noise[:-1, -1]
for _ in range(2):
  got = edt.edtsq(noise, stacked=True)
check("stack noise", got, np.stack([oracle.edtsq(v) for v in noise]))
odd = np.stack([cases.random_volume(rng, (5, 7, 9), "blocks", np.uint16) for _ in range(6)])
check("stack odd", edt.sdf(odd, black_border=True, stacked=True), np.stack([oracle.sdf(v, black_border=True) for v in odd]))
check("stack long", edt.edtsq(odd, anisotropy=(0.7, 1.3, 2.9), stacked=True, max_device_bytes=2 * 315 * 14),
      np.stack([oracle.edtsq(v, anisotropy=(0.7, 1.3, 2.9)) for v in odd]))
_, idx = edt.feature_transform(odd, stacked=True, return_distances=True)
for b in range(len(odd)):
  check("stack feature %d" % b, idx[:, b], edt.feature_transform(odd[b]))
# bounded transforms (max_distance): window passes with and without sites, a pass that falls back to
# the unbounded kernel, and a zero-radius pass; each against the oracle's transform with the band applied
def banded(unbounded, sq, d):
  keep = np.abs(sq).astype(np.float64) <= d * d
  return np.where(keep, unbounded, np.where(np.signbit(sq), -np.inf, np.inf)).astype(np.float32)
blk = np.asfortranarray(cases.random_volume(rng, (40, 36, 30), "blocks", np.uint32))
for d, an in ((2.5, (1, 1, 1)), (7.9, (0.7, 1.3, 2.9)), (40.0, (1, 4, 1)), (24.0, (6, 6, 30))):
  sq = oracle.sdfsq(blk, anisotropy=an)
  check("bounded sdf %g" % d, edt.sdf(blk, anisotropy=an, max_distance=d), banded(oracle.sdf(blk, anisotropy=an), sq, d))
  dist, _ = edt.feature_transform(blk, an, signed=True, return_distances=True, max_distance=d)
  check("bounded feature %g" % d, dist, banded(oracle.sdf(blk, anisotropy=an), sq, d))
# surface distances: every kernel (mask, count, gather) on 1-D to 3-D volumes and a stack, keys in
# shared memory, several groups, against the scipy restatement
import surface_cases as sc  # noqa: E402
for shape, an in (((33,), (2.0,)), ((14, 11), (1.0, 3.0)), ((9, 8, 10), (1.0, 2.0, 3.0))):
  a, b = sc.random_pair(rng, shape, nlabels=4, dtype=np.uint16, flips=0.1)
  keys = sc.default_keys(a, b)
  sd = edt.surface_distances(a, b, an, max_device_bytes=3 * 5 * a.size)
  for k, (ab, ba) in enumerate(sc.segments(a, b, keys, an)):
    check("surface %dd key %d" % (len(shape), k), sd.values[sd.offsets[2 * k]:sd.offsets[2 * k + 2]],
          np.concatenate([ab, ba]))
a, b = sc.random_pair(rng, (3, 7, 9, 8), nlabels=5, dtype=np.int64, flips=0.1)
check("surface stack", edt.hausdorff_distance(a, b, stacked=True),
      np.stack([sc.metric(x, y, sc.default_keys(a, b), (1.0, 1.0, 1.0), sc.hausdorff) for x, y in zip(a, b)]))
# spherical morphology: the label- and mask-writing window store (every (runs, labels) width pair), the
# select after an unbounded last pass, the float fold, the two-stage calls and a stack, against the
# threshold restatement on the oracle
import morphology_cases as mc  # noqa: E402
for dtype in (np.uint8, np.uint16, np.uint32, np.uint64, np.float32):
  lab = np.asfortranarray(cases.random_volume(rng, (21, 19, 17), "blocks", dtype))
  for op in mc.OPS:
    for r in (2.0, 4.5):
      fn = getattr(edt, "spherical_" + op)
      got = fn(lab, r) if op == "dilate" else fn(lab, r, None, True)
      check("morphology %s %s r=%g" % (op, np.dtype(dtype).name, r), mc._raw(got),
            mc._raw(mc.threshold(op, lab, r, None, op != "dilate")))
vols = np.stack([cases.random_volume(rng, (12, 14, 9), "blocks", np.uint16) for _ in range(3)])
check("morphology stack", edt.spherical_open(vols, 2.0, stacked=True),
      np.stack([mc.threshold("open", v, 2.0) for v in vols]))
# parabolic erosion / dilation: the X and Y / Z tile kernels with ragged tiles, the long-line hull, the
# brute-force minimum and the copy of an overflowing w^2, against the numpy restatement
import parabolic_cases as pc  # noqa: E402
for shape, w in (((5, 33, 37), (0.7, 1.3, 2.9)), ((3, 1100), (1.0, 0.7)), ((1100, 2), (1.3, 1.0)),
                 ((23172,), (0.7,)), ((4, 6, 7), (1e20, 1.0, 2.0))):
  for op in ("erode", "dilate"):
    f = pc.values("special", shape, rng)
    check("parabolic %s %s" % (op, shape), getattr(edt, "parabolic_" + op)(f, w), pc.restate(op, f, w))
# nearest labels: the X kernel and both later-pass variants (staged, global) on ragged tiles, every k and
# width, against the per-pass restatement
import nearest_labels_cases as nlc  # noqa: E402
for shape, d, k, dtype in (((5, 33, 37), 3.5, 2, np.uint32), ((3, 70, 9), 50.0, 4, np.uint64), ((70,), 6.0, 3, np.int8),
                           ((9, 66), 4.0, 1, np.uint16)):
  lab = nlc.volume("seeds", shape, dtype, rng)
  got, want = edt.nearest_labels(lab, d, k=k, squared=True), nlc.per_pass(lab, d, None, k)
  check("nearest_labels %s k=%d" % (shape, k), got[0], want[0])
  check("nearest_labels labels %s k=%d" % (shape, k), got[1], want[1])
# medial axis: the mark kernel over a stack, with and without distances, float labels, against the restatement
import medial_axis_cases as mac  # noqa: E402
for shape, dtype, stacked in (((4, 9, 11, 7), np.uint16, True), ((13, 30), np.float32, False), ((50,), np.int8, False)):
  lab = (rng.integers(0, 3, shape) * (rng.random(shape) < 0.9)).astype(dtype)
  got, dist = edt.medial_axis(lab, None, True, return_distance=True, stacked=stacked)
  check("medial_axis %s" % (shape,), got, mac.restate(lab, None, True, stacked=stacked)[0])
  check("medial_axis only %s" % (shape,), edt.medial_axis(lab, None, True, stacked=stacked), got)
# skeleton: the cooperative thinning kernel over a stack, 2-D and 3-D, with and without distances, against
# the restatement
import skeleton_cases as skc  # noqa: E402
for shape, dtype, stacked, w in (((3, 9, 11, 7), np.uint16, True, (1.0, 1.0, 2.0)), ((13, 30), np.int64, False, None),
                                 ((6, 10, 12), np.uint8, False, (4.0, 4.0, 40.0))):
  lab = (rng.integers(0, 3, shape) * (rng.random(shape) < 0.9)).astype(dtype)
  got, dist = edt.skeletonize(lab, w, True, return_distance=True, stacked=stacked)
  check("skeletonize %s" % (shape,), got, skc.restate(lab, w, True, stacked=stacked))
  check("skeletonize only %s" % (shape,), edt.skeletonize(lab, w, True, stacked=stacked), got)
# per-label views: a nearly full table whose probe chain wraps past its end, a table that overflows, and
# a sub-box drawn at a ragged row length; the helpers are the GPU tests' own
import each_cases as ec  # noqa: E402
import test_each_gpu as teg  # noqa: E402
keys = np.union1d(ec.colliding_keys(64, 128, 127, 4), ec.random_keys(60, 4, 1))
lab = ec.noise((6, 20, 37), keys, 2, np.int32)
teg.check_table(edt, lab, ec.distances(lab, "signed", 3), 128)
lab = ec.singletons((3, 5, 43), ec.random_keys(700, 8, 4, signed=True), 5, np.int64, background=0.2)
rc, overflow, table = teg.c_stats(edt, lab, ec.distances(lab, "inf", 6), 64)
assert rc == 0 and overflow == 1 and np.isin(table["keys"][table["keys"] != 0], ec.keys_of(lab)).all()
lab = ec.voronoi_many((5, 7, 75), 6, 7, np.uint16)
dist = ec.distances(lab, "ties", 8)
out = teg.device_bytes(np.zeros(lab.shape, np.float32))
key, box = int(ec.keys_of(lab).max()), (2, 1, 1, 68, 5, 3)
assert teg.c_extract(edt, teg.device_bytes(lab), 2, teg.device_bytes(dist), ec.dims_of(lab.shape), key, box, 0, out) == 0
check("each sub-box", out.cpu().numpy().view(np.float32).reshape(lab.shape), ec.extract(lab, dist, key, box))
print("sanitize_cases: %d results equal to the oracle" % done)
