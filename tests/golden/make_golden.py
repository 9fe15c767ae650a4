"""Generate tests/golden/reference_vectors.npz by running the UNMODIFIED compiled reference
(oracle/_ref, built by oracle/Makefile from the reference's sources) on seeded inputs.

Run where the reference's sources are present:  python tests/golden/make_golden.py
The .npz is committed, so the tests need no reference: they only read the fixture.
Each case stores the input labels, the call arguments and the reference's edtsq / edt / sdf;
the g* cases do the same for the voxel_graph= path.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import cases  # noqa: E402
from oracle import oracle  # noqa: E402

SEEDS = list(range(1000, 1048))
GRAPH_SEEDS = list(range(0, 36))


def main():
  ref = oracle.load_reference()
  if ref is None:
    raise SystemExit("oracle/_ref is not built: run `make -C oracle ref` where the reference's sources are (REF=...)")
  blob = {}
  meta = []
  for seed in SEEDS:
    labels, kwargs = cases.random_case(seed)
    an = kwargs["anisotropy"]
    key = "s%d" % seed
    blob[key + "_labels"] = labels
    blob[key + "_aniso"] = np.atleast_1d(np.asarray(an, dtype=np.float64))
    blob[key + "_border"] = np.array(kwargs["black_border"])
    blob[key + "_edtsq"] = ref.edtsq(labels, **kwargs)
    blob[key + "_edt"] = ref.edt(labels, **kwargs)
    blob[key + "_sdf"] = ref.sdf(labels, **kwargs)
    meta.append(seed)
  # the reference's own headline small config: 64^3 uint32 ones, F order, black border
  cfg1 = np.ones((64, 64, 64), dtype=np.uint32, order="F")
  blob["cfg1_edtsq"] = ref.edtsq(cfg1, black_border=True, parallel=1)
  blob["seeds"] = np.array(meta)
  # voxel_graph path (edt.pyx:514-620, 736-844): edtsq / edt / sdf under a connectivity graph
  for seed in GRAPH_SEEDS:
    labels, graph, kwargs = cases.random_graph_case(seed)
    key = "g%d" % seed
    blob[key + "_labels"] = labels
    blob[key + "_graph"] = graph
    blob[key + "_aniso"] = np.asarray(kwargs["anisotropy"], dtype=np.float64)
    blob[key + "_border"] = np.array(kwargs["black_border"])
    with np.errstate(invalid="ignore"):
      blob[key + "_edtsq"] = ref.edtsq(labels, voxel_graph=graph, **kwargs)
      blob[key + "_edt"] = ref.edt(labels, voxel_graph=graph, **kwargs)
      blob[key + "_sdf"] = ref.sdf(labels, voxel_graph=graph, **kwargs)
  blob["graph_seeds"] = np.array(GRAPH_SEEDS)
  out = os.path.join(HERE, "reference_vectors.npz")
  np.savez_compressed(out, **blob)
  print("wrote", out, os.path.getsize(out), "bytes,", len(meta), "cases")


def rounding_edge_cases():
  """Whole transforms at the float32 rounding edges: (name, labels, anisotropy, black_border).
  - tie2d / tie3d: a candidate w2 * 9 + 2^-52 that is a double-rounding tie (the reference rounds
    twice, a fused multiply-add once and one ulp higher);
  - z lines of 128 to 4096 rows at (4, 4, 40) and (1, 1, 40): integer weights, values above 2^24;
  - isotropic-in-x/y volumes at z weight 1023 and 1024, just inside and just outside the integer
    hull tests' w2 < 2^20 guard, with objects as deep as the volume."""
  out = []
  tie = np.ones((2, 4), dtype=np.uint8, order="F")
  tie[0, 0] = 0
  w_tie = float(np.float32(1.333549976348877))
  out.append(("tie2d", tie, (2.0 ** -26, w_tie), False))
  tie3 = np.ones((2, 4, 3), dtype=np.uint8, order="F")
  tie3[0, 0, :] = 0
  out.append(("tie3d", tie3, (2.0 ** -26, w_tie, 1.0), False))
  rng = np.random.default_rng(2024)
  for n in (128, 1000, 4096):
    shape = (8, 4, n) if n < 4096 else (2, 2, n)
    # Voronoi-like: runs of 60 to 1500 rows with distinct labels, no background
    cuts = np.cumsum(rng.integers(60, 1500, n))
    vor = (np.searchsorted(cuts, np.arange(n), side="right") % 250 + 1).astype(np.uint8)
    vor = np.asfortranarray(np.broadcast_to(vor, shape) + (rng.random(shape) < 0.002)).astype(np.uint8)
    # balls: all foreground but one background voxel per z line
    balls = np.ones(shape, dtype=np.uint16, order="F")
    zs = rng.integers(0, n, shape[:2])
    for (x, y), z in np.ndenumerate(zs):
      balls[x, y, z] = 0
    for kind, lab in (("voronoi", vor), ("balls", balls)):
      for an in ((4.0, 4.0, 40.0), (1.0, 1.0, 40.0)):
        for bb in (False, True):
          if n == 4096 and an[0] == 1.0 and bb:
            continue
          out.append(("z%d_%s_w%d_%s" % (n, kind, int(an[0]), "bb" if bb else "open"), lab, an, bb))
  deep = np.ones((32, 16, 40), dtype=np.uint32, order="F")
  deep[:, :, 0] = 0
  deep[rng.random(deep.shape) < 0.001] = 0
  for wz in (1023.0, 1024.0):
    out.append(("deep_wz%d" % int(wz), deep, (1.0, 1.0, wz), False))
  return out


def main_edges():
  ref = oracle.load_reference()
  if ref is None:
    raise SystemExit("oracle/_ref is not built: run `make -C oracle ref` where the reference's sources are (REF=...)")
  blob, names = {}, []
  for name, lab, an, bb in rounding_edge_cases():
    blob[name + "_labels"] = lab
    blob[name + "_aniso"] = np.asarray(an, dtype=np.float64)
    blob[name + "_border"] = np.array(bb)
    blob[name + "_edtsq"] = ref.edtsq(lab, anisotropy=an, black_border=bb)
    names.append(name)
  blob["names"] = np.array(names)
  out = os.path.join(HERE, "rounding_edges.npz")
  np.savez_compressed(out, **blob)
  print("wrote", out, os.path.getsize(out), "bytes,", len(names), "cases")


if __name__ == "__main__":
  # python tests/golden/make_golden.py [--edges]: the random / voxel-graph vectors, or the
  # rounding-edge cases (tests/golden/rounding_edges.npz)
  if "--edges" in sys.argv[1:]:
    main_edges()
  else:
    main()
