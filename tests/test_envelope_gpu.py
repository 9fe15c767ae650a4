"""GPU tests (-m gpu) of ONE later-axis pass at a time: edtb200_pass_later on arbitrary float32
samples against the oracle's envelope pass, bit for bit, in every kernel variant the launcher can
pick, at the float32 rounding edges; plus whole transforms at those edges against fixtures made by
the compiled reference (tests/golden/rounding_edges.npz).

Which variant ran is read back through edtb200_last_later_launch and collected in HIT; the last
test fails if a reachable variant was never run.  The 2-vs-3-CTA choice follows the run statistic
of the previous transform on the device, so the tests steer it by transforming a label-noise or a
constant volume first.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import envelope_cases as ec

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EDGES = os.path.join(HERE, "golden", "rounding_edges.npz")
SQRT, SIGNED = 1, 2
HIT = set()          # (label bytes, kernel, tx, tma, wide, ctas, int_hull, epilogue, all_double)
WIDTHS = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}
TIE_ANISO = (2.0 ** -26, float(np.float32(1.333549976348877)))


def steer(edt, noisy):
  """Make the next tile launch predict label noise (2 CTAs per SM) or not (3)."""
  rng = np.random.default_rng(0)
  vol = rng.integers(0, 256, (64, 64, 16), dtype=np.uint32) if noisy else np.ones((64, 64, 16), np.uint32)
  edt.edtsq(vol)


def run_pass(edt, lab, f, axis, w, lo, hi, flags=0):
  """edtb200_pass_later on C-ordered (z, y, x) arrays; returns (result, variant)."""
  import torch
  lab = np.ascontiguousarray(lab)
  nbytes = lab.dtype.itemsize
  lt = torch.from_numpy(lab.view(np.dtype("i%d" % nbytes) if nbytes > 1 else np.uint8)).cuda()
  ft = torch.from_numpy(np.ascontiguousarray(f, dtype=np.float32).copy()).cuda()
  sz, sy, sx = lab.shape
  lib = edt._lib()
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  rc = lib.edtb200_pass_later(lt.data_ptr(), nbytes, axis, sx, sy, sz, float(w), int(lo), int(hi), flags,
                              ft.data_ptr(), 0, stream)
  assert rc == 0, lib.edtb200_last_error()
  torch.cuda.synchronize()
  v = edt.last_later_launch()
  HIT.add((nbytes,) + tuple(v[k] for k in edt.LATER_LAUNCH_FIELDS))
  return ft.cpu().numpy(), v


def check_pass(edt, oracle, lab, f, axis, w, lo, hi, flags, what):
  got, v = run_pass(edt, lab, f, axis, w, lo, hi, flags)
  want = ec.expected_pass(oracle, lab, f, axis, w, lo, hi, sqrt=bool(flags & SQRT), negate=bool(flags & SIGNED))
  if not np.array_equal(got, want, equal_nan=True):
    bad = np.argwhere(~((got == want) | (np.isnan(got) & np.isnan(want))))
    first = tuple(bad[0])
    raise AssertionError("%s %s: %d voxels differ; first at %s: got %r want %r" % (
      what, v, len(bad), first, got[first], want[first]))
  return v


LENGTHS = (1, 2, 31, 32, 33, 63, 64, 65, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 1500, 2048, 4095,
           4096, 4097)


def geometries(n):
  """(shape, axis): a z line under 32 aligned x/y lines (TMA possible), under 15 lines of odd stride
  (no TMA), and a y line under 36 or 33 x lines."""
  yield (n, 4, 8), 2
  yield (n, 3, 5), 2
  if n <= 1025:
    yield (2, n, 36), 1
    yield (2, n, 33), 1


@pytest.mark.parametrize("nbytes", [1, 2, 4, 8])
def test_pass_profiles_vs_oracle(edt, oracle, nbytes):
  rng = np.random.default_rng(100 + nbytes)
  k = 0
  for n in LENGTHS:
    for shape, axis in geometries(n):
      for kind in ec.PROFILES:
        k += 1
        lab = ec.labels(rng, ec.LABELINGS[k % len(ec.LABELINGS)], shape, axis, WIDTHS[nbytes])
        f = ec.profile(rng, kind, shape)
        w = (1.0, 3.0, 0.7, 1.333549976348877)[k % 4] if kind not in ("int_ties", "zeros", "above_2_24") else \
            (1.0, 3.0)[k % 2]
        lo, hi = k % 2, (k // 2) % 2
        for flags in (0, (SQRT, SIGNED, SQRT | SIGNED)[k % 3]):
          if n <= 512:
            steer(edt, noisy=(k + flags) % 2 == 0)
          check_pass(edt, oracle, lab, f, axis, w, lo, hi, flags, (nbytes, shape, axis, kind, w, lo, hi, flags))


def test_pass_2_and_3_ctas_with_both_hulls(edt, oracle):
  """The 2-CTA and 3-CTA tile variants, each with integer and double hull tests, every label width."""
  rng = np.random.default_rng(7)
  for nbytes, dtype in WIDTHS.items():
    for noisy in (True, False):
      for kind, w in (("int_ties", 1.0), ("above_2_24", 3.0), ("real", 1.0), ("real", 0.7)):
        for labeling in ("runs", "single_rows", "one_run"):
          shape = (200, 4, 8)
          lab = ec.labels(rng, labeling, shape, 2, dtype)
          f = ec.profile(rng, kind, shape)
          for flags in (0, SQRT | SIGNED):
            steer(edt, noisy)
            v = check_pass(edt, oracle, lab, f, 2, w, 1, 0, flags, (nbytes, noisy, kind, w, labeling, flags))
            assert v["kernel"] == "tile" and v["ctas"] == (2 if noisy else 3), v


@pytest.mark.parametrize("m", [8, 9, 40])
def test_pass_hull_walk_plateau(edt, oracle, m):
  """At the first row of a chunk (64), two adjacent hull vertices whose candidates round to the
  same float32 must not stop the descent to a lower vertex farther down (integer samples above
  2^24); in the rows after it (65: three candidates round to K, 66: the exact minimiser is the
  lowest vertex again) the walk up the hull must not step past that vertex on a rounded tie.
  Both CTA variants here with the integer hull tests; the double hull tests run the same line in
  test_ab_switches_do_not_change_results (EDTB200_NO_INT_HULL), and the long-line kernel when the
  line is longer than a tile."""
  f, K, _ = ec.plateau_trap(m=m)
  shape = (len(f), 4, 8)
  vol = np.ascontiguousarray(np.broadcast_to(f.reshape(-1, 1, 1), shape))
  lab = np.ones(shape, np.uint8)
  want = ec.expected_pass(oracle, lab, vol, 2, 1.0, 0, 0)
  assert float(want[64, 0, 0]) == K - 128 and float(want[66, 0, 0]) == K
  for noisy in (False, True):
    steer(edt, noisy)
    got, v = run_pass(edt, lab, vol, 2, 1.0, 0, 0)
    assert v["kernel"] == "tile" and v["tx"] == 32 and v["tma"] == 1 and v["int_hull"] == 1, v
    assert v["ctas"] == (2 if noisy else 3), v
    for row in (64, 65, 66):
      assert np.array_equal(got[row], want[row]), (m, noisy, row, float(got[row, 0, 0]), float(want[row, 0, 0]))
    assert np.array_equal(got, want), (m, noisy)
  # the same line at the end of a 4100-row line (long-line kernel)
  long_f = np.concatenate([np.full(4100 - len(f), np.inf, np.float32), f])
  lvol = np.ascontiguousarray(np.broadcast_to(long_f.reshape(-1, 1, 1), (len(long_f), 1, 2)))
  v = check_pass(edt, oracle, np.ones(lvol.shape, np.uint8), lvol, 2, 1.0, 0, 0, 0, ("plateau long", m))
  assert v["kernel"] == "long", v


def test_transform_walk_ties_coarse_first_axis(edt, oracle):
  """Whole transforms whose X weight is much coarser than the Y weight (40 vs 4) on lines of about
  1024 voxels: values far above 2^24 with small steps between the Y candidates, where float32
  rounding ties between hull vertices are common."""
  rng = np.random.default_rng(17)
  for shape, an in (((1024, 1024), (40.0, 4.0)), ((1000, 1030), (40.0, 1.0)), ((96, 1024, 64), (40.0, 4.0, 1.0))):
    lab = np.asfortranarray((rng.random(shape) < 0.9995).astype(np.uint8))
    lab[..., 0] = 1
    for bb in (False, True):
      got = edt.edtsq(lab, anisotropy=an, black_border=bb)
      want = oracle.edtsq(lab, anisotropy=an, black_border=bb)
      bad = np.argwhere(got != want)
      assert len(bad) == 0, (shape, an, bb, len(bad), tuple(bad[0]), float(got[tuple(bad[0])]),
                             float(want[tuple(bad[0])]))


def test_pass_double_rounding_tie(edt, oracle):
  """w2 * 9 + 2^-52 is a double-rounding tie: the pass must give the reference's twice-rounded
  16.005199432373047 at row 3, not the fused multiply-add's 16.00520133972168."""
  shape = (4, 4, 8)
  f = np.full(shape, np.inf, np.float32)
  f[0] = 2.0 ** -52
  lab = np.ones(shape, np.uint8)
  got, v = run_pass(edt, lab, f, 2, TIE_ANISO[1], 0, 0)
  assert float(got[3, 0, 0]) == 16.005199432373047, (float(got[3, 0, 0]), v)
  assert v["all_double"] == 1, v
  check_pass(edt, oracle, lab, f, 2, TIE_ANISO[1], 0, 0, 0, "tie")


def test_rounding_edge_fixtures(edt):
  z = np.load(EDGES)
  for name in (str(s) for s in z["names"]):
    lab = z[name + "_labels"]
    an = tuple(float(a) for a in z[name + "_aniso"])
    bb = bool(z[name + "_border"])
    got = edt.edtsq(lab, anisotropy=an, black_border=bb)
    want = z[name + "_edtsq"]
    if not np.array_equal(got, want, equal_nan=True):
      bad = np.argwhere(got != want)
      first = tuple(bad[0])
      raise AssertionError("%s: %d voxels differ; first at %s: got %r want %r" % (
        name, len(bad), first, got[first], want[first]))


def test_integer_hull_bounds(edt, oracle):
  """Whole transforms just inside and just outside the integer hull tests' limits, with objects as
  deep as the volume: f + w2 n^2 < 2147483000 (z weight 11 vs 12 on 4096-row lines, isotropic 63
  vs 64 on 64 x 512 x 512) and w2 < 2^20 (z weight 1023 vs 1024)."""
  rng = np.random.default_rng(3)
  col = np.ones((8, 4, 4096), np.uint8, order="F")
  zs = rng.integers(0, 4096, (8, 4))
  for (x, y), zz in np.ndenumerate(zs):
    col[x, y, zz] = 0
  for wz in (11.0, 12.0):
    assert np.array_equal(edt.edtsq(col, anisotropy=(1.0, 1.0, wz)),
                          oracle.edtsq(col, anisotropy=(1.0, 1.0, wz))), wz
  big = np.ones((512, 512, 64), np.uint8, order="F")
  big[:, :, 0] = 0
  big[rng.integers(0, 512, 40), rng.integers(0, 512, 40), rng.integers(0, 64, 40)] = 0
  for w in (63.0, 64.0):
    assert np.array_equal(edt.edtsq(big, anisotropy=(w, w, w)), oracle.edtsq(big, anisotropy=(w, w, w))), w
  deep = np.ones((64, 64, 40), np.uint32, order="F")
  deep[:, :, 0] = 0
  for wz in (1023.0, 1024.0):
    assert np.array_equal(edt.edtsq(deep, anisotropy=(1.0, 1.0, wz)),
                          oracle.edtsq(deep, anisotropy=(1.0, 1.0, wz))), wz


def test_dyadic_weights_stay_on_tile_kernels(edt, oracle):
  """Weights that are multiples of a power of two below one (0.5 here) keep every sum exact in
  double, so the Z pass on 4096-row lines stays on the tile kernel."""
  rng = np.random.default_rng(29)
  lab = np.asfortranarray((rng.random((4, 8, 4096)) < 0.999).astype(np.uint16))
  for an in ((0.5, 0.5, 5.0), (0.5, 0.25, 0.75)):
    assert np.array_equal(edt.edtsq(lab, anisotropy=an), oracle.edtsq(lab, anisotropy=an)), an
    v = edt.last_later_launch()
    assert v["kernel"] == "tile" and v["all_double"] == 0, (an, v)


def battery(edt, oracle=None):
  """A fixed set of passes and transforms whose results must not depend on the A/B switches
  EDTB200_NO_INT_HULL / EDTB200_TILE_CTAS (read once per process)."""
  rng = np.random.default_rng(55)
  out = []
  f, _, _ = ec.plateau_trap(m=8)
  vol = np.ascontiguousarray(np.broadcast_to(f.reshape(-1, 1, 1), (len(f), 4, 8)))
  out.append(run_pass(edt, np.ones(vol.shape, np.uint8), vol, 2, 1.0, 0, 0)[0])
  for kind, w in (("int_ties", 1.0), ("above_2_24", 3.0), ("real", 0.7)):
    for labeling in ("runs", "single_rows"):
      shape = (300, 4, 8)
      lab = ec.labels(rng, labeling, shape, 2, np.uint16)
      out.append(run_pass(edt, lab, ec.profile(rng, kind, shape), 2, w, 1, 0, SQRT)[0])
  vor = np.asfortranarray(rng.integers(1, 4, (40, 36, 300)).repeat(3, axis=2)[:, :, :300].astype(np.uint32))
  out.append(edt.edtsq(vor, anisotropy=(4.0, 4.0, 40.0)))
  out.append(edt.sdf(vor, anisotropy=(1.0, 1.0, 1.0), black_border=True))
  return out


def test_ab_switches_do_not_change_results(edt, tmp_path):
  base = battery(edt)
  script = ("import sys, numpy as np; sys.path[:0] = [%r, %r]; import edt_b200, test_envelope_gpu as t; "
            "np.savez(sys.argv[1], *t.battery(edt_b200))") % (ROOT, HERE)
  for env in ({"EDTB200_NO_INT_HULL": "1"}, {"EDTB200_TILE_CTAS": "2"}, {"EDTB200_TILE_CTAS": "3"}):
    out = tmp_path / ("%s.npz" % "_".join("%s%s" % kv for kv in env.items()))
    proc = subprocess.run([sys.executable, "-c", script, str(out)], env=dict(os.environ, **env),
                          capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stderr[-2000:]
    z = np.load(out)
    for i, want in enumerate(base):
      assert np.array_equal(z["arr_%d" % i], want, equal_nan=True), (env, i)


def reachable():
  """Every variant launch_later / launch_tile can pick, per label width."""
  combos = set()
  for b in WIDTHS:
    for epi in (0, 1):
      for ih in (0, 1):
        combos.add((b, "tile", 32, 1, 1, 3, ih, epi, 0))
        for ctas in (2, 3):
          combos.add((b, "tile", 32, 1, 0, ctas, ih, epi, 0))
      for wide in (0, 1):
        combos.add((b, "tile", 32, 0, wide, 3, 0, epi, 0))
      for tx in (16, 8):
        for tma in (0, 1):
          combos.add((b, "tile", tx, tma, 1, 3, 0, epi, 0))
      for dbl in (0, 1):
        combos.add((b, "long", 0, 0, 0, 0, 0, epi, dbl))
  return combos


@pytest.fixture(autouse=True)
def _record_run(request):
  yield
  RAN.add(request.node.name)


RAN = set()
PRODUCERS = {"test_pass_profiles_vs_oracle[%d]" % b for b in WIDTHS} | {"test_pass_2_and_3_ctas_with_both_hulls"}


def test_every_reachable_variant_was_run():
  """The variants the tests above reached, against the reachable set.  Meaningful only after the
  tests that produce the variants have run in this process (the file's order); skipped otherwise."""
  if not PRODUCERS <= RAN:
    pytest.skip("the variant-producing tests of this file did not run before this one: %s" % sorted(PRODUCERS - RAN))
  want = reachable()
  fields = ("bytes", "kernel", "tx", "tma", "wide", "ctas", "int_hull", "epilogue", "all_double")
  print("\nlater-axis variants run (%d of %d reachable):" % (len(HIT & want), len(want)))
  print("  " + " ".join("%8s" % f for f in fields))
  for row in sorted(HIT, key=repr):
    print("  " + " ".join("%8s" % v for v in row))
  assert not HIT - want, sorted(HIT - want, key=repr)
  assert not want - HIT, sorted(want - HIT, key=repr)
