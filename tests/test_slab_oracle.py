"""CPU tests of the Z-slab split's restatements (tests/slab_cases.py): the staging layout against
the library, the fix-up restatement against the oracle of the whole volume, and proof that each
of the three defect cases is a real trap -- a fix-up with the fused arithmetic, with a walk that
stops on a rounded tie, or with two faces racing over the same rows gives a different result.
"""
import zlib

import numpy as np
import pytest

import slab_cases as sc

FNS = {(False, False): "edtsq", (True, False): "edt", (False, True): "sdfsq", (True, True): "sdf"}


def test_stage_layout_matches_library(edt):
  lib = edt._lib()
  for sx, sy in ((1, 1), (7, 3), (64, 64), (70, 54), (512, 512), (1000, 3)):
    for label_bytes in (1, 2, 4, 8):
      for halo in (1, 2, 8, 31, 32, 33, 128, 254):
        L = sc.slab_stage_layout(sx * sy, label_bytes, halo)
        assert lib.edtb200_slab_stage_bytes(sx, sy, label_bytes, halo) == L["total_bytes"], (sx, sy, label_bytes, halo)
        assert L["flag_from_lo"] == 2 * L["set_bytes"] and L["counter"] == L["flag_from_lo"] + 128
        assert all(L[k] % 256 == 0 for k in ("f_lo", "f_hi", "lab_lo", "lab_hi", "m_lo", "m_hi", "set_bytes"))
  assert lib.edtb200_slab_stage_bytes(4, 4, 3, 8) == -1 and lib.edtb200_slab_stage_bytes(4, 4, 4, 255) == -1


def test_face_runs_restatement():
  lab = np.zeros((6, 1, 5), np.int32)
  lab[:, 0, 0] = (1, 1, 1, 2, 2, 2)     # 3 rows from each face
  lab[:, 0, 1] = 4                       # spans the slab
  lab[:, 0, 2] = (0, 0, 5, 5, 5, 5)     # background at the low face: 2 rows, 4 at the high face
  lab[:, 0, 3] = (6, 7, 6, 7, 6, 7)
  runs = {0: (3, 6, 2, 1, 6), 1: (3, 6, 4, 1, 6)}        # true run lengths per face (column 4: background)
  for halo in (1, 2, 3, 4, 5, 6, 8):
    for high_face, lengths in runs.items():
      m, o = sc.face_runs(lab, high_face, halo, False)
      assert m[0].tolist() == [v if v <= halo and v < 6 else halo + 1 for v in lengths], (halo, high_face, m)
      assert o                                            # column 1 always spans the slab
  # a background run spanning the slab raises the flag only when background is a label (signed)
  bg = np.zeros((4, 1, 1), np.int32)
  assert sc.face_runs(bg, 0, 2, False) == (np.full((1, 1), 3, np.uint8), False)
  assert sc.face_runs(bg, 0, 2, True)[1]


@pytest.mark.parametrize("depths", [(6, 7), (5, 4, 6), (3, 5, 4, 4)])
@pytest.mark.parametrize("kind", ["iid", "blocks", "runs", "sparse"])
def test_restated_split_matches_whole_volume(oracle, kind, depths):
  """Where the restated fix-up's verdict is clean its stitched result is the oracle's, for all four
  transforms, with and without a black border, at integer and non-integer weights."""
  rng = np.random.default_rng(zlib.crc32(repr((kind, depths)).encode()))
  vol = sc.random_volume(rng, kind, (sum(depths), 5, 6))
  clean = 0
  for w in ((1.0, 1.0, 1.0), (3.0, 2.0, 1.0), (1.3, 0.7, 2.1), sc.TIE_W):
    for (sqrt, signed), name in FNS.items():
      for bb in (False, True):
        got, inexact = sc.split_restated(oracle, vol, depths, w, bb, sqrt, signed, 2)
        if not inexact:
          clean += 1
          want = getattr(oracle, name)(vol, anisotropy=w, black_border=bb)
          assert np.array_equal(got, want), (w, name, bb, np.argwhere(got != want)[:3])
  assert clean > 0


def test_reference_readout_keeps_earlier_vertex(oracle):
  """The one known way a split with a clean verdict differs from the reference (README, DESIGN §8):
  the reference's read-out keeps the earlier of two hull vertices on a row where their rounded
  intersection falls exactly, even when the later one is lower.  When a slab face separates the
  two sites the fix-up compares them as values.  The split then gives the least candidate, which
  is what the brute force of the definition gives too (and the single-GPU transform, see
  test_slab_gpu), one ulp below the reference, and only there."""
  vol, depths, w = sc.readout_volume(), sc.READOUT_DEPTHS, sc.TIE_W
  want = oracle.sdfsq(vol, anisotropy=w)
  got, inexact = sc.split_restated(oracle, vol, depths, w, False, False, True, 2)
  assert not inexact
  bad = {tuple(int(i) for i in p) for p in np.argwhere(got != want)}
  assert bad == set(sc.READOUT_VOXELS), bad
  for p in sc.READOUT_VOXELS:
    assert float(got[p]) == -16.005199432373047 and float(want[p]) == -16.00520133972168, p
  # the two sites and the reference's intersection of them
  w2 = np.float64(np.float32(np.float32(w[0]) ** 2))
  xy = sc.slab_xy(oracle, vol, w, False, True)
  h19, h25 = np.float64(xy[19, 0, 3]), np.float64(xy[25, 0, 3])
  assert h25 < h19 and (h25 - h19 + 6 * w2 * 44) / (12 * w2) == 22.0
  # the brute force of the Z pass over the whole volume (least double sum per voxel) agrees with the split
  import envelope_cases as ec
  brute = ec.brute_pass(vol, xy, 2, w[0], False, False)
  brute[vol == 0] *= -1.0
  assert np.array_equal(got, brute)


def test_tie_across_face_is_a_trap(oracle):
  """The double-rounding tie three rows behind a slab face: the restatement with the reference's
  double sum equals the oracle of the whole volume, the fused form (one rounding of the exact sum)
  does not."""
  for depths in ((3, 6), (3, 6, 3)):
    lab, w = sc.tie_volume(depths)
    want = oracle.edtsq(lab, anisotropy=w)
    assert float(want[depths[0] + 2, 0, 1]) == 16.005199432373047
    double, inexact = sc.split_restated(oracle, lab, depths, w, False, False, False, 2, arith="double")
    assert not inexact and np.array_equal(double, want), depths
    fused, _ = sc.split_restated(oracle, lab, depths, w, False, False, False, 2, arith="fused")
    assert float(fused[depths[0] + 2, 0, 1]) == 16.00520133972168, depths


def test_stop_trap_is_a_trap(oracle):
  """More than 4096 rows behind the face the border candidate and the in-slab one round to the
  same float32 while the exact border value is lower, and a row later the border's rounds strictly
  lower: a walk that stops on the rounded tie leaves that row wrong, the strict stop does not."""
  for depths in ((sc.TRAP_DEPTH, sc.TRAP_DEPTH), (100, sc.TRAP_DEPTH, sc.TRAP_DEPTH)):
    lab, w, (face, tie_row, low_row) = sc.stop_trap(depths)
    assert tie_row - face > 4096
    want = oracle.edtsq(lab, anisotropy=w)
    w2 = np.float64(np.float32(np.float32(w[0]) ** 2))
    h = np.float64(np.float32(np.float32(w[2]) ** 2))
    for row, rel in ((tie_row, "=="), (low_row, "<")):
      j = row - face
      outside, inside = np.float32(w2 * (j + 1) ** 2), np.float32(w2 * j * j + h)
      exact_gap = (sc.Fraction(float(w2)) * (j + 1) ** 2) - (sc.Fraction(float(w2)) * j * j + sc.Fraction(float(h)))
      assert exact_gap < 0, row
      assert (outside == inside) if rel == "==" else (outside < inside), (row, outside, inside)
      assert want[row, 0, 1] == min(outside, inside)
    strict, inexact = sc.split_restated(oracle, lab, depths, w, False, False, False, 2, stop="strict")
    assert not inexact and np.array_equal(strict, want), depths
    tie, _ = sc.split_restated(oracle, lab, depths, w, False, False, False, 2, stop="tie")
    bad = np.argwhere(tie != want)
    assert len(bad) and tuple(bad[0]) == (low_row, 0, 1), (depths, bad[:3])


@pytest.mark.parametrize("sqrt,signed", [(False, False), (True, True)])
def test_spanning_run_faces_overlap(oracle, sqrt, signed):
  """The middle slab of (5, 5, 4) has only +inf Z-pass values on the run through it; folding in its
  low face alone and its high face alone both write every row, with different values, so two walks
  racing over that line would leave whichever stored last."""
  lab = sc.span_volume()
  depths, halo = (5, 5, 4), 2
  xy = [sc.slab_xy(oracle, lab[s:s + d], (1.0, 1.0, 1.0), False, signed) for s, d in ((0, 5), (5, 5), (10, 4))]
  mid = lab[5:10]
  z = sc.slab_z(oracle, mid, xy[1], 1.0, False, False, sqrt, signed)
  assert np.all(np.isinf(z))
  faces = []
  for high_face, nb, nlab in ((0, 0, lab[0:5]), (1, 2, lab[10:14])):
    nb_m, _ = sc.face_runs(nlab, 1 - high_face, halo, signed)
    assert np.all(nb_m == 2)
    nb_f = xy[nb][-halo:] if high_face == 0 else xy[nb][:halo]
    alone = z.copy()
    assert not sc.face_fixup(mid, alone, high_face, halo, 1.0, sqrt, signed, lab[4 if high_face == 0 else 10],
                             nb_m, nb_f)
    faces.append(alone)
  lo, hi = faces
  assert np.all(np.isfinite(lo)) and np.all(np.isfinite(hi))
  assert np.any(lo > hi) and np.any(hi > lo)          # whichever walk stores last, some row is wrong
  want = getattr(oracle, FNS[(sqrt, signed)])(lab)
  got, inexact = sc.split_restated(oracle, lab, depths, (1.0, 1.0, 1.0), False, sqrt, signed, halo)
  assert not inexact and np.array_equal(got, want)
  assert np.array_equal(got[5:10], np.minimum(lo, hi))
