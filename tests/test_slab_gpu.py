"""GPU tests (-m gpu) of the Z-slab split's face kernels on ONE device: every rank of a split is
simulated in this process on cuda:0.

  * edtb200_slab_face_runs and edtb200_slab_face_fixup against the numpy restatements of
    tests/slab_cases.py, bit for bit, verdicts included;
  * the NCCL path of distributed.slab_transform step by step (per-axis passes, face runs, halo
    planes, Z pass with open inner faces, low then high face fix-up) against the oracle of the
    whole volume wherever the verdict is clean, and against the restatement's verdict;
  * the fused step edtb200_slab_step, each rank with its own zero-filled staging buffer.  Before
    each step every flag word is preset to the step, every rank runs once to publish its faces
    (those results are discarded), then every rank runs again and those results are compared.
    No kernel waits on a flag that nothing raises, and everything runs on one stream.
  * the three defect cases of slab_cases (double-rounding tie across a face, a walk stopping on a
    rounded tie far from the face, two faces walking the same run) through both fix-up kernels.
"""
import zlib

import numpy as np
import pytest
import torch

import envelope_cases as ec
import slab_cases as sc

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
TORCH = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}
NUMPY = {1: np.uint8, 2: np.int16, 4: np.int32, 8: np.int64}
FNS = {(False, False): "edtsq", (True, False): "edt", (False, True): "sdfsq", (True, True): "sdf"}
HALOS = (1, 2, 31, 32, 33, 127, 128, 129, 254)


@pytest.fixture(scope="module")
def passes(edt):
  from edt_b200 import distributed as ed
  return ed.CudaPasses(DEV)


def cuda_labels(lab):
  lab = np.ascontiguousarray(lab)
  nbytes = lab.dtype.itemsize
  return torch.from_numpy(lab.view(NUMPY[nbytes])).to(DEV)


def wide_labels(rng, shape, nbytes, halo):
  """Labels whose z runs are about `halo` long, from a table of values that differ only in their
  top bits, so that a comparison of fewer bytes than the label width shows."""
  top = 1 << (8 * nbytes - 2)
  table = np.array([0, top, top | 1, 1, 2 * top], dtype=np.uint64).astype(NUMPY[nbytes])
  run = np.cumsum(rng.random(shape) < 1.0 / (halo + 1), axis=0)       # run lengths of mean halo + 1
  idx = (run + rng.integers(0, 5, shape[1:])) % 5                     # adjacent runs differ
  idx = np.where(rng.random(shape[1:]) < 0.3, idx[0], idx)          # some lines are one run
  return np.ascontiguousarray(table[idx])


@pytest.mark.parametrize("nbytes", [1, 2, 4, 8])
def test_face_runs_vs_restatement(passes, nbytes):
  rng = np.random.default_rng(40 + nbytes)
  for halo in HALOS:
    for nz in sorted({1, 2, halo, halo + 1, halo + 2, 2 * halo + 5}):
      lab = wide_labels(rng, (nz, 3, 95), nbytes, halo)
      lt = cuda_labels(lab)
      for high_face in (0, 1):
        for signed in (False, True):
          overflow = torch.zeros(1, dtype=torch.int32, device=DEV)
          got = passes.face_runs(lt, high_face, halo, signed, overflow).cpu().numpy()
          want, want_over = sc.face_runs(lab, high_face, halo, signed)
          assert np.array_equal(got, want), (nbytes, halo, nz, high_face, signed, np.argwhere(got != want)[:3])
          assert bool(overflow.item()) == want_over, (nbytes, halo, nz, high_face, signed)


def run_fixup(passes, lab, z, high_face, halo, wz, sqrt, signed, nb_label, nb_m, nb_f):
  """edtb200_slab_face_fixup on copies of the arrays; returns (result, inexact)."""
  f = torch.from_numpy(np.ascontiguousarray(z, dtype=np.float32)).to(DEV)
  inexact = torch.zeros(1, dtype=torch.int32, device=DEV)
  passes.face_fixup(cuda_labels(lab), f, high_face, halo, wz, sqrt, signed, cuda_labels(nb_label),
                    torch.from_numpy(np.ascontiguousarray(nb_m)).to(DEV),
                    torch.from_numpy(np.ascontiguousarray(nb_f, dtype=np.float32)).to(DEV), inexact)
  return f.cpu().numpy(), bool(inexact.item())


def check_fixup(passes, lab, z, high_face, halo, wz, sqrt, signed, nb_label, nb_m, nb_f, what):
  got, got_inexact = run_fixup(passes, lab, z, high_face, halo, wz, sqrt, signed, nb_label, nb_m, nb_f)
  want = np.array(z, dtype=np.float32)
  want_inexact = sc.face_fixup(lab, want, high_face, halo, wz, sqrt, signed, nb_label, nb_m, nb_f)
  if not np.array_equal(got, want, equal_nan=True):
    bad = np.argwhere(got != want)
    first = tuple(bad[0])
    raise AssertionError("%s: %d voxels differ; first at %s: got %r want %r (input %r)" % (
      what, len(bad), first, got[first], want[first], z[first]))
  assert got_inexact == want_inexact, (what, got_inexact, want_inexact)
  return got, got_inexact


@pytest.mark.parametrize("kind", ec.PROFILES)
def test_face_fixup_profiles_vs_restatement(passes, kind):
  """Arbitrary float32 samples as the slab's Z-pass values and as the neighbour's rows, neighbour
  runs of every length up to halo + 1, including more than 32 and more than 128 rows within reach
  of the face values (the site caches of the two fix-up kernels)."""
  rng = np.random.default_rng(zlib.crc32(kind.encode()))
  k = 0
  for halo in (1, 2, 33, 130, 254):
    nz = 40 if halo > 100 else 70
    shape = (nz, 3, 11)
    for nbytes in (1, 2, 4, 8):
      k += 1
      lab = wide_labels(rng, shape, nbytes, 6)
      z = np.abs(ec.profile(rng, kind, shape))
      nb_f = ec.profile(rng, kind, (halo,) + shape[1:])
      other = rng.random(shape[1:]) >= 0.8         # lines whose neighbour label differs at the face
      nb_m = rng.integers(1, halo + 2, shape[1:]).astype(np.uint8)
      nb_m[0, :3] = halo                            # every neighbour row of the run, but it ends there
      nb_m[1, :3] = halo + 1                        # the run goes on behind the halo
      for wz in ((1.0, 3.0) if kind in ("int_ties", "above_2_24") else (1.0, 0.7, sc.TIE_W[0])):
        for sqrt, signed in ((False, False), (True, (k % 2) == 1)):
          zz = np.sqrt(z) if sqrt else z
          if signed:
            zz = np.where(lab == 0, -zz, zz)
          for high_face in (0, 1):
            nb_label = np.where(other, lab[nz // 2], lab[-1 if high_face else 0])
            check_fixup(passes, lab, zz, high_face, halo, wz, sqrt, signed, nb_label, nb_m, nb_f,
                        (kind, halo, nbytes, wz, sqrt, signed, high_face))


def nccl_split(passes, vol, depths, w, bb, sqrt, signed, halo, restate=True):
  """The NCCL path of slab_transform on one device, every rank in turn.  Returns the stitched
  result, its verdict, and (with `restate`) the restatement's result and verdict from the same
  Z-pass outputs."""
  n = len(depths)
  starts = np.cumsum([0] + list(depths[:-1]))
  labs = [cuda_labels(vol[s:s + d]) for s, d in zip(starts, depths)]
  fs = [passes.empty_f32(tuple(l.shape)) for l in labs]
  for lt, f in zip(labs, fs):
    passes.pass_first(lt, f, w[2], bb, signed)
    passes.pass_later(lt, f, 1, w[1], bb, bb)
  overflow = torch.zeros(1, dtype=torch.int32, device=DEV)
  m = [{face: passes.face_runs(lt, face, halo, signed, overflow) for face in (0, 1)} for lt in labs]
  planes = [{0: f[:halo].clone(), 1: f[-halo:].clone()} for f in fs]
  for i, (lt, f) in enumerate(zip(labs, fs)):
    passes.pass_later(lt, f, 2, w[0], bb and i == 0, bb and i == n - 1, sqrt=sqrt, negate=signed)
  zpass = [f.cpu().numpy() for f in fs]
  inexact = torch.zeros(1, dtype=torch.int32, device=DEV)
  restated, restated_inexact = [], False
  for i, (lt, f) in enumerate(zip(labs, fs)):
    z = zpass[i].copy()
    for high_face, nb in ((0, i - 1), (1, i + 1)):
      if 0 <= nb < n:
        nb_label = labs[nb][-1 if high_face == 0 else 0].contiguous()
        nb_m, nb_f = m[nb][1 - high_face], planes[nb][1 - high_face]
        passes.face_fixup(lt, f, high_face, halo, w[0], sqrt, signed, nb_label, nb_m, nb_f, inexact)
        if restate:
          restated_inexact |= sc.face_fixup(vol[starts[i]:starts[i] + depths[i]], z, high_face, halo, w[0], sqrt,
                                            signed, nb_label.cpu().numpy(), nb_m.cpu().numpy(), nb_f.cpu().numpy())
    restated.append(z)
  got = torch.cat(fs).cpu().numpy()
  return got, bool(inexact.item()), np.concatenate(restated) if restate else None, restated_inexact


def fused_split(passes, vols, depths, w, bb, sqrt, signed, halo):
  """edtb200_slab_step for every rank on cuda:0, steps 1, 2, 3, ... one volume each (see the module
  docstring).  Returns [(stitched result, status of every rank)] per volume."""
  n = len(depths)
  sy, sx = vols[0].shape[1:]
  nbytes = vols[0].dtype.itemsize
  L = sc.slab_stage_layout(sy * sx, nbytes, halo)
  bufs = [torch.zeros(L["total_bytes"], dtype=torch.uint8, device=DEV) for _ in range(n)]
  starts = np.cumsum([0] + list(depths[:-1]))
  out = []
  for step, vol in enumerate(vols, start=1):
    labs = [cuda_labels(vol[s:s + d]) for s, d in zip(starts, depths)]
    fs = [passes.empty_f32(tuple(l.shape)) for l in labs]
    status = [torch.zeros(1, dtype=torch.int32, device=DEV) for _ in range(n)]
    for b in bufs:
      for key in ("flag_from_lo", "flag_from_hi"):
        b[L[key]:L[key] + 8].view(torch.int64).fill_(step)
    for publish in (True, False):
      for i in range(n):
        passes.slab_step(labs[i], fs[i], (w[2], w[1], w[0]), bb, i > 0, i < n - 1, sqrt, signed, halo,
                         bufs[i].data_ptr(), bufs[i - 1].data_ptr() if i > 0 else 0,
                         bufs[i + 1].data_ptr() if i < n - 1 else 0, step, status[i])
      if publish:
        for s in status:
          s.zero_()
    out.append((torch.cat(fs).cpu().numpy(), [int(s.item()) for s in status]))
  return out


def expect_equal(got, want, what):
  if not np.array_equal(got, want, equal_nan=True):
    bad = np.argwhere(got != want)
    first = tuple(bad[0])
    raise AssertionError("%s: %d voxels differ; first at %s: got %r want %r" % (
      what, len(bad), first, got[first], want[first]))


WEIGHTS = ((1.0, 1.0, 1.0), (3.0, 2.0, 1.0), (1.3, 0.7, 2.1), sc.TIE_W)
SPLITS = ((11, 9), (7, 12, 6), (5, 9, 6, 7))


@pytest.mark.parametrize("kind", ["iid", "blocks", "runs", "sparse"])
def test_nccl_split_vs_oracle(passes, oracle, kind):
  rng = np.random.default_rng(zlib.crc32(kind.encode()))
  clean = 0
  for depths in SPLITS:
    vol = sc.random_volume(rng, kind, (sum(depths), 9, 13))
    for w in WEIGHTS:
      for (sqrt, signed), name in FNS.items():
        for bb in (False, True):
          what = (kind, depths, w, name, bb)
          got, inexact, restated, restated_inexact = nccl_split(passes, vol, depths, w, bb, sqrt, signed, 2)
          expect_equal(got, restated, what)
          assert inexact == restated_inexact, what
          if not inexact:
            clean += 1
            expect_equal(got, getattr(oracle, name)(vol, anisotropy=w, black_border=bb), what)
  assert clean >= 10, clean                 # the sparse volumes mostly need a deeper halo


def test_nccl_split_large_vs_whole_volume(passes, edt):
  """A 150 x 64 x 70 volume of runs and blocks in 3 and 4 uneven slabs, halo 8, against edt_cuda
  on the whole volume."""
  rng = np.random.default_rng(77)
  vol = sc.random_volume(rng, "blocks", (150, 64, 70))
  vol[40:90] = sc.random_volume(rng, "runs", (50, 64, 70))
  whole = cuda_labels(vol)
  clean = 0
  for depths in ((50, 61, 39), (30, 45, 40, 35)):
    for w, bb, sqrt, signed in (((1.0, 1.0, 1.0), False, False, False), ((3.0, 1.0, 2.0), True, True, True),
                                (sc.TIE_W, False, True, False)):
      got, inexact, _, _ = nccl_split(passes, vol, depths, w, bb, sqrt, signed, 8, restate=False)
      what = (depths, w, bb, sqrt, signed)
      if not inexact:
        clean += 1
        want = edt.edt_cuda(whole, w, bb, sqrt=sqrt, signed=signed).cpu().numpy()
        expect_equal(got, want, what)
  assert clean >= 2, clean


@pytest.mark.parametrize("nbytes", [1, 2, 4, 8])
def test_fused_step_vs_nccl_split(passes, oracle, nbytes):
  """edtb200_slab_step at steps 1, 2, 3 on different volumes (a wrong staging-set parity reads the
  previous step's faces): bit-equal to the NCCL path, the same verdict, never a time-out."""
  rng = np.random.default_rng(90 + nbytes)
  for depths, halo in (((11, 9), 2), ((7, 12, 6), 3), ((5, 9, 6, 7), 4), ((40, 38, 45), 33)):
    kinds = ("blocks", "runs", "iid")
    vols = [sc.random_volume(rng, k, (sum(depths), 6, 37), NUMPY[nbytes]) for k in kinds]
    for w, bb, sqrt, signed in (((1.0, 1.0, 1.0), False, False, False), ((3.0, 2.0, 1.0), True, True, True),
                                ((1.3, 0.7, 2.1), False, False, True), (sc.TIE_W, True, True, False)):
      fused = fused_split(passes, vols, depths, w, bb, sqrt, signed, halo)
      for vol, (got, status) in zip(vols, fused):
        what = (nbytes, depths, halo, w, bb, sqrt, signed)
        want, inexact, _, _ = nccl_split(passes, vol, depths, w, bb, sqrt, signed, halo, restate=False)
        assert all(s & 2 == 0 for s in status), (what, status)
        assert any(s & 1 for s in status) == inexact, (what, status, inexact)
        expect_equal(got, want, what)
        if not inexact:
          expect_equal(got, getattr(oracle, FNS[(sqrt, signed)])(vol, anisotropy=w, black_border=bb), what)


def test_reference_readout_keeps_earlier_vertex(passes, oracle, edt):
  """slab_cases.readout_volume: the reference keeps the earlier of two hull vertices on a row where
  their rounded intersection falls exactly, although the later one is lower.  The whole-volume
  transform on the GPU and a split whose face separates the two sites (both fix-up kernels, and
  the restatement) all give the least candidate: one ulp below the reference, at those voxels only."""
  vol, depths, w = sc.readout_volume(), sc.READOUT_DEPTHS, sc.TIE_W
  want = oracle.sdfsq(vol, anisotropy=w)
  whole = edt.edt_cuda(cuda_labels(vol), w, False, signed=True).cpu().numpy()
  got, inexact, restated, restated_inexact = nccl_split(passes, vol, depths, w, False, False, True, 2)
  assert not inexact and not restated_inexact
  expect_equal(got, restated, "nccl")
  expect_equal(got, whole, "nccl vs whole volume")
  (fused, status), = fused_split(passes, [vol], depths, w, False, False, True, 2)
  assert status == [0] * len(depths), status
  expect_equal(fused, restated, "fused")
  bad = {tuple(int(i) for i in p) for p in np.argwhere(got != want)}
  assert bad == set(sc.READOUT_VOXELS), bad
  for p in sc.READOUT_VOXELS:
    assert float(got[p]) == -16.005199432373047 and float(want[p]) == -16.00520133972168, p


def test_tie_across_face(passes, oracle):
  """The double-rounding tie behind a face: both fix-up kernels give the reference's
  16.005199432373047, not the fused multiply-add's 16.00520133972168."""
  for depths in ((3, 6), (3, 6, 3)):
    lab, w = sc.tie_volume(depths)
    want = oracle.edtsq(lab, anisotropy=w)
    row = depths[0] + 2
    got, inexact, _, _ = nccl_split(passes, lab, depths, w, False, False, False, 2)
    assert not inexact and float(got[row, 0, 1]) == 16.005199432373047, ("nccl", depths, float(got[row, 0, 1]))
    expect_equal(got, want, ("nccl", depths))
    (fused, status), = fused_split(passes, [lab], depths, w, False, False, False, 2)
    assert status == [0] * len(depths) and float(fused[row, 0, 1]) == 16.005199432373047, ("fused", depths, status)
    expect_equal(fused, want, ("fused", depths))


def test_stop_trap(passes, oracle):
  """A rounded tie 5217 rows behind the face, a strictly lower row after it: neither fix-up may
  stop its walk on the tie."""
  for depths in ((sc.TRAP_DEPTH, sc.TRAP_DEPTH), (100, sc.TRAP_DEPTH, sc.TRAP_DEPTH)):
    lab, w, (_, _, low_row) = sc.stop_trap(depths)
    want = oracle.edtsq(lab, anisotropy=w)
    for halo in (2, 8):
      got, inexact, _, _ = nccl_split(passes, lab, depths, w, False, False, False, halo)
      assert not inexact and got[low_row, 0, 1] == want[low_row, 0, 1], ("nccl", depths, halo, got[low_row, 0, 1])
      expect_equal(got, want, ("nccl", depths, halo))
      (fused, status), = fused_split(passes, [lab], depths, w, False, False, False, halo)
      assert status == [0] * len(depths), status
      expect_equal(fused, want, ("fused", depths, halo))


@pytest.mark.parametrize("nbytes", [1, 4])
def test_spanning_run_of_a_middle_slab(passes, oracle, nbytes):
  """A run through the whole middle slab, walked from both faces over every row: the result must be
  the lesser of the two walks on every row (the oracle's), in both fix-up kernels.  On a plane of
  512 x 300 lines, so that the fused kernel runs many blocks."""
  for shape in ((14, 3, 4), (14, 300, 512)):
    lab = sc.span_volume(shape).astype(NUMPY[nbytes])
    for w, sqrt, signed in (((1.0, 1.0, 1.0), False, False), ((2.0, 1.0, 1.0), True, True)):
      want = getattr(oracle, FNS[(sqrt, signed)])(lab, anisotropy=w)
      got, inexact, restated, _ = nccl_split(passes, lab, (5, 5, 4), w, False, sqrt, signed, 2,
                                             restate=shape[1] == 3)
      assert not inexact
      expect_equal(got, want, ("nccl", shape, w))
      (fused, status), = fused_split(passes, [lab], (5, 5, 4), w, False, sqrt, signed, 2)
      assert status == [0, 0, 0], status
      expect_equal(fused, want, ("fused", shape, w))
