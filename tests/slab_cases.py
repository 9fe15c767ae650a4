"""Inputs and plain restatements for the tests of the Z-slab split (tests/test_slab_*.py and the
gloo tests in tests/test_distributed.py), and `OraclePasses`, the stand-in for
distributed.CudaPasses that those gloo tests hand to slab_transform.

The Z-slab split runs the third-axis pass of every slab with its inner faces open and then folds
the neighbour's rows of every run that crosses a face into the slab (face_runs_kernel and
face_fixup_kernel, slab_stage_kernel and slab_fixup_kernel, all in csrc/edt_slab.cuh).  This module restates those two steps in numpy on C-ordered (z, y, x) arrays,
restates the byte layout of the fused step's staging buffer, and builds seeded volumes, among them
three that are traps for a fix-up that is subtly wrong:

  tie_volume     a double-rounding tie (the tie2d pattern of tests/golden/rounding_edges.npz turned
                 into z) lying across a slab face: only the reference's double sum rounded once
                 gives the reference's value;
  stop_trap      a run whose outside and inside candidates round to the same float32 at a row
                 more than 4096 rows from the face while a later row rounds strictly lower: a walk
                 that stops on a rounded tie misses it;
  span_volume    a run that spans a middle slab with no site in it, and ends within the halo on
                 both sides: both faces' walks write every row of that slab.
"""
from fractions import Fraction

import numpy as np
import torch

TIE_W = (float(np.float32(1.333549976348877)), 1.0, 2.0 ** -26)        # (w_z, w_y, w_x)
# stop_trap: with w_z^2 = 1.5390757 and an in-plane height of w_x^2 = 16064.0 at the face row, the
# candidates of row 5217 tie in float32 while the exact outside one is lower, and row 5218 rounds
# strictly lower (found by search; test_stop_trap_is_a_trap checks it)
TRAP_W = (1.2405948638916016, 1.0, 126.74388885498047)
TRAP_DEPTH = 6000
TRAP_ROWS = (5217, 5218)                      # (the rounded tie, the row after it that is lower)


# ---------------------------------------------------------------------------------------------
# restatements
# ---------------------------------------------------------------------------------------------

def face_runs(lab, high_face, halo, signed):
  """face_runs_kernel: (m, overflow) for C-ordered labels (nz, sy, sx).  m[y, x] = length of the run
  of equal labels that touches the face, capped at halo + 1 ("longer than the halo, or spanning
  the slab"); overflow is True when that happens to a foreground run (any run when signed)."""
  lab = np.asarray(lab)
  nz = lab.shape[0]
  rows = range(nz - 1, -1, -1) if high_face else range(nz)
  face = lab[nz - 1 if high_face else 0]
  m = np.zeros(face.shape, dtype=np.int64)
  alive = np.ones(face.shape, dtype=bool)
  for k, r in enumerate(rows):
    if k > halo:
      break
    alive &= lab[r] == face
    m += alive
  too_long = (m > halo) | (m >= nz)
  m[too_long] = halo + 1
  overflow = bool(np.any(too_long & ((face != 0) | bool(signed))))
  return m.astype(np.uint8), overflow


def round_f32(x):
  """A Fraction (or +inf) rounded ONCE to the nearest float32, ties to even."""
  if x == np.inf:
    return np.float32(np.inf)
  near = np.float32(float(x))
  cands = (np.nextafter(near, np.float32(-np.inf)), near, np.nextafter(near, np.float32(np.inf)))
  return min(cands, key=lambda c: (abs(Fraction(float(c)) - x), int(c.view(np.uint32)) & 1))


def _candidate(w2, d, height, arith):
  """w2 * d^2 + height as float32: the double sum rounded to float32 (the reference), or the exact
  sum rounded once (what a fused multiply-add gives)."""
  if arith == "double":
    return np.float32(np.float64(w2) * d * d + np.float64(height))
  if not np.isfinite(height):
    return np.float32(np.inf)
  return round_f32(Fraction(float(w2)) * d * d + Fraction(float(height)))


def face_fixup(lab, arr, high_face, halo, wz, sqrt, signed, nb_label, nb_m, nb_f, arith="double", stop="strict"):
  """face_fixup_kernel on numpy arrays: folds the neighbour's sites into `arr` (the slab's Z-pass
  result, float32 (nz, sy, sx), updated in place) and returns the `inexact` verdict.
  nb_label / nb_m: the neighbour's face plane of labels and its face_runs; nb_f: `halo` planes of
  the neighbour's Y-pass distances in its own z order.  arith: "double" (the double sum rounded
  once, as the reference) or "fused" (the exact sum rounded once).  stop: "strict" (the walk ends
  at the first row whose best outside candidate is strictly above the row's value, and stores only
  strictly lower values) or "tie" (it ends at the first row that does not improve)."""
  assert arith in ("double", "fused") and stop in ("strict", "tie")
  lab, nbl, nbm, nbf = np.asarray(lab), np.asarray(nb_label), np.asarray(nb_m), np.asarray(nb_f)
  nz, sy, sx = lab.shape
  w2 = np.float32(np.float32(wz) * np.float32(wz))
  inexact = False
  for y in range(sy):
    for x in range(sx):
      row0, step = (nz - 1, -1) if high_face else (0, 1)
      lab0 = lab[row0, y, x]
      if lab0 == 0 and not signed:
        continue
      m_raw = int(nbm[y, x]) if nbl[y, x] == lab0 else 0
      unseen = m_raw > halo           # the neighbour's part of the run goes on behind the halo
      m = min(m_raw, halo)
      for j in range(nz):
        r = row0 + step * j
        if j > 0 and lab[r, y, x] != lab0:
          break
        best = np.float32(np.inf) if unseen else _candidate(w2, j + 1 + m, 0.0, arith)
        for k in range(m):
          src = k if high_face else halo - 1 - k
          best = min(best, _candidate(w2, j + 1 + k, nbf[src, y, x], arith))
        if sqrt:
          best = np.sqrt(np.float32(best))
        cur = abs(arr[r, y, x])
        if unseen:
          bound = _candidate(w2, j + halo, 0.0, arith)
          if sqrt:
            bound = np.sqrt(bound)
          if not (min(best, cur) <= bound):
            inexact = True
        if (best > cur) if stop == "strict" else not (best < cur):
          break
        if best < cur:
          arr[r, y, x] = -best if (signed and lab0 == 0) else best
  return inexact


def slab_stage_layout(plane, label_bytes, halo):
  """SlabStageLayout (csrc/edt_slab.cuh): offsets of one staging set, the set size, and the flag
  words and CTA counter after both sets, every piece rounded up to 256 bytes."""
  off, L = 0, {}
  for name, nbytes in (("f_lo", halo * plane * 4), ("f_hi", halo * plane * 4), ("lab_lo", plane * label_bytes),
                       ("lab_hi", plane * label_bytes), ("m_lo", plane), ("m_hi", plane)):
    L[name] = off
    off += (nbytes + 255) // 256 * 256
  L["set_bytes"] = off
  L["flag_from_lo"] = 2 * off
  L["flag_from_hi"] = L["flag_from_lo"] + 64
  L["counter"] = L["flag_from_hi"] + 64
  L["total_bytes"] = L["counter"] + 64
  return L


# ---------------------------------------------------------------------------------------------
# the pipeline of one slab, restated on the oracle's passes (numpy, C-ordered)
# ---------------------------------------------------------------------------------------------

def slab_xy(oracle, lab, w, black_border, signed):
  """The X and Y passes of one slab as the device runs them: background is a label when signed."""
  lab = np.asarray(lab).astype(np.int64)
  shifted = lab + 1 if signed else lab
  f = oracle.pass_first(shifted, w[2], black_border)
  oracle.pass_later(lab + 1, f, 1, w[1], black_border, black_border)
  if not signed:
    f[lab == 0] = 0.0
  return f


def slab_z(oracle, lab, f, wz, border_lo, border_hi, sqrt, signed):
  """The Z pass of one slab (faces open where border_* is 0), with the store's epilogue."""
  lab = np.asarray(lab).astype(np.int64)
  out = f.copy()
  oracle.pass_later(lab + 1, out, 2, wz, border_lo, border_hi)
  if not signed:
    out[lab == 0] = 0.0
  if sqrt:
    np.sqrt(out, out=out)
  if signed:
    out[lab == 0] *= -1.0
  return out


def split_restated(oracle, vol, depths, w, black_border, sqrt, signed, halo, arith="double", stop="strict"):
  """The whole NCCL-path split of `vol` into slabs of `depths`, every step restated: returns the
  stitched result and the verdict (True = some fix-up raised `inexact`)."""
  starts = np.cumsum([0] + list(depths[:-1]))
  slabs = [vol[s:s + d] for s, d in zip(starts, depths)]
  xy = [slab_xy(oracle, s, w, black_border, signed) for s in slabs]
  n = len(slabs)
  out, inexact = [], False
  for i, (lab, f) in enumerate(zip(slabs, xy)):
    z = slab_z(oracle, lab, f, w[0], black_border and i == 0, black_border and i == n - 1, sqrt, signed)
    for high_face, nb in ((0, i - 1), (1, i + 1)):
      if nb < 0 or nb >= n:
        continue
      nlab = slabs[nb]
      nb_m, _ = face_runs(nlab, 1 - high_face, halo, signed)
      nb_label = nlab[-1 if high_face == 0 else 0]
      nb_f = xy[nb][-halo:] if high_face == 0 else xy[nb][:halo]
      inexact |= face_fixup(lab, z, high_face, halo, w[0], sqrt, signed, nb_label, nb_m, nb_f, arith, stop)
    out.append(z)
  return np.concatenate(out, axis=0), inexact


class OraclePasses:
  """Stand-in for CudaPasses: same interface, numpy arithmetic from oracle/ (tests only)."""

  def __init__(self, packed=True):
    from oracle import oracle
    self.oracle = oracle
    self.signed = False
    if not packed:                  # hide `repartition`: the transposition then slices and concatenates
      self.repartition = None

  def __getattribute__(self, name):
    value = object.__getattribute__(self, name)
    if name == "repartition" and value is None:
      raise AttributeError(name)
    return value

  def empty_f32(self, shape):
    return torch.zeros(shape, dtype=torch.float32)

  def pass_first(self, labels, f, wx, black_border, signed):
    lab = labels.numpy()
    self.signed = bool(signed)
    if signed:                      # background as an ordinary label == shift every label by one
      lab = lab.astype(np.int64) + 1
    f.copy_(torch.from_numpy(self.oracle.pass_first(lab, wx, black_border)))

  def pass_later(self, labels, f, axis, w, border_lo, border_hi, sqrt=False, negate=False):
    lab = labels.numpy().astype(np.int64)
    zero = lab == 0
    arr = f.numpy()
    self.oracle.pass_later(lab + 1, arr, axis, w, border_lo, border_hi)   # +1: every run is foreground...
    if not self.signed:
      # ...except that plain EDT keeps background at 0 (its rows hold 0 already and stay 0)
      arr[zero] = 0.0
    if sqrt:
      np.sqrt(arr, out=arr)
    if negate:
      arr[zero] *= -1.0


  # torch restatement of slab_pack_kernel (edt_slab.cuh): slab (zc, sy, row) <-> per-rank blocks
  def repartition(self, src, dst, ysplit, unpack=False):
    slab = dst if unpack else src
    zc, sy, row = slab.shape
    flat = (src if unpack else dst).reshape(-1)
    for s, c in ysplit:
      block = flat[zc * s * row:zc * (s + c) * row].view(zc, c, row)
      if unpack:
        dst[:, s:s + c, :] = block
      else:
        block.copy_(src[:, s:s + c, :])

  # the two slab-face kernels (edt_slab.cuh: face_runs_kernel, face_fixup_kernel), restated above
  def face_runs(self, labels, high_face, halo, signed, overflow, out=None):
    m, too_long = face_runs(labels.numpy(), high_face, halo, signed)
    if too_long:
      overflow[0] = 1
    return torch.from_numpy(m)

  def face_fixup(self, labels, f, high_face, halo, wz, sqrt, signed, nb_label, nb_m, nb_f, inexact):
    if face_fixup(labels.numpy(), f.numpy(), high_face, halo, wz, sqrt, signed, nb_label.numpy(),
                  nb_m.numpy(), nb_f.numpy()):
      inexact[0] = 1


# ---------------------------------------------------------------------------------------------
# volumes
# ---------------------------------------------------------------------------------------------

def random_volume(rng, kind, shape, dtype=np.int32):
  """Seeded labels: "iid" label noise, "blocks" of 5^3 voxels, z "runs" of random lengths over a
  few labels, or "sparse" background in one label (long runs, the halo's reach matters)."""
  if kind == "iid":
    vol = rng.integers(0, 4, shape)
  elif kind == "blocks":
    small = rng.integers(0, 3, tuple((s + 4) // 5 for s in shape))
    vol = np.repeat(np.repeat(np.repeat(small, 5, 0), 5, 1), 5, 2)[:shape[0], :shape[1], :shape[2]]
  elif kind == "runs":
    cuts = np.cumsum(rng.geometric(0.15, (shape[0],) + tuple(shape[1:])), axis=0)
    vol = (cuts * 7 + rng.integers(0, 3, shape)) % 5
    vol = np.where(rng.random(shape) < 0.5, np.repeat(vol[:1], shape[0], 0), vol)
  elif kind == "sparse":
    vol = np.where(rng.random(shape) < 0.02, 0, 3)
  else:
    raise ValueError(kind)
  return np.ascontiguousarray(vol.astype(dtype))


def tie_volume(depths):
  """(labels, anisotropy (w_z, w_y, w_x)): a (sum(depths), 1, 2) volume whose x = 1 line holds ONE
  site, of height w_x^2 = 2^-52, on the last row of the first slab (background beside it at
  x = 0).  Three rows further, in the second slab, the candidate w_z^2 * 9 + 2^-52 is a
  double-rounding tie.  With a third slab the run ends where it starts (a new label)."""
  nz = int(sum(depths))
  site = depths[0] - 1
  lab = np.ones((nz, 1, 2), np.int32)
  lab[site, 0, 0] = 0
  if len(depths) > 2:
    lab[depths[0] + depths[1]:] = 2
  return lab, TIE_W


def stop_trap(depths):
  """(labels, anisotropy, (face row, tie row, lower row)): a (sum(depths), 1, 2) volume whose last
  slab (TRAP_DEPTH rows) is one run at x = 1 with a single site, of height w_x^2, on its first row
  (label 3 beside it at x = 0); every slab before it holds another label, alternating, so every
  face is a run border.  Along the last slab the outside candidate w_z^2 (j + 1)^2 (the border
  at the face) and the inside one w_z^2 j^2 + w_x^2 tie in float32 at row TRAP_ROWS[0] from the
  face while the exact outside value is lower, and round strictly lower a row later."""
  assert depths[-1] == TRAP_DEPTH
  nz = int(sum(depths))
  lab = np.empty((nz, 1, 2), np.int32)
  start = nz
  for k, d in enumerate(reversed(depths)):
    lab[start - d:start] = (1, 2, 4)[0 if k == 0 else 1 + (k - 1) % 2]
    start -= d
  face = nz - depths[-1]
  lab[face, 0, 0] = 3
  return lab, TRAP_W, (face, face + TRAP_ROWS[0], face + TRAP_ROWS[1])


READOUT_DEPTHS = (5, 9, 6, 7, 6)
READOUT_VOXELS = ((22, 0, 3), (22, 0, 4))


def readout_volume():
  """A seeded 33 x 9 x 13 volume on which the reference does NOT return the least candidate, and a
  split that cuts between the two candidates does (sdfsq, tie weights, slabs READOUT_DEPTHS).
  On the line (y, x) = (0, 3) the background run 15..29 has sites at rows 19 and 25, three rows
  either side of row 22, with X-pass heights 1.09e-14 and 8.9e-16: the site at 25 is lower.  The
  reference's hull read-out computes their intersection in double as exactly 22.0 and keeps the
  earlier vertex on that row, giving 16.00520133972168; the exact least candidate rounds to
  16.005199432373047.  The slab face at row 20 lies between the two sites, so the fix-up compares
  them as values and keeps the lower one.  The same happens at (22, 0, 4)."""
  return random_volume(np.random.default_rng(105), "blocks", (33, 9, 13))


def span_volume(shape=(14, 3, 4), bg=(2, 12)):
  """One label everywhere but two background planes: split into three slabs (5, 5, 4) the middle
  slab's plane has no boundary (its Z-pass values are +inf), and the run through it ends two rows
  behind each of its faces."""
  lab = np.ones(shape, np.int32)
  for z in bg:
    lab[z] = 0
  return lab
