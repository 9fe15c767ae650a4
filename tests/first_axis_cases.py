"""Inputs of the per-pass first-axis tests (tests/test_first_axis_*.py): seeded row labelings, the
weights, what edtb200_pass_first must produce (from the oracle), and a plain statement of the pass
from its definition.

A row is a line of sx voxels along x.  For a voxel p with label l, kL is the number of steps to the
nearest voxel on its left whose label differs from l -- or to the face just before voxel 0 when the
border is on -- and kR the same to the right (the face just after voxel sx - 1); the pass gives
T[min(kL, kR)], with T[k] the float32 square of the float32 SEQUENTIAL sum of k weights
(src/edt.hpp:92-118 of the reference accumulates d[i] = d[i-1] + w), +inf when neither side has
such a voxel, and 0 for background (label 0) unless background counts as a label.
"""
import functools

import numpy as np

SQRT, SIGNED = 1, 2                  # EDTB200_SQRT, EDTB200_SIGNED (include/edt_b200.h)
FLAG_SETS = (0, SQRT, SIGNED, SQRT | SIGNED)
WIDTHS = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}

# 1 and 3 are exact in every sum; the others are not (1.333549976348877 is the float32 weight of
# the later-axis rounding ties); 1e19's square overflows to +inf from k = 2 on.
WEIGHTS = (1.0, 3.0, 0.7, 0.1, 1.333549976348877, 1e-3, 1e19)
OVERFLOW_WEIGHT = 1e19
INEXACT_WEIGHTS = (0.7, 0.1, 1.333549976348877, 1e-3)

LABELINGS = ("one_run", "runs", "single", "noise", "aligned4", "aligned32", "aligned128",
             "mostly_background", "all_background", "top_bit", "upper_half")


def _runs_to_labels(starts, n, rng, dtype, values=None):
  """Labels of a row cut into runs at `starts` (booleans, starts[0] ignored): neighbouring runs
  always differ, values from `values` (cycled) or 1..4."""
  run = np.cumsum(starts) - starts[0]
  if values is None:
    values = 1 + rng.permutation(4)
  values = np.asarray(values, dtype=np.uint64)
  return values[run % len(values)].astype(dtype)


def labeling(rng, kind, n, nbytes):
  """One row of n labels of width nbytes (see LABELINGS):
    one_run            one label over the whole row
    runs               runs of random (geometric) length
    single             every voxel a run of its own
    noise              labels 0..2 drawn per voxel (adjacent equal labels merge)
    aligned4/32/128    runs of exactly 4 / 32 / 128 voxels: label changes fall on the edges of a
                       lane's 4 voxels, a 32-bit boundary word, and a 128-voxel vector block
    mostly_background  about nine voxels in ten background, short runs between
    all_background     label 0 everywhere
    top_bit            runs that differ only in the top (sign) bit of the label
    upper_half         runs that differ only in the upper half of the label (the upper 32 bits of an
                       8-byte label)"""
  dtype = WIDTHS[nbytes]
  bits = 8 * nbytes
  pos = np.arange(n)
  if kind == "one_run":
    return np.full(n, 1 + rng.integers(0, 4), dtype)
  if kind == "runs":
    return _runs_to_labels(rng.random(n) < 1.0 / max(2, min(n, 64) // 4), n, rng, dtype)
  if kind == "single":
    return _runs_to_labels(np.ones(n, bool), n, rng, dtype)
  if kind == "noise":
    return rng.integers(0, 3, n).astype(dtype)
  if kind.startswith("aligned"):
    size = int(kind[len("aligned"):])
    return _runs_to_labels(pos % size == 0, n, rng, dtype)
  if kind == "mostly_background":
    lab = np.where(rng.random(n) < 0.1, rng.integers(1, 4, n), 0)
    return lab.astype(dtype)
  if kind == "all_background":
    return np.zeros(n, dtype)
  if kind == "top_bit":
    low = np.uint64(1 + rng.integers(0, 3))
    top = np.uint64(1) << np.uint64(bits - 1)
    return _runs_to_labels(rng.random(n) < 0.2, n, rng, dtype, values=[low, low | top])
  if kind == "upper_half":
    low = np.uint64(1 + rng.integers(0, 3))
    half = np.uint64(bits // 2)
    values = [low | (np.uint64(v) << half) for v in (0, 1, 2, 5)]
    return _runs_to_labels(rng.random(n) < 0.2, n, rng, dtype, values=values)
  raise ValueError(kind)


def rows(rng, n, nbytes):
  """Every labeling as one row of n voxels: a (len(LABELINGS), n) array."""
  return np.stack([labeling(rng, kind, n, nbytes) for kind in LABELINGS])


def relabel_background(lab):
  """lab with label 0 replaced by a value it does not hold, as uint64: background then behaves as an
  ordinary label (EDTB200_SIGNED on the first pass)."""
  lab = np.asarray(lab).astype(np.uint64)
  present = np.unique(lab)
  spare = np.setdiff1d(np.arange(1, len(present) + 2, dtype=np.uint64), present)[0]
  return np.where(lab == 0, spare, lab)


def expected_first(oracle, lab, w, border, flags):
  """What edtb200_pass_first must give for labels lab (..., sx) under ABI flags:
    0       oracle.pass_first
    SIGNED  the same after relabelling 0 to a value the labels do not hold (no sign is applied)
    SQRT    np.sqrt of it in float32."""
  lab = np.asarray(lab)
  sx = lab.shape[-1]
  if flags & SIGNED:
    lab = relabel_background(lab)
  want = oracle.pass_first(lab.reshape(1, -1, sx), w, border).reshape(lab.shape)
  if flags & SQRT:
    np.sqrt(want, out=want)
  return want


@functools.lru_cache(maxsize=None)
def step_table(w, count):
  """T[0..count): the float32 square of the float32 sequential sum of k weights (read-only)."""
  w = np.float32(w)
  t = np.empty(count, np.float32)
  a = np.float32(0.0)
  t[0] = 0.0
  with np.errstate(over="ignore"):
    for k in range(1, count):
      a = np.float32(a + w)
      t[k] = a * a
  t.flags.writeable = False
  return t


def steps(lab, border):
  """(kL, kR) per voxel of rows lab (..., sx) as int64, sx + 1 standing for "no such voxel"."""
  lab = np.asarray(lab)
  sx = lab.shape[-1]
  none = sx + 1
  p = np.arange(sx)
  differs = lab[..., 1:] != lab[..., :-1]          # voxels j - 1 and j differ, j = 1 .. sx - 1
  # nearest differing voxel on the left: j - 1 for the largest change j <= p
  left = np.where(differs, p[1:] - 1, -2)
  left = np.concatenate([np.full(lab.shape[:-1] + (1,), -2), left], axis=-1)
  left = np.maximum.accumulate(left, axis=-1)
  kl = np.where(left >= 0, p - left, p + 1 if border else none)
  # nearest differing voxel on the right: j for the smallest change j > p
  right = np.where(differs, p[1:], sx + 2)
  right = np.concatenate([right, np.full(lab.shape[:-1] + (1,), sx + 2)], axis=-1)
  right = np.minimum.accumulate(right[..., ::-1], axis=-1)[..., ::-1]
  kr = np.where(right <= sx, right - p, sx - p if border else none)
  return np.minimum(kl, none), np.minimum(kr, none)


def brute_first(lab, w, border, background_is_label=False):
  """The first-axis pass from its definition (see the module docstring)."""
  lab = np.asarray(lab)
  sx = lab.shape[-1]
  kl, kr = steps(lab, border)
  table = np.append(step_table(float(np.float32(w)), sx + 1), np.float32(np.inf))
  out = table[np.minimum(kl, kr)]
  if not background_is_label:
    out[lab == 0] = 0.0
  return out
