"""CPU checks of the first-axis test inputs (tests/first_axis_cases.py): the statement of the pass from
its definition agrees with the oracle on every labeling, label width and weight; the background-as-
label expectation is the magnitude of the oracle's sdfsq on 1-D lines; and the cases are sharp
enough that a subtly wrong kernel -- products instead of sequential sums, a missing border, a
boundary counted on the wrong voxel -- would change some expected value."""
import numpy as np
import pytest

import first_axis_cases as fc

# the row lengths of the GPU tests up to 4097 (the longer ones only add more of the same runs)
LENGTHS = (1, 2, 3, 4, 5, 31, 32, 33, 124, 127, 128, 129, 132, 252, 256, 257, 260, 508, 512, 513, 516,
           1020, 1023, 1024, 1025, 1028, 1056, 2048, 4096, 4097)


def assert_same(got, want, what):
  if not np.array_equal(got, want, equal_nan=True):
    bad = np.argwhere(got != want)
    first = tuple(bad[0])
    raise AssertionError("%s: %d voxels differ; first at %s: got %r want %r" % (
      what, len(bad), first, got[first], want[first]))


@pytest.mark.parametrize("nbytes", sorted(fc.WIDTHS))
def test_brute_first_matches_oracle(oracle, nbytes):
  rng = np.random.default_rng(10 + nbytes)
  for n in LENGTHS:
    lab = fc.rows(rng, n, nbytes)
    for w in fc.WEIGHTS:
      for border in (0, 1):
        want = oracle.pass_first(lab.reshape(1, -1, n), w, border).reshape(lab.shape)
        assert_same(fc.brute_first(lab, w, border), want, (nbytes, n, w, border))
        signed = fc.expected_first(oracle, lab, w, border, fc.SIGNED)
        assert_same(fc.brute_first(lab, w, border, background_is_label=True), signed,
                    (nbytes, n, w, border, "signed"))
        assert_same(fc.expected_first(oracle, lab, w, border, fc.SQRT), np.sqrt(want),
                    (nbytes, n, w, border, "sqrt"))


def test_labelings_have_what_they_promise():
  rng = np.random.default_rng(1)
  for nbytes, dtype in fc.WIDTHS.items():
    bits = 8 * nbytes
    for n in (128, 1024):
      lab = dict(zip(fc.LABELINGS, fc.rows(rng, n, nbytes)))
      assert all(v.dtype == dtype for v in lab.values())
      for size in (4, 32, 128):
        change = np.flatnonzero(np.diff(lab["aligned%d" % size].astype(np.uint64))) + 1
        assert np.array_equal(change, np.arange(size, n, size)), (nbytes, n, size)
      assert not lab["all_background"].any()
      assert (lab["mostly_background"] == 0).mean() > 0.8
      assert len(np.unique(lab["one_run"])) == 1 and lab["one_run"][0] != 0
      assert np.all(np.diff(lab["single"].astype(np.uint64)) != 0)
      for kind, mask in (("top_bit", 1 << (bits - 1)),
                         ("upper_half", ((1 << bits) - 1) ^ ((1 << (bits // 2)) - 1))):
        vals = [int(v) for v in np.unique(lab[kind])]
        assert len(vals) >= 2, (nbytes, kind)
        assert len({v & ~mask for v in vals}) == 1, (nbytes, kind, vals)   # equal outside the mask


@pytest.mark.parametrize("nbytes", (1, 8))
def test_signed_expectation_is_sdfsq_magnitude(oracle, nbytes):
  """On a 1-D line, background counted as a label gives every voxel its distance to the nearest voxel
  of another label, or of any label for background: |sdfsq|, whose two transforms give the same."""
  rng = np.random.default_rng(20 + nbytes)
  for n in (1, 5, 33, 129, 1024, 1025):
    for kind, line in zip(fc.LABELINGS, fc.rows(rng, n, nbytes)):
      for w in fc.WEIGHTS:
        for border in (0, 1):
          got = fc.expected_first(oracle, line.reshape(1, n), w, border, fc.SIGNED)[0]
          want = np.abs(oracle.sdfsq(line, anisotropy=w, black_border=bool(border)))
          assert_same(got, want, (nbytes, n, kind, w, border))


def test_sequential_sums_tell_products_apart():
  """For every weight whose multiples are inexact, the step table differs at some tested k from the
  squares of the products k w (rounded once or twice): a kernel that multiplied would fail."""
  top = max(LENGTHS) + 1
  k = np.arange(top, dtype=np.float64)
  for w in fc.INEXACT_WEIGHTS:
    w32 = np.float32(w)
    table = fc.step_table(float(w32), top)
    once = (k * float(w32)) ** 2
    twice = (k * w32).astype(np.float32).astype(np.float64) ** 2
    for name, guess in (("rounded once", once), ("product rounded", twice)):
      guess = guess.astype(np.float32)
      assert np.any(guess != table), (w, name)
      first = int(np.flatnonzero(guess != table)[0])
      assert first <= 1056, (w, name, first)        # within the shorter tested rows
  for w in (1.0, 3.0):
    assert np.array_equal(fc.step_table(w, top), ((k * w) ** 2).astype(np.float32))
  big = fc.step_table(float(np.float32(fc.OVERFLOW_WEIGHT)), 4)
  assert np.isfinite(big[1]) and np.all(np.isinf(big[2:]))


# Kernels that are subtly wrong, as changes to (kL, kR): no border, or a label change credited to the
# wrong one of the two voxels it lies between -- on one side (a distance measured to the last voxel
# of the own run instead of the first voxel of the other), or on both sides the other way round, so
# that a voxel halfway between two changes takes the wrong side.
MUTANTS = ("border ignored", "left change on the own voxel", "right change on the own voxel",
           "sides swapped")


def mutant_value(kind, lab, w, border):
  sx = lab.shape[-1]
  far = 1 << 40
  kl, kr = fc.steps(lab, 0 if kind == "border ignored" else border)
  kl = np.where(kl > sx, far, kl)
  kr = np.where(kr > sx, far, kr)
  if kind == "left change on the own voxel":
    kl = kl - 1
  elif kind == "right change on the own voxel":
    kr = kr - 1
  elif kind == "sides swapped":
    kl, kr = kl - 1, kr + 1
  k = np.minimum(kl, kr)
  table = np.append(fc.step_table(float(np.float32(w)), sx + 2), np.float32(np.inf))
  out = table[np.where(k >= far // 2, sx + 2, k)]
  out[lab == 0] = 0.0
  return out


@pytest.mark.parametrize("nbytes", (1, 8))
def test_cases_catch_wrong_kernels(oracle, nbytes):
  """Every mutant changes some expected value at every tested row length, among the labelings,
  weights and borders the GPU tests run there."""
  rng = np.random.default_rng(30 + nbytes)
  for n in LENGTHS:
    lab = fc.rows(rng, n, nbytes)
    want = {(w, b): fc.expected_first(oracle, lab, w, b, 0) for w in fc.WEIGHTS for b in (0, 1)}
    for kind in MUTANTS:
      assert any(not np.array_equal(mutant_value(kind, lab, w, b), v) for (w, b), v in want.items()), \
          (nbytes, n, kind)
