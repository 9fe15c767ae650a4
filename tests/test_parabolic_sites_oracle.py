"""CPU tests: the numpy restatement of the parabolic sites (parabolic_sites_cases.py) against the definition
evaluated one voxel at a time with Fraction, its values against parabolic_cases.py, the chain identity,
the edtsq of a mask, and that each planted defect is noticed."""
import numpy as np
import pytest

import parabolic_cases as pc
import parabolic_sites_cases as sc

OPS = ["erode", "dilate"]
WEIGHTS = [(1.0, 1.0, 1.0), (0.7, 1.3, 2.9), (6.0, 6.0, 30.0), (1e20, 1.0, 1e20), (2.0 ** -26,) * 3]


@pytest.mark.parametrize("family", pc.FAMILIES)
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("w", WEIGHTS, ids=["1", "frac", "6-6-30", "overflow", "tiny"])
def test_restatement_is_the_definition(family, op, w):
  rng = np.random.default_rng(pc.FAMILIES.index(family))
  for shape in ((3, 4, 6), (5, 7), (9,)):
    f = pc.values(family, shape, rng)
    ww = w[:len(shape)]
    vals, idx = sc.restate(op, f, ww)
    bvals, bidx = sc.restate(op, f, ww, line=sc.brute_line)
    assert pc.same_bits(vals, bvals) and pc.same_bits(vals, pc.restate(op, f, ww))
    assert np.array_equal(idx, bidx), (family, op, w, shape)
    assert idx.shape == (len(shape),) + shape and idx.dtype == np.int32


@pytest.mark.parametrize("family", pc.FAMILIES)
@pytest.mark.parametrize("op", OPS)
@pytest.mark.parametrize("order", ["C", "F"])
def test_the_value_is_the_chain_of_candidates_from_f_at_the_site(family, op, order):
  rng = np.random.default_rng(40 + pc.FAMILIES.index(family))
  f = pc.values(family, (6, 9, 11), rng)
  if order == "F":
    f = np.asfortranarray(f)
  for w in WEIGHTS:
    vals, idx = sc.restate(op, f, w, order=order)
    assert pc.same_bits(vals, sc.chain(op, f, idx, w, order=order)), (family, op, order, w)
    none = idx[0] < 0
    assert np.all(idx[:, none] == -1)
    q = np.where(none, 0, idx)
    fq = np.asarray(f, np.float32)[tuple(q)]
    assert not np.isnan(fq[~none]).any()
    assert np.all(vals[none] == (np.inf if op == "erode" else -np.inf))


def test_stacks_are_volumes_of_their_own():
  rng = np.random.default_rng(9)
  f = pc.values("special", (4, 5, 6), rng)
  vals, idx = sc.restate("erode", f, (1.3, 0.7), stacked=True)
  assert idx.shape == (2, 4, 5, 6)
  for b in range(4):
    v, i = sc.restate("erode", f[b], (1.3, 0.7))
    assert pc.same_bits(vals[b], v) and np.array_equal(idx[:, b], i)
  fv, fi = sc.restate("erode", np.asfortranarray(f.T), (0.7, 1.3), order="F", stacked=True)
  assert pc.same_bits(fv.T, vals) and np.array_equal(fi[::-1].transpose(0, 3, 2, 1), idx)


@pytest.mark.parametrize("w", [(1.0, 1.0, 1.0), (2.0, 3.0, 5.0), (1.0, 4.0, 2.0)])
def test_a_mask_gives_its_edtsq_at_the_index(oracle, w):
  rng = np.random.default_rng(11)
  mask = rng.random((7, 8, 9)) < 0.85
  vals, idx = sc.restate("erode", np.where(mask, np.inf, 0), w)
  P = np.indices(mask.shape)
  d2 = sum((w[k] * (P[k] - idx[k]).astype(np.float64)) ** 2 for k in range(3))
  want = oracle.edtsq(mask.astype(np.uint8), anisotropy=w)
  assert np.array_equal(d2.astype(np.float32), want) and pc.same_bits(vals, want)
  assert np.all(~mask[tuple(idx)])


def test_the_long_line_rule_is_the_float64_argmin():
  # past EXACT_N: the least j with the least float64 candidate (j == i: the sample itself)
  rng = np.random.default_rng(14)
  n = sc.EXACT_N + 1
  f = pc._load(pc.values("special", (1, n), rng))
  w = 0.7
  vals, sites = sc.line_sites(f, w)
  assert pc.same_bits(vals, pc.line_pass(f, w))
  j = np.arange(n)
  for i in (0, 1, 5000, n - 1):
    c = np.where(f[0] == np.inf, np.inf, sc._w2(w) * ((i - j) ** 2).astype(np.float64) + f[0].astype(np.float64))
    c[i] = np.inf if f[0, i] == np.inf else f[0, i]
    assert sites[0, i] == (int(np.argmin(c)) if np.isfinite(c.min()) or c.min() < 0 else -1)


@pytest.mark.parametrize("op", OPS)
def test_the_last_index_defect_is_noticed_on_integers(op):
  rng = np.random.default_rng(12)
  f = pc.values("integers", (6, 9, 11), rng)
  _, good = sc.restate(op, f, (1.0, 1.0, 1.0))
  _, bad = sc.restate(op, f, (1.0, 1.0, 1.0), defect="last")
  assert not np.array_equal(good, bad)


def test_the_rounded_defect_is_noticed_on_near_ties_and_the_cancelling_lines():
  # one near-tie line on every row: its Y pass compares equal values above 2^24, where X + 1 rounds to X
  rng = np.random.default_rng(13)
  f = np.repeat(pc.values("near_tie", (1, 700), rng), 4, axis=0)
  _, good = sc.restate("erode", f, (1.0, pc.NEAR_TIE_W))
  _, bad = sc.restate("erode", f, (1.0, pc.NEAR_TIE_W), defect="rounded")
  assert not np.array_equal(good, bad)
  for case in (0, 1):
    # the patterns negated (their +inf padding kept): 2^60 and 2^60 - 1 round alike one row apart
    line = pc.cancel_line(8, case, 2)[None, :]
    line = np.where(np.isinf(line), line, -line)
    _, good = sc.restate("erode", line, (1.0, pc.CANCEL_W))
    _, bad = sc.restate("erode", line, (1.0, pc.CANCEL_W), defect="rounded")
    assert not np.array_equal(good, bad), case
