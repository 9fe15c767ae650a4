"""Inputs of the per-pass envelope tests (tests/test_envelope_*.py): labels and float32 sample
profiles for ONE later-axis pass, all seeded and deterministic, and a plain brute-force statement
of that pass.

Arrays are C-ordered (z, y, x) like oracle.pass_later takes them; a pass along axis 1 runs down y,
along axis 2 down z.  The brute force reads the pass straight from its definition: for every voxel
the least of w2 * d^2 + f over the samples of its run, and of the border terms, formed in float64
and rounded once to float32 (src/edt.hpp:225-242 of the reference).
"""
import numpy as np

PROFILES = ("int_ties", "inf_rich", "zeros", "real", "above_2_24", "tiny")


def profile(rng, kind, shape):
  """float32 samples of one kind for a (z, y, x) volume."""
  n = int(np.prod(shape))
  if kind == "int_ties":        # few distinct integer heights: exact ties between candidates
    f = rng.integers(0, 6, n) ** 2 * rng.choice([1, 4, 9], n)
  elif kind == "inf_rich":      # mostly +inf, some whole lines with no site at all
    f = np.where(rng.random(n) < 0.85, np.inf, rng.integers(0, 400, n))
  elif kind == "zeros":         # zeros inside runs of positive heights
    f = np.where(rng.random(n) < 0.1, 0.0, rng.integers(1, 5000, n))
  elif kind == "real":          # real-valued heights
    f = rng.random(n) * 1000.0
  elif kind == "above_2_24":    # integer heights above 2^24, so candidates round to float32
    f = rng.integers(1 << 24, 1 << 27, n)
  elif kind == "tiny":          # a sample far below the others: candidate sums inexact in double
    f = rng.random(n) * 50.0
    f[rng.random(n) < 0.05] = 2.0 ** -52
  else:
    raise ValueError(kind)
  f = np.asarray(f, dtype=np.float32).reshape(shape)
  if kind == "inf_rich" and shape[-1] > 2:
    f[..., 1] = np.inf          # the lines through x = 1 hold no site
  return f


LABELINGS = ("one_run", "chunk_aligned", "runs", "single_rows", "noise")


def labels(rng, kind, shape, axis, dtype):
  """Labels whose runs along `axis` are: the whole line, 32-row runs (chunk-aligned), runs of
  random lengths (crossing one or many 32-row chunks), many one-row runs, or label noise."""
  n = shape[0] if axis == 2 else shape[1]
  if kind == "one_run":
    run = np.zeros(n, np.int64)
  elif kind == "chunk_aligned":
    run = np.arange(n) // 32
  elif kind == "runs":
    cuts = np.cumsum(rng.geometric(1.0 / max(2, n // 6), n))
    run = np.searchsorted(cuts, np.arange(n), side="right")
  elif kind == "single_rows":
    run = np.where(rng.random(n) < 0.6, np.arange(n), 0)
  elif kind == "noise":
    lab = rng.integers(0, 3, shape)
    return lab.astype(dtype)
  else:
    raise ValueError(kind)
  # per line: the run index plus a line-dependent offset, 0 kept for background
  along = run.reshape((-1, 1, 1) if axis == 2 else (1, -1, 1))
  offset = rng.integers(0, 3, tuple(1 if i == (0 if axis == 2 else 1) else s for i, s in enumerate(shape)))
  lab = (along + offset) % 5
  return np.broadcast_to(lab, shape).astype(dtype)


def brute_pass(lab, f, axis, w, border_lo, border_hi):
  """One later-axis pass by definition (every run alike, label 0 included; +inf is no site)."""
  w2 = float(np.float32(np.float32(w) * np.float32(w)))
  along = 0 if axis == 2 else 1
  lab = np.ascontiguousarray(np.moveaxis(np.asarray(lab), along, 0))
  src = np.ascontiguousarray(np.moveaxis(np.asarray(f, np.float32), along, 0))
  n = src.shape[0]
  out = np.empty_like(src)
  lines_l = lab.reshape(n, -1)
  lines_f = src.reshape(n, -1).astype(np.float64)
  res = out.reshape(n, -1)
  d2 = np.arange(n + 1, dtype=np.float64) ** 2
  for j in range(lines_f.shape[1]):
    l, v = lines_l[:, j], lines_f[:, j]
    a = 0
    while a < n:
      b = a + 1
      while b < n and l[b] == l[a]:
        b += 1
      sites = [p for p in range(a, b) if np.isfinite(v[p])]
      for i in range(a, b):
        best = np.inf
        for p in sites:
          best = min(best, w2 * d2[abs(i - p)] + v[p])
        if a > 0 or border_lo:
          best = min(best, w2 * d2[i - a + 1])
        if b < n or border_hi:
          best = min(best, w2 * d2[b - i])
        res[i, j] = np.float32(best)
      a = b
  return np.ascontiguousarray(np.moveaxis(out, 0, along))


def expected_pass(oracle, lab, f, axis, w, border_lo, border_hi, sqrt=False, negate=False):
  """What edtb200_pass_later must produce: the oracle's envelope pass with every run treated as
  foreground (the device pass envelopes background runs too), then the store's epilogue."""
  want = np.ascontiguousarray(f, dtype=np.float32).copy()
  oracle.pass_later(np.asarray(lab).astype(np.int64) + 1, want, axis, w, border_lo, border_hi)
  if sqrt:
    np.sqrt(want, out=want)
  if negate:
    want[np.asarray(lab) == 0] *= -1.0
  return want


def plateau_trap(n=96, row=64, m=8):
  """One line of n samples (one run, w = 1, no border) built so that at `row`, the first row of a
  32-row chunk, the nearest hull vertex and the one below it round to the SAME float32 while a
  farther vertex is lower.  With K = 2^30 + 256 m (float32 spacing 128 there) the three sites at
  distances 7, 12 and 36 below `row` have heights that are multiples of 128 and candidate values
  c = d^2 + f = K + 49, K + 16 and K - 112 at `row`: the first two round to K, the third to
  K - 128.  All three are vertices of the lower envelope (the middle one owns row + 3 alone);
  every other sample is +inf.  Returns (f, K, the vertex positions from the lowest)."""
  K = (1 << 30) + 256 * m
  dist = (36, 12, 7)
  value = (K - 112, K + 16, K + 49)
  f = np.full(n, np.inf, np.float32)
  for d, c in zip(dist, value):
    f[row - d] = c - d * d
    assert float(f[row - d]) == c - d * d and (c - d * d) % 128 == 0
  return f, K, tuple(row - d for d in dist)
