"""GPU tests (-m gpu) of the label-noise plan (plan_noise): for every row of its decision table -- label
width, function, integral or non-integral weights, rows 4-aligned, unaligned or longer than 512 voxels,
lines longer than 512 rows, 2-D, 3-D and stacks -- the last later pass's launch on the first call after
a structured volume (no noise predicted) and on the second call (noise predicted), and both results
bit for bit against the oracle.

  python tests/test_noise_plan_gpu.py OUT.json    (EDTB200_LIBRARY=... for another build)

writes the kernels and grids that every case launches (torch.profiler) to OUT.json.
"""
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from noise_cases import noise  # noqa: E402

pytestmark = pytest.mark.gpu

U8, U16, U32, U64 = np.uint8, np.uint16, np.uint32, np.uint64
ONES, FRAC = (1.0, 1.0, 1.0), (1.0, 0.7, 1.0)    # array order (z, y, x); 0.7: no integer hull
# dtype, function, shape (C order; a stack where it has more axes than the anisotropy), anisotropy; then
# the last later pass's tma, wide, int_hull and, with noise predicted, ctas and settled (tx = 32 and the
# tile kernel throughout)
CASES = [
    (U8, "edtsq", (20, 40, 128), ONES, 1, 0, 1, 2, 0),       # narrow labels: no planes
    (U16, "edt", (20, 40, 128), ONES, 1, 0, 1, 2, 0),
    (U32, "edtsq", (20, 40, 128), ONES, 1, 0, 1, 2, 1),      # planes, settled tiles skipped
    (U64, "edtsq", (20, 40, 128), ONES, 1, 0, 1, 2, 1),
    (U32, "edt", (20, 40, 128), ONES, 1, 0, 1, 2, 0),        # epilogue: planes read, no skip
    (U64, "sdf", (20, 40, 128), ONES, 1, 0, 1, 2, 0),        # signed: no planes
    (U32, "edtsq", (20, 40, 128), FRAC, 1, 0, 0, 2, 0),      # planes read, no skip
    (U64, "edt", (20, 40, 128), FRAC, 1, 0, 0, 2, 0),
    (U32, "edtsq", (20, 40, 130), ONES, 1, 0, 1, 2, 0),      # rows unaligned: no planes, Z lines aligned
    (U8, "edtsq", (20, 41, 130), ONES, 0, 0, 0, 3, 0),       # Z lines unaligned: no TMA
    (U32, "edtsq", (8, 20, 600), ONES, 1, 0, 1, 2, 0),       # rows > 512: no planes
    (U64, "edtsq", (600, 8, 32), ONES, 1, 1, 1, 3, 0),       # Z lines > 512 rows: wide, its plane unread
    (U16, "sdf", (600, 8, 32), ONES, 1, 1, 1, 3, 0),
    (U32, "edtsq", (40, 128), ONES[1:], 1, 0, 1, 2, 1),
    (U64, "edt", (40, 128), ONES[1:], 1, 0, 1, 2, 0),
    (U8, "sdf", (40, 128), ONES[1:], 1, 0, 1, 2, 0),
    (U64, "edtsq", (40, 128), FRAC[1:], 1, 0, 0, 2, 0),
    (U32, "edtsq", (40, 130), ONES[1:], 0, 0, 0, 3, 0),
    (U32, "edtsq", (3, 10, 20, 128), ONES, 1, 0, 1, 2, 1),
    (U64, "edt", (3, 10, 20, 128), ONES, 1, 0, 1, 2, 0),
    (U8, "edtsq", (4, 40, 128), ONES[1:], 1, 0, 1, 2, 0),
]
IDS = ["%s-%s-%s-%s" % (c[0].__name__, c[1], "x".join(map(str, c[2])), "int" if c[3][1] == 1 else "frac")
       for c in CASES]


def calls(edt, case):
  """The first and second call of one case after a structured volume: (result, last_later_launch())."""
  dtype, fn, shape, w = case[:4]
  lab = noise(shape, dtype, sum(shape))
  edt.edtsq(np.zeros((4, 9, 512), np.uint32))
  out = []
  for _ in range(2):
    got = getattr(edt, fn)(lab, anisotropy=w, stacked=len(shape) > len(w))
    out.append((got, edt.last_later_launch()))
  return lab, out


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_noise_plan(edt, oracle, case):
  fn, shape, w, (tma, wide, int_hull, ctas, settled) = case[1], case[2], case[3], case[4:]
  lab, out = calls(edt, case)
  stacked = len(shape) > len(w)
  vols = lab if stacked else [lab]
  want = [getattr(oracle, fn)(np.ascontiguousarray(v), anisotropy=w) for v in vols]
  for call, (got, info) in enumerate(out):
    expect = dict(kernel="tile", tx=32, tma=tma, wide=wide, int_hull=int_hull, epilogue=int(fn != "edtsq"),
                  ctas=ctas, settled=settled if call else 0)
    # the first call plans with no noise predicted: 3 CTAs per SM, or the noise plan's where a later
    # pass reads the prediction at its launch, after the first call's own X pass published noise
    if call == 0 and info["ctas"] == 3:
      expect["ctas"] = 3
    assert {k: info[k] for k in expect} == expect, (call, info)
    for v, (g, x) in enumerate(zip(got if stacked else [got], want)):
      assert np.array_equal(g, x), (call, v, int((g != x).sum()))


def kernel_list(path):
  import torch
  from torch.profiler import ProfilerActivity, profile
  import edt_b200 as edt
  rows = {}
  for name, case in zip(IDS, CASES):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      calls(edt, case)
      torch.cuda.synchronize()
    trace = path + ".trace.json"
    prof.export_chrome_trace(trace)
    with open(trace) as f:
      events = json.load(f)["traceEvents"]
    os.remove(trace)
    rows[name] = [[e["name"], e["args"].get("grid")] for e in sorted(events, key=lambda e: e.get("ts", 0))
                  if e.get("cat") == "kernel"]
  with open(path, "w") as f:
    json.dump(rows, f, indent=1)


if __name__ == "__main__":
  kernel_list(sys.argv[1])
