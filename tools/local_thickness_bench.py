#!/usr/bin/env python
"""Local thickness on one GPU against the composition of public calls it replaces.

  python tools/local_thickness_bench.py [--n 512] [--steps 1] [--warmup 1] [--rounds 3] [--out FILE]

Device-resident n^3 volumes, the workloads of morphology_bench.py: 32-bit Voronoi cells (200 seeds), 32-bit
labels in 32^3 blocks, 8-bit balls (workloads.py) and an 8-bit single mask (one ball).  For n = 8, 25 and 50
default levels, without black_border:
  - local_thickness(t, sizes=n) against the composition at the levels it returned: one spherical_open per
    level and a torch.maximum of where(open != 0, r, 0), alternating round by round (CUDA events around each
    round of `steps` calls, after warm-up; the median round is printed);
  - whether the two outputs are equal, byte for byte;
  - the device memory each takes beyond its input and output: the drop in free device memory over one call
    with everything released first (the library keeps its scratch pool's high-water mark,
    EDTB200_POOL_KEEP_MB; torch keeps what its caching allocator took), less the output's bytes.
Then one scipy row at 128^3 for context: porespy's definition on the one-ball mask with
scipy.ndimage.distance_transform_edt at the 8 levels the native call returned, one thread.  The card's name,
power limit and maximum SM clock are read in the same run.
"""
import argparse
import os
import sys
import time

os.environ.setdefault("EDTB200_POOL_KEEP_MB", str(1 << 20))     # keep the pool's high-water mark

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import edt_b200 as edt  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402
from morphology_bench import extra_bytes, smi, timed_pair, volumes  # noqa: E402

LEVELS = (8, 25, 50)
LINES = []


def say(line=""):
  print(line, flush=True)
  LINES.append(line)


def composed(t, levels):
  """The maximum over one spherical_open per level."""
  out = torch.zeros(t.shape, dtype=torch.float32, device=t.device)
  zero = torch.zeros((), dtype=torch.float32, device=t.device)
  for r in levels:
    out = torch.maximum(out, torch.where(edt.spherical_open(t, r) != 0, torch.tensor(np.float32(r), device=t.device),
                                         zero))
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--steps", type=int, default=1)
  ap.add_argument("--warmup", type=int, default=1)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  say("local_thickness_bench: %s, power limit %s, max SM clock %s"
      % (smi("name"), smi("power.limit"), smi("clocks.max.sm")))
  say("n=%d steps=%d warmup=%d rounds=%d; ms per call (median round); MiB of device memory beyond input and output"
      % (a.n, a.steps, a.warmup, a.rounds))
  say("%-9s %6s %10s %10s %6s %9s %9s %s" % ("workload", "levels", "composed", "native", "x", "MiB comp", "MiB nat",
                                             "equal"))
  for name, t in volumes(a.n):
    for m in LEVELS:
      got, lv = edt.local_thickness(t, sizes=m, return_sizes=True)
      levels = lv.cpu().tolist()                    # the composition runs at the levels the call used
      ok = torch.equal(got, composed(t, levels))
      del got
      t_comp, t_nat = timed_pair(lambda: composed(t, levels), lambda: edt.local_thickness(t, sizes=m), a.steps,
                                 a.warmup, a.rounds)
      m_comp = extra_bytes(lambda: composed(t, levels))
      m_nat = extra_bytes(lambda: edt.local_thickness(t, sizes=m))
      say("%-9s %6d %10.2f %10.2f %6.2f %9.0f %9.0f %s" % (name, m, t_comp, t_nat, t_comp / t_nat, m_comp / 2**20,
                                                          m_nat / 2**20, "yes" if ok else "NO"))
    del t
    torch.cuda.empty_cache()
  say()
  from scipy import ndimage
  n = 128
  c = np.arange(n, dtype=np.float64) - (n - 1) / 2
  mask = (c[:, None, None] ** 2 + c[None, :, None] ** 2 + c[None, None, :] ** 2 <= (0.4 * n) ** 2)
  ours, lv = edt.local_thickness(mask.astype(np.uint8), sizes=8, return_sizes=True)
  t0 = time.perf_counter()
  d = ndimage.distance_transform_edt(mask)
  ref = np.zeros(mask.shape, np.float32)
  for r in lv:
    covered = ndimage.distance_transform_edt(~(d > r)) <= r
    ref = np.maximum(ref, np.where(covered & mask, np.float32(r), np.float32(0)))
  dt = time.perf_counter() - t0
  say("scipy.ndimage restatement, 128^3 one-ball mask, 8 levels, one thread: %.3f s; local_thickness equal: %s"
      % (dt, "yes" if np.array_equal(ours, ref) else "NO (%d voxels differ)" % int((ours != ref).sum())))
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
      fh.write("\n".join(LINES) + "\n")


if __name__ == "__main__":
  main()
