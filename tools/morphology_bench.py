#!/usr/bin/env python
"""Spherical morphology on one GPU against the compositions of public calls it replaces.

  python tools/morphology_bench.py [--n 512] [--steps 5] [--warmup 2] [--rounds 3] [--sweep] [--out FILE]

Device-resident n^3 volumes: 32-bit Voronoi cells (200 seeds), 32-bit labels in 32^3 blocks, 8-bit balls
(workloads.py) and an 8-bit single mask (one ball).  For each of erode, open, dilate and close at
r in {1, 2, 4, 8, 16}, without black_border:
  - the new call against the composition of public calls it replaces, both device-resident:
      erode   edtsq(max_distance=r), then torch.where on (labels != 0) & (d2 > r^2)
      open    that, then edtsq(max_distance=r) of the kept mask and torch.where
      dilate  sdfsq(max_distance=r), then (labels != 0) | (|s| <= r^2)
      close   that, then edtsq(max_distance=r) of the dilation and a compare
    alternating round by round (CUDA events around each round of `steps` calls, after warm-up; the
    median round is printed);
  - whether the two outputs are equal (the radii are integers, so r^2 is exact in float32);
  - the device memory each takes beyond its input and output: the drop in free device memory over one
    call with everything released first (the library keeps its scratch pool's high-water mark,
    EDTB200_POOL_KEEP_MB; torch keeps what its caching allocator took), less the output's bytes.
Then one scipy.ndimage row at 128^3 (balls, r = 4, one thread) for context.
--sweep adds the erode and open times with every later pass forced onto the window kernel
(EDTB200_BOUNDED_RMAX=128) at radii 2..8, against the default plan, to place the window / tile crossover
of the label-writing store.  The card's name, power limit and maximum SM clock are read in the same run.
"""
import argparse
import os
import subprocess
import sys
import time

os.environ.setdefault("EDTB200_POOL_KEEP_MB", str(1 << 20))     # keep the pool's high-water mark

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import edt_b200 as edt  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402
from edt_b200 import workloads  # noqa: E402

RADII = (1, 2, 4, 8, 16)
OPS = ("erode", "open", "dilate", "close")
LINES = []


def say(line=""):
  print(line, flush=True)
  LINES.append(line)


def smi(fields):
  try:
    return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + fields, "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or "unknown"
  except Exception as e:
    return "unknown (%s)" % e


def volumes(n):
  yield "voronoi32", workloads.generate("voronoi", n, "cuda")[0]
  g = torch.Generator(device="cuda")
  g.manual_seed(5)
  k = 32
  small = torch.randint(0, 1 << 20, (-(-n // k),) * 3, dtype=torch.int32, device="cuda", generator=g)
  blocks = small.repeat_interleave(k, 0).repeat_interleave(k, 1).repeat_interleave(k, 2)[:n, :n, :n].contiguous()
  del small
  yield "blocks32", blocks
  del blocks
  yield "balls8", workloads.generate("balls", n, "cuda")[0]
  c = torch.arange(n, device="cuda", dtype=torch.float32) - (n - 1) / 2
  d2 = c.view(-1, 1, 1) ** 2 + c.view(1, -1, 1) ** 2 + c.view(1, 1, -1) ** 2
  mask = (d2 <= (0.4 * n) ** 2).to(torch.uint8)
  del d2
  yield "mask8", mask


def composed(op, t, r):
  """The composition of public calls that op replaces."""
  rr = float(r) * float(r)
  zero = torch.zeros((), dtype=t.dtype, device=t.device)
  if op in ("erode", "open"):
    kept = torch.where((t != 0) & (edt.edtsq(t, max_distance=r) > rr), t, zero)
    if op == "erode":
      return kept
    return torch.where((t != 0) & (edt.edtsq((kept == 0).to(torch.uint8), max_distance=r) <= rr), t, zero)
  dil = (t != 0) | (edt.sdfsq(t, max_distance=r).abs() <= rr)
  if op == "dilate":
    return dil
  return dil & (edt.edtsq(dil.to(torch.uint8), max_distance=r) > rr)


def native(op, t, r):
  return getattr(edt, "spherical_" + op)(t, float(r))


def timed_pair(fa, fb, steps, warmup, rounds):
  """Median per-call ms of fa and fb, alternating round by round."""
  for _ in range(warmup):
    fa(); fb()
  torch.cuda.synchronize()
  ta, tb = [], []
  for _ in range(rounds):
    for f, acc in ((fa, ta), (fb, tb)):
      s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      s.record()
      for _ in range(steps):
        f()
      e.record()
      e.synchronize()
      acc.append(s.elapsed_time(e) / steps)
  return sorted(ta)[len(ta) // 2], sorted(tb)[len(tb) // 2]


def extra_bytes(f):
  """Device memory one call takes beyond its input and output (its output kept alive)."""
  torch.cuda.synchronize()
  edt.release()
  torch.cuda.empty_cache()
  free0 = torch.cuda.mem_get_info()[0]
  out = f()
  torch.cuda.synchronize()
  free1 = torch.cuda.mem_get_info()[0]
  nbytes = out.numel() * out.element_size()
  del out
  return free0 - free1 - nbytes


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--steps", type=int, default=5)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--sweep", action="store_true")
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  say("morphology_bench: %s, power limit %s, max SM clock %s" % (smi("name"), smi("power.limit"), smi("clocks.max.sm")))
  say("n=%d steps=%d warmup=%d rounds=%d; ms per call (median round); MiB of device memory beyond input and output"
      % (a.n, a.steps, a.warmup, a.rounds))
  say("%-9s %-6s %3s %10s %10s %6s %9s %9s %s" % ("workload", "op", "r", "composed", "native", "x", "MiB comp",
                                                  "MiB nat", "equal"))
  sweep_vols = {}
  for name, t in volumes(a.n):
    for op in OPS:
      for r in RADII:
        got, exp = native(op, t, r), composed(op, t, r)
        ok = got.dtype == exp.dtype and torch.equal(got, exp)
        del got, exp
        t_comp, t_nat = timed_pair(lambda: composed(op, t, r), lambda: native(op, t, r), a.steps, a.warmup, a.rounds)
        m_comp = extra_bytes(lambda: composed(op, t, r))
        m_nat = extra_bytes(lambda: native(op, t, r))
        say("%-9s %-6s %3d %10.3f %10.3f %6.2f %9.0f %9.0f %s" % (
            name, op, r, t_comp, t_nat, t_comp / t_nat, m_comp / 2**20, m_nat / 2**20, "yes" if ok else "NO"))
    if a.sweep and name in ("voronoi32", "balls8"):
      say()
      say("sweep %s: the default plan (window kernel up to R = 2) against every later pass on the window kernel "
          "(EDTB200_BOUNDED_RMAX=128)" % name)
      say("%-6s %3s %10s %10s %6s %s" % ("op", "r", "default", "window", "x", "equal"))
      for op in ("erode", "open"):
        for r in (2, 3, 4, 6, 8):
          ok = torch.equal(_forced(op, t, r), native(op, t, r))
          t_def, t_win = timed_pair(lambda: native(op, t, r), lambda: _forced(op, t, r), a.steps, a.warmup, a.rounds)
          say("%-6s %3d %10.3f %10.3f %6.2f %s" % (op, r, t_def, t_win, t_def / t_win, "yes" if ok else "NO"))
      say()
    del t
    torch.cuda.empty_cache()
  say()
  from scipy import ndimage
  sys.path.insert(0, os.path.join(ROOT, "tests"))
  import morphology_cases as mc
  small = workloads.generate("balls", 128, "cpu")[0].numpy() != 0
  B = mc.ball(4.0, (1.0, 1.0, 1.0))
  for op, f in (("erode", lambda: ndimage.binary_erosion(small, B, border_value=1)),
                ("dilate", lambda: ndimage.binary_dilation(small, B, border_value=0))):
    t0 = time.perf_counter()
    ref = f()
    dt = time.perf_counter() - t0
    ours = getattr(edt, "spherical_" + op)(small, 4.0)
    say("scipy.ndimage binary_%s, 128^3 balls, r = 4, one thread: %.3f s; spherical_%s equal: %s" % (
        "erosion" if op == "erode" else "dilation", dt, op, "yes" if np.array_equal(ours != 0, ref) else "NO"))
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
      fh.write("\n".join(LINES) + "\n")


def _forced(op, t, r):
  os.environ["EDTB200_BOUNDED_RMAX"] = "128"
  try:
    return native(op, t, r)
  finally:
    del os.environ["EDTB200_BOUNDED_RMAX"]


if __name__ == "__main__":
  main()
