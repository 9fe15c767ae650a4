#!/usr/bin/env python
"""Bounded transforms (max_distance) on one GPU against the unbounded ones.

  python tools/bounded_bench.py [--n 512] [--steps 10] [--warmup 2] [--rounds 3] [--sweep] [--out FILE]

Device-resident n^3 volumes of workloads.py (cfg2, cfg2b, cfg3, balls, voronoi) and d in {2.5, 8, 24}:
  - edtsq (edt_cuda) unbounded against bounded, and feature_transform(return_distances=True)
    unbounded against bounded: the two calls of a pair alternate over `rounds` rounds of `steps`
    calls each (CUDA events around each round, after warm-up); the median round is printed;
  - the device memory of each feature call beyond the labels, read as tools/feature_bench.py reads it:
    the library's scratch pool keeps what it took (EDTB200_POOL_KEEP_MB), everything is released
    first, so the drop in free device memory over one call, its results still alive, is its peak
    (other work on the same card would show up in it too);
  - an equality check of every bounded result against the unbounded one with the band applied.
The plan of every case is printed beside it: per later axis the radius, then w (window kernel) or u
(unbounded kernel) for the transform and for the feature transform.
--sweep adds the run that chose EDTB200_BOUNDED_WINDOW_MAX: every later pass forced onto the window
kernel (EDTB200_BOUNDED_RMAX=128) at radii 2..32 on balls, voronoi and cfg2, against the unbounded call.
The card's name, power limit and maximum SM clock are read in the same run.
"""
import argparse
import ctypes
import os
import subprocess
import sys

os.environ.setdefault("EDTB200_POOL_KEEP_MB", str(1 << 20))     # keep the pool's high-water mark

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import edt_b200 as edt  # noqa: E402
import torch  # noqa: E402
from edt_b200 import workloads  # noqa: E402

WORKLOADS = ("cfg2", "cfg2b", "cfg3", "balls", "voronoi")
DISTANCES = (2.5, 8.0, 24.0)
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


def peak_bytes(f):
  """Device memory one call takes beyond what is alive before it (its results kept alive)."""
  torch.cuda.synchronize()
  edt.release()
  torch.cuda.empty_cache()
  free0 = torch.cuda.mem_get_info()[0]
  out = f()
  torch.cuda.synchronize()
  free1 = torch.cuda.mem_get_info()[0]
  del out
  return free0 - free1


def plan_text(lab, w, d):
  dims = list(lab.shape)[::-1]
  ws = list(w)[::-1]
  r = (ctypes.c_int64 * 3)()
  win = (ctypes.c_int * 3)()
  edt._lib().edtb200_bounded_plan(3, *dims, *ws, d, r, win)
  # per later axis: its radius, then w / u for the window or the unbounded kernel in the transform's
  # plan and in the feature transform's (edtb200_bounded_plan's bits 0 and 1)
  return " ".join("%s:R%d/%s%s" % ("yz"[k - 1], r[k], "wu"[not win[k] & 1], "wu"[not win[k] & 2]) for k in (1, 2))


def banded(unbounded, sq, d):
  keep = sq.abs().double() <= d * d
  return torch.where(keep, unbounded, torch.where(torch.signbit(sq), -float("inf"), float("inf")).to(sq.dtype))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--steps", type=int, default=10)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--sweep", action="store_true")
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  say("bounded_bench: %s, power limit %s, max SM clock %s" % (smi("name"), smi("power.limit"), smi("clocks.max.sm")))
  say("n=%d steps=%d warmup=%d rounds=%d; ms per call (median round), memory beyond the labels" %
      (a.n, a.steps, a.warmup, a.rounds))
  say("%-8s %5s  %-22s %9s %9s %6s | %9s %9s %6s | %8s %8s | %s" % (
      "workload", "d", "plan", "edtsq", "bounded", "x", "feature", "bounded", "x", "GiB unb", "GiB bnd", "equal"))
  for name in WORKLOADS:
    lab, w, border = workloads.generate(name, a.n, "cuda")
    sq = edt.edt_cuda(lab, w, border)
    full = edt.edt_cuda(lab, w, border, sqrt=True)
    for d in DISTANCES:
      ok = torch.equal(edt.edt_cuda(lab, w, border, max_distance=d).view(torch.int32),
                       banded(sq, sq, d).view(torch.int32))
      dist, idx = edt.feature_transform(lab, w, border, return_distances=True, max_distance=d)
      inside = sq.double() <= d * d
      ok = ok and torch.equal(dist.view(torch.int32), banded(full, sq, d).view(torch.int32))
      ok = ok and bool((idx[:, ~inside] == -1).all())
      del dist, idx, inside
      t_unb, t_bnd = timed_pair(lambda: edt.edt_cuda(lab, w, border),
                                lambda: edt.edt_cuda(lab, w, border, max_distance=d), a.steps, a.warmup, a.rounds)
      f_unb, f_bnd = timed_pair(lambda: edt.feature_transform(lab, w, border, return_distances=True),
                                lambda: edt.feature_transform(lab, w, border, return_distances=True, max_distance=d),
                                max(1, a.steps // 2), a.warmup, a.rounds)
      m_unb = peak_bytes(lambda: edt.feature_transform(lab, w, border, return_distances=True))
      m_bnd = peak_bytes(lambda: edt.feature_transform(lab, w, border, return_distances=True, max_distance=d))
      say("%-8s %5.1f  %-22s %9.3f %9.3f %6.2f | %9.3f %9.3f %6.2f | %8.2f %8.2f | %s" % (
          name, d, plan_text(lab, w, d), t_unb, t_bnd, t_unb / t_bnd, f_unb, f_bnd, f_unb / f_bnd,
          m_unb / 2**30, m_bnd / 2**30, "yes" if ok else "NO"))
    del lab, sq, full
    torch.cuda.empty_cache()
  if a.sweep:
    say()
    say("sweep: every later pass on the window kernel (EDTB200_BOUNDED_RMAX=128), d = R (unit weights)")
    say("%-8s %4s %9s %9s %6s | %9s %9s %6s" % ("workload", "R", "edtsq", "window", "x", "feature", "window", "x"))
    for name in ("balls", "voronoi", "cfg2"):
      lab, w, border = workloads.generate(name, a.n, "cuda")
      for r in (2, 4, 8, 12, 16, 20, 24, 32):
        os.environ["EDTB200_BOUNDED_RMAX"] = "128"
        t_unb, t_bnd = timed_pair(lambda: edt.edt_cuda(lab, w, border),
                                  lambda: edt.edt_cuda(lab, w, border, max_distance=float(r)),
                                  a.steps, a.warmup, a.rounds)
        f_unb, f_bnd = timed_pair(lambda: edt.feature_transform(lab, w, border, return_distances=True),
                                  lambda: edt.feature_transform(lab, w, border, return_distances=True,
                                                                max_distance=float(r)),
                                  max(1, a.steps // 2), a.warmup, a.rounds)
        del os.environ["EDTB200_BOUNDED_RMAX"]
        say("%-8s %4d %9.3f %9.3f %6.2f | %9.3f %9.3f %6.2f" % (
            name, r, t_unb, t_bnd, t_unb / t_bnd, f_unb, f_bnd, f_unb / f_bnd))
      del lab
      torch.cuda.empty_cache()
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
      fh.write("\n".join(LINES) + "\n")


if __name__ == "__main__":
  main()
