#!/usr/bin/env python
"""Time feature_transform against edtsq on the same device-resident 512^3 volumes.

  python tools/feature_bench.py [--n 512] [--steps 10] [--warmup 2] [--out FILE]

For each workload (workloads.py: cfg2, cfg2b, cfg3, balls, voronoi) it times, with CUDA events
after warm-up, edtsq, feature_transform (indices only) and feature_transform(return_distances=True),
all on torch CUDA tensors, and reads the device memory each call takes beyond the input labels: the
library's scratch pool is set to keep what it took (EDTB200_POOL_KEEP_MB), so the drop in free
device memory over one call, its outputs still alive, is that call's peak.  The card's name, power
limit and maximum SM clock are printed with the numbers, and the SM clock nvidia-smi reads right after
each timed loop is printed beside it.
"""
import argparse
import os
import subprocess
import sys

os.environ.setdefault("EDTB200_POOL_KEEP_MB", str(1 << 20))     # keep the pool's high-water mark

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)

WORKLOADS = ("cfg2", "cfg2b", "cfg3", "balls", "voronoi")


def smi(fields):
  try:
    return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + fields, "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
  except Exception as e:        # the numbers below still stand; say what is missing
    return "nvidia-smi unavailable (%s)" % e


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--steps", type=int, default=10)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  import torch
  import edt_b200
  from edt_b200 import workloads
  lines = []

  def emit(s):
    print(s, flush=True)
    lines.append(s)

  emit("card (name, power limit, maximum SM clock): %s | torch %s" % (smi("name,power.limit,clocks.max.sm"),
                                                                      torch.__version__))
  emit("%d^3, device-resident, CUDA events, %d steps after %d warm-up; mem = device memory beyond the labels"
       % (args.n, args.steps, args.warmup))
  emit("%-8s %-22s %10s %10s %9s  %s" % ("workload", "call", "ms/call", "Mvox/s", "mem GiB", "SM clock after"))
  for name in WORKLOADS:
    lab, an, bb = workloads.generate(name, args.n, "cuda")
    calls = (("edtsq", lambda: edt_b200.edtsq(lab, an, bb)),
             ("feature_transform", lambda: edt_b200.feature_transform(lab, an, bb)),
             ("feature_transform+dist", lambda: edt_b200.feature_transform(lab, an, bb, return_distances=True)))
    for cname, fn in calls:
      torch.cuda.synchronize()
      edt_b200.release()
      torch.cuda.empty_cache()
      free0 = torch.cuda.mem_get_info()[0]
      out = fn()
      torch.cuda.synchronize()
      mem = (free0 - torch.cuda.mem_get_info()[0]) / 2 ** 30
      del out
      for _ in range(args.warmup):
        fn()
      start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      start.record()
      for _ in range(args.steps):
        fn()
      stop.record()
      stop.synchronize()
      clock = smi("clocks.sm")
      ms = start.elapsed_time(stop) / args.steps
      emit("%-8s %-22s %10.3f %10.0f %9.2f  %s" % (name, cname, ms, lab.numel() / ms / 1e3, mem, clock))
    del lab
    torch.cuda.empty_cache()
  if args.out:
    with open(args.out, "w") as fh:
      fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
  main()
