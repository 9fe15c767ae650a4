#!/usr/bin/env python
"""skeletonize on one GPU: the edtsq and the thinning apart, and the numpy restatement for scale.

  python tools/skeleton_bench.py [--n 512] [--n_host 128] [--steps 3] [--warmup 1] [--rounds 3] [--out FILE]

Device-resident n^3 inputs: 8-bit balls (64) and 32-bit Voronoi cells (200 seeds) (workloads.py), 32-bit
labels in 32^3 blocks, an 8-bit single mask (one ball), and the 32-bit Voronoi cells with weights
(4, 4, 40).  For each (CUDA events around each round of `steps` calls, after warm-up; the median round):
  total     edt.skeletonize(labels) in ms per call
  edtsq     edt.edtsq(labels) in ms per call: the first step of the call, the same passes
  thin      total - edtsq
  rounds, cycles, steps   the thinning's counts, from one EDT_B200_VERBOSE=1 call in a child process
  MiB       device memory taken beyond the input and the output (the drop in free device memory over one call
            with everything released first; the library keeps its pool's high-water mark)
and the skeleton voxels per labelled voxel.  Then the numpy restatement (tests/skeleton_cases.py) of the
first two workloads at n_host^3 on one host thread, against the GPU call at that size (the skeletons are
compared byte for byte).  The card's name, power limit and maximum SM clock are read in the same run.
"""
import argparse
import os
import re
import subprocess
import sys
import time

for var in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):
  os.environ.setdefault(var, "1")
os.environ.setdefault("EDTB200_POOL_KEEP_MB", str(1 << 20))     # keep the pool's high-water mark

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import edt_b200 as edt  # noqa: E402
import torch  # noqa: E402
from edt_b200 import workloads  # noqa: E402

LINES = []
WORKLOADS = ("balls8", "voronoi32", "blocks32", "mask8", "voronoi32_4_4_40")


def say(line=""):
  print(line, flush=True)
  LINES.append(line)


def smi(fields):
  try:
    return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + fields, "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or "unknown"
  except Exception as e:
    return "unknown (%s)" % e


def volume(name, n):
  """(labels on the device, weights)."""
  if name == "balls8":
    return workloads.generate("balls", n, "cuda")[0], None
  if name.startswith("voronoi32"):
    return workloads.generate("voronoi", n, "cuda")[0], (None if name == "voronoi32" else (4.0, 4.0, 40.0))
  if name == "blocks32":
    g = torch.Generator(device="cuda")
    g.manual_seed(5)
    k = 32
    small = torch.randint(0, 1 << 20, (-(-n // k),) * 3, dtype=torch.int32, device="cuda", generator=g)
    return small.repeat_interleave(k, 0).repeat_interleave(k, 1).repeat_interleave(k, 2)[:n, :n, :n].contiguous(), None
  c = torch.arange(n, device="cuda", dtype=torch.float32) - (n - 1) / 2
  d2 = c.view(-1, 1, 1) ** 2 + c.view(1, -1, 1) ** 2 + c.view(1, 1, -1) ** 2
  return (d2 <= (0.4 * n) ** 2).to(torch.uint8), None


def timed(f, steps, warmup, rounds):
  for _ in range(warmup):
    f()
  torch.cuda.synchronize()
  acc = []
  for _ in range(rounds):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
      f()
    e.record()
    e.synchronize()
    acc.append(s.elapsed_time(e) / steps)
  return sorted(acc)[len(acc) // 2]


def extra_bytes(f):
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


def counts(name, n):
  """(rounds, cycles, steps) of one verbose call in a child process."""
  env = dict(os.environ, EDT_B200_VERBOSE="1")
  r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", name, "--n", str(n)], env=env,
                     capture_output=True, text=True)
  m = re.search(r"rounds (\d+)\s+cycles (\d+)\s+steps (\d+)", r.stderr)
  return tuple(int(v) for v in m.groups()) if m else ("?", "?", "?")


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--n_host", type=int, default=128)
  ap.add_argument("--steps", type=int, default=3)
  ap.add_argument("--warmup", type=int, default=1)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--out", default=None)
  ap.add_argument("--child", default=None)
  a = ap.parse_args()
  if a.child:
    t, w = volume(a.child, a.n)
    edt.skeletonize(t, w)
    torch.cuda.synchronize()
    return
  say("skeleton_bench: %s, power limit %s, max SM clock %s" % (smi("name"), smi("power.limit"), smi("clocks.max.sm")))
  say("n=%d, steps=%d warmup=%d rounds=%d; ms per call (median round); MiB of device memory beyond input and "
      "output; skeleton voxels per labelled voxel" % (a.n, a.steps, a.warmup, a.rounds))
  say("%-17s %9s %9s %9s %7s %7s %7s %7s %9s" % ("workload", "total", "edtsq", "thin", "rounds", "cycles", "steps",
                                                 "MiB", "skeleton"))
  for name in WORKLOADS:
    t, w = volume(name, a.n)
    got = edt.skeletonize(t, w)
    frac = float(got.sum()) / max(1.0, float((t != 0).sum()))
    del got
    total = timed(lambda: edt.skeletonize(t, w), a.steps, a.warmup, a.rounds)
    sq = timed(lambda: edt.edtsq(t, w), a.steps, a.warmup, a.rounds)
    mib = extra_bytes(lambda: edt.skeletonize(t, w)) / 2**20
    del t
    torch.cuda.empty_cache()
    r, c, s = counts(name, a.n)
    say("%-17s %9.2f %9.3f %9.2f %7s %7s %7s %7.0f %9.5f" % (name, total, sq, total - sq, r, c, s, mib, frac))
  import numpy as np
  import skeleton_cases as skc
  say()
  say("numpy restatement on one host thread against the GPU call, n_host=%d" % a.n_host)
  say("%-17s %12s %10s %8s %s" % ("workload", "restated s", "GPU ms", "x", "equal"))
  for name in WORKLOADS[:2]:
    t, w = volume(name, a.n_host)
    gpu_ms = timed(lambda: edt.skeletonize(t, w), a.steps, a.warmup, a.rounds)
    got = edt.skeletonize(t, w).cpu().numpy()
    host = t.cpu().numpy()
    t0 = time.perf_counter()
    want = skc.restate(host, w)
    sec = time.perf_counter() - t0
    say("%-17s %12.2f %10.3f %8.0f %s" % (name, sec, gpu_ms, sec * 1e3 / gpu_ms,
                                          "yes" if np.array_equal(got, want) else "NO"))
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
      fh.write("\n".join(LINES) + "\n")


if __name__ == "__main__":
  main()
