#!/usr/bin/env python
"""Parabolic erosion and dilation on one GPU.

  python tools/parabolic_bench.py [--n 512] [--steps 5] [--warmup 2] [--rounds 3] [--big] [--out FILE]

Device-resident float32 n^3 volumes (and with --big the 1024^3 uniform case and a 20000^2 image, whose
lines take the long-line hull):
  mask64     0 on the background of the 64-balls workload (workloads.py), +inf on the balls: the erosion
             is edtsq of that mask, timed against edtsq of the same uint8 mask (outputs compared)
  uniform    uniform random floats in [0, 1000)
  smooth     a sum of 16 Gaussians
  reverse    the reverse distance transform of a sparse radius map: dilation of r^2 at 0.1 % of the
             voxels (r uniform in [2, 12]), -inf elsewhere
each eroded and dilated.  Per case: the tile kernels at 1, 2 and 4 warps per CTA
(EDTB200_PARABOLIC_WARPS; the settings alternate round by round, median round), then at the default:
the median ms per call over `rounds` rounds of `steps` calls (CUDA
events, after warm-up), the per-pass ms and kernels (one call in a child process with
EDT_B200_VERBOSE=1), the device memory beyond input and output (the drop in free memory over one call
with everything released first, less the output), and the fraction of the HBM floor: 8 bytes per voxel
per pass at 3.35 TB/s (the H100 SXM data sheet) over the measured time.  The card's name, power limit
and maximum SM clock are read in the same run.
"""
import argparse
import os
import subprocess
import sys

os.environ.setdefault("EDTB200_POOL_KEEP_MB", str(1 << 20))     # keep the pool's high-water mark

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import edt_b200 as edt  # noqa: E402
import torch  # noqa: E402
from edt_b200 import workloads  # noqa: E402

HBM = 3.35e12
WARPS = (1, 2, 4)
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


def case_volume(name, n):
  g = torch.Generator(device="cuda")
  g.manual_seed(1)
  if name == "mask64":
    balls = workloads.generate("balls", n, "cuda")[0]
    return torch.where(balls != 0, float("inf"), 0.0).to(torch.float32)
  if name == "uniform":
    return torch.rand((n,) * 3, generator=g, device="cuda") * 1000.0
  if name == "uniform2d":
    return torch.rand((n, n), generator=g, device="cuda") * 1000.0
  if name == "smooth":
    c = torch.arange(n, device="cuda", dtype=torch.float32)
    f = torch.zeros((n,) * 3, device="cuda")
    for _ in range(16):
      mu = torch.rand(3, generator=g, device="cuda") * n
      s = 0.05 * n + torch.rand(1, generator=g, device="cuda").item() * 0.1 * n
      gz = torch.exp(-((c - mu[0]) / s) ** 2 / 2).view(-1, 1, 1)
      gy = torch.exp(-((c - mu[1]) / s) ** 2 / 2).view(1, -1, 1)
      gx = torch.exp(-((c - mu[2]) / s) ** 2 / 2).view(1, 1, -1)
      f += 100.0 * gz * gy * gx
    return f
  if name == "reverse":
    r = 2.0 + 10.0 * torch.rand((n,) * 3, generator=g, device="cuda")
    medial = torch.rand((n,) * 3, generator=g, device="cuda") < 1e-3
    return torch.where(medial, r * r, float("-inf"))
  raise ValueError(name)


def timed(f, steps, warmup, rounds):
  for _ in range(warmup):
    f()
  torch.cuda.synchronize()
  ms = []
  for _ in range(rounds):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
      f()
    e.record()
    e.synchronize()
    ms.append(s.elapsed_time(e) / steps)
  return sorted(ms)[len(ms) // 2]


def extra_bytes(f):
  torch.cuda.synchronize()
  edt.release()
  torch.cuda.empty_cache()
  free0 = torch.cuda.mem_get_info()[0]
  out = f()
  torch.cuda.synchronize()
  free1 = torch.cuda.mem_get_info()[0]
  return max(0, free0 - free1 - out.numel() * out.element_size())


def per_pass(name, n, op):
  """One call in a child process with EDT_B200_VERBOSE=1: the library's per-pass line."""
  env = dict(os.environ, EDT_B200_VERBOSE="1")
  res = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", name, "--n", str(n), "--op", op],
                       env=env, capture_output=True, text=True, timeout=1800)
  lines = [ln for ln in res.stderr.splitlines() if "parabolic" in ln]
  return lines[-1].split("] ", 1)[-1] if lines else "no per-pass line (rc %d): %s" % (res.returncode, res.stderr[-300:])


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--steps", type=int, default=5)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--big", action="store_true")
  ap.add_argument("--out")
  ap.add_argument("--one")
  ap.add_argument("--op", default="erode")
  a = ap.parse_args()
  if a.one:
    f = case_volume(a.one, a.n)
    getattr(edt, "parabolic_" + a.op)(f)
    torch.cuda.synchronize()
    return
  say("# card: %s | power limit: %s | max SM clock: %s" % (smi("name"), smi("power.limit"), smi("clocks.max.sm")))
  say("# device-resident float32, median ms per call of %d rounds x %d calls; floor = 8 B/voxel/pass at 3.35 TB/s"
      % (a.rounds, a.steps))
  cases = [(name, a.n, op) for name in ("mask64", "uniform", "smooth", "reverse") for op in ("erode", "dilate")]
  if a.big:
    cases += [("uniform", 1024, "erode"), ("uniform2d", 20000, "erode")]
  for name, n, op in cases:
    f = case_volume(name, n)
    passes = f.dim()
    call = lambda: getattr(edt, "parabolic_" + op)(f)              # noqa: E731
    steps = a.steps if name != "uniform2d" else 1
    floor = 8.0 * f.numel() * passes / HBM * 1e3
    shape = "x".join(str(s) for s in f.shape)
    if name != "uniform2d":                    # the tile kernels at 1, 2 and 4 warps per CTA
      sweep = {}
      for _ in range(a.rounds):
        for warps in WARPS:
          os.environ["EDTB200_PARABOLIC_WARPS"] = str(warps)
          sweep.setdefault(warps, []).append(timed(call, steps, a.warmup, 1))
      os.environ.pop("EDTB200_PARABOLIC_WARPS")
      say("%-9s %-6s %-15s %s" % (name, op, shape, "  ".join(
          "%d warp%s %8.3f ms" % (w, "s" if w > 1 else " ", sorted(v)[len(v) // 2]) for w, v in sweep.items())))
    ms = timed(call, steps, 1 if name == "uniform2d" else a.warmup, a.rounds)
    extra = extra_bytes(call)
    say("%-9s %-6s %-15s %9.3f ms  floor %.3f ms (%.0f%% of floor)  extra %d MiB  (default)" %
        (name, op, shape, ms, floor, 100.0 * floor / ms, extra >> 20))
    if name == "mask64" and op == "erode":
      mask = (f != 0).to(torch.uint8)
      ms_e = timed(lambda: edt.edtsq(mask), a.steps, a.warmup, a.rounds)
      same = bool(torch.equal(call().view(torch.int32), edt.edtsq(mask).view(torch.int32)))
      say("%-9s %-6s %-15s %9.3f ms  (edtsq of the same uint8 mask; outputs bit-equal: %s)" % (name, "edtsq", shape, ms_e, same))
      del mask
    say("          per pass: %s" % per_pass(name, n, op))
    del f
    torch.cuda.empty_cache()
  if a.out:
    with open(a.out, "w") as fh:
      fh.write("\n".join(LINES) + "\n")


if __name__ == "__main__":
  main()
