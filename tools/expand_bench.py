#!/usr/bin/env python
"""expand_labels on one GPU: the gather kernel (edtb200_expand_gather) against the chain of torch ops
that gathered the labels before it, and stacked calls against a Python loop of per-volume calls.

  python tools/expand_bench.py [--n 512] [--steps 10] [--warmup 2] [--rounds 3] [--reps 10] [--out FILE]

1. Device-resident n^3 volumes of tools/feature_bench.py (workloads.py: cfg2, cfg2b, cfg3, balls,
   voronoi), distance 2.5.  The torch gather is restated below (`torch_gather`) and runs on the same
   feature-transform output as the kernel; the two alternate over `rounds` rounds of `steps` calls each
   (CUDA events, after warm-up), and their results are compared byte for byte.  Timed twice: the
   gather alone, and the whole call (the signed feature transform and the gather).  The device memory
   beyond the labels is read as feature_bench.py reads it: the library's scratch pool keeps what it
   took (EDTB200_POOL_KEEP_MB) and torch's cache is emptied first, so the drop in free device memory
   over one call, its result still alive, is that call's peak.  For the gather alone the feature
   transform's outputs are held before the reading starts.
2. Device-resident stacks of the tools/stack_bench.py shapes (4096 x 128^2 uint8 masks, 1024 x 512^2
   uint32 slices, 64 x 64^3 uint8 balls), expand_labels(stacked=True) against a Python loop of
   per-volume calls; every stacked result is compared with the loop's.

The card's name, power limit and maximum SM clock are read in the same run, and the SM clock
nvidia-smi reads right after each timed loop of part 1 is printed beside it.
"""
import argparse
import ctypes
import os
import subprocess
import sys

os.environ.setdefault("EDTB200_POOL_KEEP_MB", str(1 << 20))     # keep the pool's high-water mark

import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import edt_b200 as edt  # noqa: E402
import torch  # noqa: E402
from stack_bench import balls, masks, segmentation  # noqa: E402

WORKLOADS = ("cfg2", "cfg2b", "cfg3", "balls", "voronoi")
DISTANCE = 2.5
LINES = []


def say(line=""):
  print(line, flush=True)
  LINES.append(line)


def smi(fields):
  try:
    return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + fields, "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or "unknown"
  except Exception as e:          # no nvidia-smi: say so rather than guess
    return "unknown (%s)" % e


def same_size_signed(t):
  for name, signed in (("uint16", torch.int16), ("uint32", torch.int32), ("uint64", torch.int64)):
    if t.dtype == getattr(torch, name, None):
      return t.view(signed)
  return t


def torch_gather(t, dist, idx, distance):
  """The gather expand_labels ran on the device before the kernel: an int64 C-order linear site index
  built axis by axis, a clamp, three masks, a float64 copy of |dist|, a gather, a where and a copy."""
  lin = torch.zeros(t.shape, dtype=torch.int64, device=t.device)
  step = 1
  for k in reversed(range(t.dim())):
    lin += idx[k].to(torch.int64) * step
    step *= int(t.shape[k])
  take = same_size_signed(t)
  grow = (take == 0) & (idx[0] >= 0) & (dist.abs().to(torch.float64) <= float(distance) ** 2)
  grown = torch.where(grow, take.reshape(-1)[lin.clamp(min=0)], take)
  out = torch.empty_like(t)
  same_size_signed(out).copy_(grown)
  return out


def signed_features(t, anisotropy):
  """(squared signed distances, index planes) of a device volume: the feature transform expand_labels runs."""
  v = edt._Volume("expand_bench", t).order()
  v.set_weights(anisotropy, positive=False, rule="first")
  return edt._feature(v, False, edt.FLAG_SIGNED, True)


def kernel_gather(t, dist, idx, distance):
  """edtb200_expand_gather on a C-contiguous volume and the feature transform's planes."""
  nd = t.dim()
  (sx, sy, sz), _ = edt._x_fastest(t.shape, (1.0,) * nd, False)
  ptrs = (ctypes.c_void_p * nd)(*[idx[nd - 1 - j].data_ptr() for j in range(nd)])
  out = torch.empty_like(t)
  flags = edt.FLAG_LABELS_ON_DEVICE | edt.FLAG_OUT_ON_DEVICE | (edt.FLAG_LABELS_FLOAT if t.is_floating_point() else 0)
  rc = edt._lib().edtb200_expand_gather(t.data_ptr(), t.element_size(), nd, sx, sy, sz, 1, dist.data_ptr(), ptrs,
                                        float(distance) ** 2, flags, out.data_ptr(), t.device.index,
                                        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
  if rc:
    raise RuntimeError(edt._lib().edtb200_last_error())
  return out


def bytes_equal(a, b):
  return a.shape == b.shape and a.dtype == b.dtype and torch.equal(same_size_signed(a), same_size_signed(b))


def timed(fn, steps):
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(steps):
    fn()
  stop.record()
  stop.synchronize()
  return start.elapsed_time(stop) / steps


def peak_gib(fn):
  torch.cuda.synchronize()
  edt.release()
  torch.cuda.empty_cache()
  free0 = torch.cuda.mem_get_info()[0]
  out = fn()
  torch.cuda.synchronize()
  mem = (free0 - torch.cuda.mem_get_info()[0]) / 2 ** 30
  del out
  return mem


def volume_rows(args):
  from edt_b200 import workloads
  say("1. %d^3 device-resident volumes, distance %.1f; CUDA events, %d rounds of %d calls after %d warm-up, the two "
      "sides alternating; ms/call is the median round [fastest, slowest]; mem = device memory beyond the labels, "
      "result included" % (args.n, DISTANCE, args.rounds, args.steps, args.warmup))
  say("%-8s %-7s %-13s %24s %9s  %-15s %s" % ("workload", "part", "side", "ms/call", "mem GiB", "SM clock after",
                                              "result"))
  ok = True
  for name in WORKLOADS:
    lab, an, _ = workloads.generate(name, args.n, "cuda")
    dist, idx = signed_features(lab, an)
    torch.cuda.synchronize()
    parts = (
      ("gather", (("kernel", lambda: kernel_gather(lab, dist, idx, DISTANCE)),
                  ("torch ops", lambda: torch_gather(lab, dist, idx, DISTANCE)))),
      ("whole", (("expand_labels", lambda: edt.expand_labels(lab, DISTANCE, an)),
                 ("feature+torch", lambda: torch_gather(lab, *signed_features(lab, an), DISTANCE)))),
    )
    for part, sides in parts:
      results = [fn() for _, fn in sides]
      same = bytes_equal(results[0], results[1])
      grown = int((results[0] != lab).sum())
      del results
      ok &= same
      mems = [peak_gib(fn) for _, fn in sides]
      for _, fn in sides:
        for _ in range(args.warmup):
          fn()
      times, clocks = [[] for _ in sides], [None for _ in sides]
      for _ in range(args.rounds):
        for i, (_, fn) in enumerate(sides):
          times[i].append(timed(fn, args.steps))
          clocks[i] = smi("clocks.sm")
      for i, (side, _) in enumerate(sides):
        t = sorted(times[i])
        say("%-8s %-7s %-13s %8.3f [%6.3f, %6.3f] %9.2f  %-15s %s" % (
          name, part, side, float(np.median(t)), t[0], t[-1], mems[i], clocks[i],
          ("byte-identical, %d voxels grew" % grown if same else "DIFFERENT") if i == 0 else ""))
    del lab, dist, idx
    torch.cuda.empty_cache()
  return ok


def device_ms(fn, reps):
  """Median of `reps` timings of fn() on the current stream, after two warm-up calls."""
  fn(); fn()
  torch.cuda.synchronize()
  times = []
  for _ in range(reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    times.append(a.elapsed_time(b))
  return float(np.median(times))


def stack_row(name, host, reps):
  t = torch.from_numpy(host.view(np.int32) if host.dtype == np.uint32 else host).cuda()
  got = {}

  def stacked():
    got["s"] = edt.expand_labels(t, DISTANCE, stacked=True)

  def loop():
    got["l"] = [edt.expand_labels(t[b], DISTANCE) for b in range(t.shape[0])]

  loop_reps = max(3, reps // 4)
  ms_s, ms_l = device_ms(stacked, reps), device_ms(loop, loop_reps)
  torch.cuda.synchronize()
  ok = bytes_equal(got["s"], torch.stack(got["l"]))
  vox = t.numel()
  say("%-30s %9.3f ms %10.3f ms %7.1fx %8.0f Mvox/s  %s" % (name, ms_s, ms_l, ms_l / ms_s, vox / ms_s / 1e3,
                                                             "equal" if ok else "DIFFERENT"))
  return ok


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--steps", type=int, default=10)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--reps", type=int, default=10)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  say("expand_bench: expand_labels' gather kernel against the torch-op gather, and stacked against a loop")
  say("card (name, power limit, maximum SM clock; read in this run): %s" % smi("name,power.limit,clocks.max.sm"))
  say("torch %s, CUDA %s" % (torch.__version__, torch.version.cuda))
  say()
  ok = volume_rows(args)
  say()
  rng = np.random.default_rng(0)
  loop_reps = max(3, args.reps // 4)
  say("2. device-resident stacks, distance %.1f (median of %d stacked calls / %d loops, CUDA events)" % (
    DISTANCE, args.reps, loop_reps))
  say("%-30s %12s %13s %8s %15s" % ("workload", "stacked", "loop", "speedup", "stacked rate"))
  ok &= stack_row("4096 x 128^2 uint8 masks", masks(rng, 4096, 128), args.reps)
  ok &= stack_row("1024 x 512^2 uint32 slices", segmentation(rng, 1024, 512), args.reps)
  ok &= stack_row("64 x 64^3 uint8 balls", balls(rng, 64, 64), args.reps)
  say()
  say("every kernel result byte-identical to the torch gather's, every stacked result equal to the loop's: %s"
      % ("yes" if ok else "NO"))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
      f.write("\n".join(LINES) + "\n")
  return 0 if ok else 1


if __name__ == "__main__":
  sys.exit(main())
