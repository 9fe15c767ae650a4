#!/usr/bin/env python
"""Device time of hausdorff_distance(percentile=95) and surface_dice on the GPU, against the numpy / scipy
restatement of tests/surface_cases.py on the CPU, with the outputs compared.

Workloads (a prediction against a reference):
  voronoi512   one 512^3 volume of 200 Voronoi cells (uint32) against the cells of the same seeds moved
               by up to 2 voxels along each axis: 200 keys, 400 slots of 512^3
  stack256     4 x 256^3 (stacked=True) of 8 Voronoi cells each, against the same perturbation: 64 slots
The scipy restatement transforms one full volume per key and direction, minutes for the 512^3 case, so
it runs on the first --scipy-keys keys of voronoi512 and on the first volume of stack256; the GPU is
compared on exactly those keys and volumes (rtol 1e-12).

  python tools/surface_bench.py [--reps 3] [--scipy-keys 2] [--out FILE]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import edt_b200 as edt  # noqa: E402
import surface_cases as sc  # noqa: E402


def voronoi(torch, shape, seeds):
  """int32 labels 1..len(seeds) of the nearest seed, slice by slice on the GPU."""
  nz, ny, nx = shape
  yy, xx = torch.meshgrid(torch.arange(ny, device="cuda", dtype=torch.float32),
                          torch.arange(nx, device="cuda", dtype=torch.float32), indexing="ij")
  out = torch.empty(shape, dtype=torch.int32, device="cuda")
  for z in range(nz):
    d = ((seeds[:, 0].view(-1, 1, 1) - z) ** 2 + (seeds[:, 1].view(-1, 1, 1) - yy) ** 2 +
         (seeds[:, 2].view(-1, 1, 1) - xx) ** 2)
    out[z] = d.argmin(0).to(torch.int32) + 1
  return out


def pair(torch, shape, nseeds, gen):
  seeds = torch.rand((nseeds, 3), device="cuda", generator=gen) * torch.tensor(shape, device="cuda")
  moved = seeds + (torch.rand((nseeds, 3), device="cuda", generator=gen) * 4 - 2)
  return voronoi(torch, shape, moved), voronoi(torch, shape, seeds)


def timed(torch, fn, reps):
  fn()
  torch.cuda.synchronize()
  ms = []
  for _ in range(reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    out = fn()
    end.record()
    torch.cuda.synchronize()
    ms.append(start.elapsed_time(end))
  return out, ms


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--scipy-keys", type=int, default=2)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  import torch
  if not torch.cuda.is_available():
    raise SystemExit("surface_bench: no CUDA device")
  lines = []

  def say(s):
    print(s, flush=True)
    lines.append(s)

  gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  say("GPU: %s" % gpu)
  gen = torch.Generator(device="cuda")
  gen.manual_seed(0)
  work = [("voronoi512", pair(torch, (512, 512, 512), 200, gen), False)]
  a4, b4 = zip(*[pair(torch, (256, 256, 256), 8, gen) for _ in range(4)])
  work.append(("stack256", (torch.stack(a4), torch.stack(b4)), True))
  for name, (a, b), stacked in work:
    sd = edt.surface_distances(a, b, stacked=stacked)
    keys = sd.labels.cpu().numpy()
    nseg = sd.offsets.numel() - 1
    say("%s: shape %s, %d keys, %d segments, %d surface distances" % (name, tuple(a.shape), len(keys), nseg,
                                                                     sd.values.numel()))
    del sd
    kw = dict(stacked=stacked)
    hd95, ms_hd = timed(torch, lambda: edt.hausdorff_distance(a, b, percentile=95, **kw), args.reps)
    dice, ms_dice = timed(torch, lambda: edt.surface_dice(a, b, 1.0, **kw), args.reps)
    _, ms_sd = timed(torch, lambda: edt.surface_distances(a, b, **kw), args.reps)
    say("  GPU surface_distances            ms: %s" % " ".join("%.1f" % m for m in ms_sd))
    say("  GPU hausdorff_distance(p=95)     ms: %s" % " ".join("%.1f" % m for m in ms_hd))
    say("  GPU surface_dice(tolerance=1)    ms: %s" % " ".join("%.1f" % m for m in ms_dice))
    # the scipy restatement on a part, and the GPU on the same part
    if stacked:
      na, nb = a[0].cpu().numpy(), b[0].cpu().numpy()
      part, what = keys, "volume 0, all %d keys" % len(keys)
      want_hd, want_dice = hd95.cpu().numpy()[0], dice.cpu().numpy()[0]
    else:
      na, nb = a.cpu().numpy(), b.cpu().numpy()
      part = keys[:args.scipy_keys]
      what = "keys %s of %d" % ([int(k) for k in part], len(keys))
      want_hd, want_dice = hd95.cpu().numpy()[:len(part)], dice.cpu().numpy()[:len(part)]
    t0 = time.perf_counter()
    segs = sc.segments(na, nb, part, (1.0, 1.0, 1.0))
    ref_hd = np.array([sc.hausdorff(x, y, percentile=95) for x, y in segs])
    ref_dice = np.array([sc.dice(x, y, 1.0) for x, y in segs])
    cpu_s = time.perf_counter() - t0
    ok = np.allclose(want_hd, ref_hd, rtol=1e-12, atol=0) and np.allclose(want_dice, ref_dice, rtol=1e-12, atol=0)
    say("  scipy restatement (%s): %.1f s for both metrics (%.2f s per key)" % (what, cpu_s, cpu_s / len(part)))
    say("  outputs equal to the restatement (rtol 1e-12): %s" % ok)
    say("  hd95 %s  dice %s" % (np.array2string(ref_hd[:4], precision=4), np.array2string(ref_dice[:4], precision=4)))
    if not ok:
      say("  GPU hd95 %s  dice %s" % (want_hd[:8], want_dice[:8]))
  if args.out:
    with open(args.out, "w") as f:
      f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
  main()
