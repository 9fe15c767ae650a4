#!/usr/bin/env python
"""Stacked transforms (stacked=True, edtb200_transform_stack) against a Python loop of per-volume
calls, on one GPU:

  python tools/stack_bench.py [--out FILE] [--reps N]

Device-resident workloads (torch CUDA tensors, edt_cuda): 4096 x 128^2 uint8 masks, 1024 x 512^2
uint32 segmentation slices, 64 x 64^3 uint8 balls, 8 x 256^3 uint32 blocks.  Host workload: 512 x
1024^2 uint32 slices from pinned and from pageable memory, stacked against transform_batch and a loop
of edt2dsq.  Every stacked result is compared with the loop's bit for bit.  Also: kernel launches per
stacked call from torch.profiler at two stack sizes, and the stacked 2-D masks against one 8192^2 image
of the same 2^26 voxels.  The card's
name and power limit are read in the same run."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import edt_b200 as edt  # noqa: E402
import torch  # noqa: E402

LINES = []


def say(line=""):
  print(line, flush=True)
  LINES.append(line)


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                          "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    return out or "unknown"
  except Exception as e:          # no nvidia-smi: say so rather than guess
    return "unknown (%s)" % e


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


def host_ms(fn, reps):
  fn()
  times = []
  for _ in range(reps):
    t0 = time.perf_counter()
    fn()
    times.append((time.perf_counter() - t0) * 1e3)
  return float(np.median(times))


def masks(rng, n, size):
  """Random discs on a background: binary masks, as for a distance-map loss."""
  yy, xx = np.mgrid[:size, :size]
  out = np.zeros((n, size, size), np.uint8)
  for b in range(n):
    for _ in range(3):
      cy, cx, r = rng.integers(0, size, 2).tolist() + [int(rng.integers(size // 16, size // 4))]
      out[b][(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = 1
  return out


def segmentation(rng, n, size, cell=16):
  """uint32 label slices of cell-sized blocks (an oversegmentation's look), a little background."""
  small = rng.integers(0, 1 << 20, (n, size // cell + 1, size // cell + 1)).astype(np.uint32)
  out = np.repeat(np.repeat(small, cell, 1), cell, 2)[:, :size, :size]
  out[:, ::37, :] = 0
  return np.ascontiguousarray(out)


def balls(rng, n, size):
  zz, yy, xx = np.ogrid[:size, :size, :size]
  out = np.zeros((n, size, size, size), np.uint8)
  for b in range(n):
    c = rng.integers(size // 4, 3 * size // 4, 3)
    r = int(rng.integers(size // 6, size // 3))
    out[b][(zz - c[0]) ** 2 + (yy - c[1]) ** 2 + (xx - c[2]) ** 2 < r * r] = 1
  return out


def blocks3(rng, n, size, cell=8):
  small = rng.integers(0, 1 << 20, (n, size // cell, size // cell, size // cell)).astype(np.uint32)
  return np.ascontiguousarray(np.repeat(np.repeat(np.repeat(small, cell, 1), cell, 2), cell, 3))


def bits_equal(a, b):
  return torch.equal(a.view(torch.int32), b.view(torch.int32))


def device_row(name, host, reps):
  t = torch.from_numpy(host.view(np.int32) if host.dtype == np.uint32 else host).cuda()
  out = torch.empty(t.shape, dtype=torch.float32, device=t.device)
  loop_out = torch.empty_like(out)

  def stacked():
    edt.edt_cuda(t, out=out, stacked=True)

  def loop():
    for b in range(t.shape[0]):
      edt.edt_cuda(t[b], out=loop_out[b])

  ms_s, ms_l = device_ms(stacked, reps), device_ms(loop, max(3, reps // 4))
  torch.cuda.synchronize()
  ok = bits_equal(out, loop_out)
  vox = t.numel()
  say("%-34s %9.3f ms %9.3f ms %7.1fx %8.0f Mvox/s  %s" % (name, ms_s, ms_l, ms_l / ms_s, vox / ms_s / 1e3,
                                                              "equal" if ok else "DIFFERENT"))
  return ok


def launches(small, big):
  """CUDA kernels of this library that one stacked call launches at each of two stack sizes, from one
  torch.profiler session; a torch kernel between the two calls separates them."""
  from torch.profiler import profile, ProfilerActivity
  outs = [torch.empty(t.shape, dtype=torch.float32, device=t.device) for t in (small, big)]
  marker = torch.zeros(1, device=small.device)
  for t, o in zip((small, big), outs):
    edt.edt_cuda(t, out=o, stacked=True)                  # step tables built outside the session
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    edt.edt_cuda(small, out=outs[0], stacked=True)
    torch.cuda.synchronize()
    marker.add_(1)
    torch.cuda.synchronize()
    edt.edt_cuda(big, out=outs[1], stacked=True)
    torch.cuda.synchronize()
  kernels = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and "memcpy" not in e.name.lower()
                    and "memset" not in e.name.lower()), key=lambda e: e.time_range.start)
  cut = next(i for i, e in enumerate(kernels) if "edtb200" not in e.name)
  return (sum("edtb200" in e.name for e in kernels[:cut]), sum("edtb200" in e.name for e in kernels[cut + 1:]))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None)
  ap.add_argument("--reps", type=int, default=20)
  args = ap.parse_args()
  rng = np.random.default_rng(0)
  say("stack_bench: stacked=True against a Python loop of per-volume calls, one GPU")
  say("card: %s (name, power limit, max SM clock; read in this run)" % card())
  say("torch %s, CUDA %s" % (torch.__version__, torch.version.cuda))
  say()
  say("device-resident (edt_cuda, edtsq; median of %d stacked calls / %d loops, CUDA events)" % (args.reps,
                                                                                             max(3, args.reps // 4)))
  say("%-34s %12s %12s %8s %15s" % ("workload", "stacked", "loop", "speedup", "stacked rate"))
  ok = True
  m = masks(rng, 4096, 128)
  ok &= device_row("4096 x 128^2 uint8 masks", m, args.reps)
  ok &= device_row("1024 x 512^2 uint32 slices", segmentation(rng, 1024, 512), args.reps)
  ok &= device_row("64 x 64^3 uint8 balls", balls(rng, 64, 64), args.reps)
  ok &= device_row("8 x 256^3 uint32 blocks", blocks3(rng, 8, 256), args.reps)
  say()
  # one 8192^2 image of the same 2^26 voxels
  big = torch.from_numpy(masks(rng, 1, 8192)[0]).cuda()
  big_out = torch.empty(big.shape, dtype=torch.float32, device=big.device)
  ms_big = device_ms(lambda: edt.edt_cuda(big, out=big_out), args.reps)
  tm = torch.from_numpy(m).cuda()
  tm_out = torch.empty(tm.shape, dtype=torch.float32, device=tm.device)
  ms_m = device_ms(lambda: edt.edt_cuda(tm, out=tm_out, stacked=True), args.reps)
  say("same voxels: 4096 x 128^2 uint8 masks stacked %.3f ms, one 8192^2 uint8 image %.3f ms (%.3fx); the image's"
      % (ms_m, ms_big, ms_m / ms_big))
  say("  8192-voxel rows take the generic X kernel and its 8192-row columns the long-line Y kernel")
  n_small, n_big = launches(tm[:64].contiguous(), tm)
  say("kernel launches per stacked call (torch.profiler): %d at 64 masks, %d at 4096 masks" % (n_small, n_big))
  ok &= n_small == n_big
  say()
  # host: 512 x 1024^2 uint32 per-slice transforms
  host = segmentation(rng, 512, 1024)
  pinned = torch.empty(host.shape, dtype=torch.int32, pin_memory=True).numpy().view(np.uint32)
  pinned[...] = host
  pinned_out = [torch.empty((1024, 1024), dtype=torch.float32, pin_memory=True).numpy() for _ in range(512)]
  say("host 512 x 1024^2 uint32 slices, edtsq (median of %d, wall clock)" % max(3, args.reps // 4))
  say("%-34s %12s %12s %12s" % ("memory", "stacked", "batch", "edt2dsq loop"))
  want = None
  for name, src, outs in (("pinned", pinned, pinned_out), ("pageable", host, None)):
    got = {}
    ms_s = host_ms(lambda: got.__setitem__("s", edt.edtsq(src, stacked=True)), max(3, args.reps // 4))
    ms_b = host_ms(lambda: got.__setitem__("b", edt.transform_batch(list(src), outs=outs)), max(3, args.reps // 4))
    ms_l = host_ms(lambda: got.__setitem__("l", [edt.edt2dsq(v) for v in src]), max(3, args.reps // 4))
    want = np.stack(got["l"]) if want is None else want
    same = all(np.array_equal(x.view(np.uint32), want.view(np.uint32))
               for x in (got["s"], np.stack(got["b"]), np.stack(got["l"])))
    ok &= same
    say("%-34s %9.1f ms %9.1f ms %9.1f ms  %s" % (name, ms_s, ms_b, ms_l, "equal" if same else "DIFFERENT"))
  say()
  say("all stacked results equal the per-volume calls bit for bit: %s" % ("yes" if ok else "NO"))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
      f.write("\n".join(LINES) + "\n")
  return 0 if ok else 1


if __name__ == "__main__":
  sys.exit(main())
