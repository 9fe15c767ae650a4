#!/usr/bin/env python
"""What the indices of parabolic erosion and dilation cost, on one GPU.

  python tools/parabolic_sites_bench.py [--n 512] [--steps 5] [--rounds 5] [--seeds 4000] [--no-big] [--out FILE]

Device-resident float32 n^3 volumes: the four workloads of tools/parabolic_bench.py (mask64, uniform,
smooth, reverse; each eroded and dilated), a power diagram (`seeds` seeds at random voxels with integer
weights omega in [0, 400): -omega on the seeds, +inf elsewhere, eroded), and unless --no-big 1024^3
uniform noise eroded.  For each: the call without and with return_indices=True, alternating round by
round (median ms per call over `rounds` rounds of `steps` calls, CUDA events after warm-up), the device
memory each takes beyond its input and outputs (the drop in free memory over one call with everything
released first), and whether the values are byte-identical with and without indices.  The card's name,
power limit and maximum SM clock are read in the same run.
"""
import argparse
import os
import sys

os.environ.setdefault("EDTB200_POOL_KEEP_MB", str(1 << 20))     # keep the pool's high-water mark

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import edt_b200 as edt  # noqa: E402
import torch  # noqa: E402
from parabolic_bench import case_volume, smi, timed  # noqa: E402

LINES = []


def say(line=""):
  print(line, flush=True)
  LINES.append(line)


def power_volume(n, seeds):
  g = torch.Generator(device="cuda")
  g.manual_seed(2)
  f = torch.full((n,) * 3, float("inf"), device="cuda")
  at = torch.randperm(n ** 3, generator=g, device="cuda")[:seeds]
  f.view(-1)[at] = -torch.randint(0, 400, (seeds,), generator=g, device="cuda").to(torch.float32)
  return f


def extra_bytes(call):
  torch.cuda.synchronize()
  edt.release()
  torch.cuda.empty_cache()
  free0 = torch.cuda.mem_get_info()[0]
  res = call()
  torch.cuda.synchronize()
  free1 = torch.cuda.mem_get_info()[0]
  outs = res if isinstance(res, tuple) else (res,)
  return max(0, free0 - free1 - sum(o.numel() * o.element_size() for o in outs))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--steps", type=int, default=5)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--seeds", type=int, default=4000)
  ap.add_argument("--no-big", action="store_true")
  ap.add_argument("--out")
  a = ap.parse_args()
  say("# card: %s | power limit: %s | max SM clock: %s" % (smi("name"), smi("power.limit"), smi("clocks.max.sm")))
  say("# device-resident float32; median ms per call of %d rounds x %d calls, the two calls alternating round by "
      "round; extra = device memory beyond input and outputs" % (a.rounds, a.steps))
  cases = [(name, a.n, op) for name in ("mask64", "uniform", "smooth", "reverse") for op in ("erode", "dilate")]
  cases.append(("power", a.n, "erode"))
  if not a.no_big:
    cases.append(("uniform", 1024, "erode"))
  for name, n, op in cases:
    f = power_volume(n, a.seeds) if name == "power" else case_volume(name, n)
    fn = getattr(edt, "parabolic_" + op)
    plain = lambda: fn(f)                                         # noqa: E731
    sites = lambda: fn(f, return_indices=True)                   # noqa: E731
    times = {"plain": [], "sites": []}
    steps = a.steps if n < 1024 else 1
    for r in range(a.rounds):
      for key, call in (("plain", plain), ("sites", sites)):
        times[key].append(timed(call, steps, a.warmup if r == 0 else 1, 1))
    ms = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    extra = {"plain": extra_bytes(plain), "sites": extra_bytes(sites)}
    v0 = plain()
    v1, idx = sites()
    same = bool(torch.equal(v0.view(torch.int32), v1.view(torch.int32)))
    none = int((idx[0] < 0).sum().item())
    del v0, v1, idx
    shape = "x".join(str(s) for s in f.shape)
    label = "power %d" % a.seeds if name == "power" else name
    say("%-10s %-6s %-13s plain %9.3f ms  indices %9.3f ms  (x%.2f)  extra %5d / %5d MiB  values identical: %s  "
        "no site: %d" % (label, op, shape, ms["plain"], ms["sites"], ms["sites"] / ms["plain"],
                         extra["plain"] >> 20, extra["sites"] >> 20, same, none))
    del f
    torch.cuda.empty_cache()
  if a.out:
    with open(a.out, "w") as fh:
      fh.write("\n".join(LINES) + "\n")


if __name__ == "__main__":
  main()
