#!/usr/bin/env python
"""What nearest_labels costs, on one GPU.

  python tools/nearest_labels_bench.py [--n 512] [--steps 3] [--warmup 2] [--rounds 5] [--no-compose] [--out FILE]

Device-resident n^3 label volumes: a Voronoi partition of 200 seeds (int32), random labels in blocks of 32^3
(int32), 64 balls each with its own label on background (uint8), and iid label noise (int32, 0..255).  For
each, max_distance d in {2.5, 8, 24} and k in {1, 2, 4}: the median ms per call over `rounds` rounds of
`steps` calls (CUDA events after warm-up; the k values of one workload and d alternate round by round), the
device memory beyond input and outputs (the drop in free memory over one call with everything released
first), and the bytes the passes move per voxel with the HBM floor that gives at the data-sheet 3.35 TB/s.
Unless --no-compose, at 256^3 Voronoi: the composition a user has without nearest_labels -- one bounded
edtsq per label of that label's mask, stacked, then a torch sort -- against nearest_labels, with the values
checked equal.  The card's name, power limit and maximum SM clock are read in the same run.
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

LINES = []
HBM = 3.35e12


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
  if name == "voronoi":
    return workloads.generate("voronoi", n, "cuda")[0]
  if name == "blocks32":
    return workloads.generate("cfg2b", n, "cuda")[0]
  if name == "noise":
    return workloads.generate("cfg2", n, "cuda")[0]
  g = torch.Generator(device="cuda")
  g.manual_seed(0)
  ax = torch.arange(n, device="cuda", dtype=torch.float32)
  z, y, x = ax.view(n, 1, 1), ax.view(1, n, 1), ax.view(1, 1, n)
  lab = torch.zeros((n,) * 3, dtype=torch.uint8, device="cuda")
  c = torch.rand((64, 3), device="cuda", generator=g) * n
  r = (40 + 50 * torch.rand((64,), device="cuda", generator=g)) * (n / 512.0)
  for b in range(64):
    inside = ((z - c[b, 0]) ** 2 + (y - c[b, 1]) ** 2 + (x - c[b, 2]) ** 2) <= r[b] ** 2
    lab = torch.where(inside, torch.full_like(lab, b + 1), lab)
  return lab


def timed(f, steps, warmup):
  for _ in range(warmup):
    f()
  torch.cuda.synchronize()
  s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  s.record()
  for _ in range(steps):
    f()
  e.record()
  e.synchronize()
  return s.elapsed_time(e) / steps


def extra_bytes(call):
  torch.cuda.synchronize()
  edt.release()
  torch.cuda.empty_cache()
  free0 = torch.cuda.mem_get_info()[0]
  res = call()
  torch.cuda.synchronize()
  free1 = torch.cuda.mem_get_info()[0]
  return max(0, free0 - free1 - sum(o.numel() * o.element_size() for o in res))


def moved_bytes(k, lb):
  """Bytes per voxel the three passes read and write: X reads the labels and writes k entries, Y and Z each
  read and write k entries (4 + lb bytes each)."""
  entry = k * (4 + lb)
  return lb + entry + 4 * entry


def compose(lab, d, k):
  """The composition without nearest_labels: one bounded edtsq per label's mask, stacked, then sorted."""
  ids = torch.unique(lab)
  ids = ids[ids != 0]
  per = torch.stack([edt.edtsq((lab != m).to(torch.uint8), max_distance=d) for m in ids.tolist()]).view(len(ids), -1)
  v = torch.empty((k, per.shape[1]), device=per.device)
  step = 1 << 22                                # sorted in slices of voxels, so that the indices fit beside it
  for s in range(0, per.shape[1], step):
    v[:, s:s + step] = torch.sort(per[:, s:s + step], dim=0, stable=True).values[:k]
  return v.view((k,) + tuple(lab.shape)), None


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--steps", type=int, default=3)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--no-compose", action="store_true")
  ap.add_argument("--out")
  a = ap.parse_args()
  say("# card: %s | power limit: %s | max SM clock: %s" % (smi("name"), smi("power.limit"), smi("clocks.max.sm")))
  say("# nearest_labels, device-resident n=%d; median ms per call of %d rounds x %d calls (spread: min-max of the "
      "rounds), the (d, k) cases of a workload alternating round by round; extra = device memory beyond input and "
      "outputs; floor = moved bytes at 3.35 TB/s" % (a.n, a.rounds, a.steps))
  cases = [(d, k) for d in (2.5, 8.0, 24.0) for k in (1, 2, 4)]
  for name in ("voronoi", "blocks32", "balls64", "noise"):
    lab = volume(name, a.n)
    lb = lab.element_size()
    times = {c: [] for c in cases}
    for r in range(a.rounds):
      for d, k in cases:
        times[(d, k)].append(timed(lambda: edt.nearest_labels(lab, d, k=k), a.steps, a.warmup if r == 0 else 0))
    for d, k in cases:
      t = sorted(times[(d, k)])
      extra = extra_bytes(lambda: edt.nearest_labels(lab, d, k=k))
      _, variant = plan(lab.shape, d, k, lb)
      mb = moved_bytes(k, lb)
      floor = mb * lab.numel() / HBM * 1e3
      say("%-9s %s d=%-4g k=%d  %9.3f ms (%.3f-%.3f)  extra %5d MiB  moved %3d B/voxel  floor %6.2f ms (%3.0f%%)  "
          "passes %s" % (name, lab.dtype, d, k, t[len(t) // 2], t[0], t[-1], extra >> 20, mb, floor,
                         100.0 * floor / t[len(t) // 2], variant))
    del lab
    torch.cuda.empty_cache()
  if not a.no_compose:
    n = 256
    lab = workloads.generate("voronoi", n, "cuda")[0]
    for d, k in ((8.0, 2), (24.0, 4)):
      ours = edt.nearest_labels(lab, d, k=k, squared=True)
      theirs = compose(lab, d, k)
      same = bool(torch.equal(ours[0].view(torch.int32), theirs[0].view(torch.int32)))
      t_ours = sorted(timed(lambda: edt.nearest_labels(lab, d, k=k, squared=True), a.steps, 1) for _ in range(3))[1]
      t_comp = timed(lambda: compose(lab, d, k), 1, 0)
      peak0 = torch.cuda.max_memory_allocated()
      say("compose   voronoi %d^3 d=%g k=%d: nearest_labels %8.3f ms, %d bounded edtsq + sort %9.1f ms (x%.0f), "
          "values equal: %s, torch peak %d MiB" % (n, d, k, t_ours, int(torch.unique(lab).numel()), t_comp,
                                                    t_comp / t_ours, same, peak0 >> 20))
      del ours, theirs
      torch.cuda.empty_cache()
  if a.out:
    with open(a.out, "w") as fh:
      fh.write("\n".join(LINES) + "\n")


def plan(shape, d, k, lb):
  import ctypes
  radius = (ctypes.c_int64 * 3)()
  variant = (ctypes.c_int * 3)()
  z, y, x = shape
  edt._check(edt._lib().edtb200_nearest_labels_plan(3, x, y, z, 1.0, 1.0, 1.0, d, k, lb, radius, variant))
  names = {0: "rows", 1: "staged", 2: "global", -1: "-"}
  return list(radius), "/".join("%s(R=%d)" % (names[v], r) for v, r in zip(variant, radius))


if __name__ == "__main__":
  main()
