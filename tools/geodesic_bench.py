#!/usr/bin/env python
"""geodesic_distance on one GPU: distances alone and with indices, the rounds each phase took, and scipy's
Dijkstra on the same definition for scale.

  python tools/geodesic_bench.py [--n 512] [--n_host 96] [--steps 3] [--warmup 1] [--rounds 3] [--out FILE]

Device-resident n^3 inputs:
  ball          an 8-bit ball mask (radius 0.45 n) seeded at its centre
  voronoi       32-bit Voronoi cells of 200 sites, one seed per cell at its site
  blocks        32-bit labels in 32^3 blocks, one seed per block at its low corner
  maze          an 8-bit serpentine maze: walls of label 0 across every 8th y row, open at alternate ends,
                extruded along z, seeded at one corner
  voronoi_aniso the Voronoi cells with weights (4, 4, 40)
For each (CUDA events around each round of `steps` calls, after warm-up; the median round):
  dist      edt.geodesic_distance(labels, seeds) in ms per call
  indices   the same with return_indices=True
  rounds / visits   of the distance phase and the index phase, from one EDT_B200_VERBOSE=1 call in a child
            process (tile visits: the tiles relaxed, summed over the rounds)
  MiB       device memory taken beyond the inputs and the outputs by the call with indices (the drop in free
            device memory over one call with everything released first)
Then scipy.sparse.csgraph.dijkstra on the graph of the definition (tests/geodesic_cases.py) at n_host^3
against the GPU call at that size, with distances and index planes compared bit for bit.  The card's name,
power limit and maximum SM clock are read in the same run.
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

LINES = []
WORKLOADS = ("ball", "voronoi", "blocks", "maze", "voronoi_aniso")


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
  """(labels, seeds, weights) on the device, (z, y, x) C order."""
  g = torch.Generator(device="cuda")
  g.manual_seed(0)
  seeds = torch.zeros((n, n, n), dtype=torch.uint8, device="cuda")
  if name == "ball":
    c = torch.arange(n, device="cuda", dtype=torch.float32) - (n - 1) / 2
    d2 = c.view(-1, 1, 1) ** 2 + c.view(1, -1, 1) ** 2 + c.view(1, 1, -1) ** 2
    seeds[n // 2, n // 2, n // 2] = 1
    return (d2 <= (0.45 * n) ** 2).to(torch.uint8), seeds, None
  if name.startswith("voronoi"):
    z = torch.arange(n, device="cuda", dtype=torch.float32).view(n, 1, 1)
    y = z.view(1, n, 1)
    x = z.view(1, 1, n)
    c = torch.rand((200, 3), device="cuda", generator=g) * n
    best = torch.full((n, n, n), float("inf"), device="cuda")
    lab = torch.zeros((n, n, n), dtype=torch.int32, device="cuda")
    for k in range(200):
      d = (z - c[k, 0]) ** 2 + (y - c[k, 1]) ** 2 + (x - c[k, 2]) ** 2
      m = d < best
      best = torch.where(m, d, best)
      lab = torch.where(m, torch.full_like(lab, k + 1), lab)
    at = c.long().clamp(0, n - 1)
    seeds[at[:, 0], at[:, 1], at[:, 2]] = 1
    return lab, seeds, (None if name == "voronoi" else (4.0, 4.0, 40.0))
  if name == "blocks":
    k = 32
    small = torch.randint(1, 1 << 20, (-(-n // k),) * 3, dtype=torch.int32, device="cuda", generator=g)
    lab = small.repeat_interleave(k, 0).repeat_interleave(k, 1).repeat_interleave(k, 2)[:n, :n, :n].contiguous()
    seeds[::k, ::k, ::k] = 1
    return lab, seeds, None
  # the serpentine maze
  lab = torch.ones((n, n, n), dtype=torch.uint8, device="cuda")
  for j, y in enumerate(range(7, n - 1, 8)):
    lab[:, y, :] = 0
    lab[:, y, n - 1 if j % 2 == 0 else 0] = 1
  seeds[:, 0, 0] = 0
  seeds[0, 0, 0] = 1
  return lab, seeds, None


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
  nbytes = sum(o.numel() * o.element_size() for o in out)
  del out
  return free0 - free1 - nbytes


def counts(name, n):
  """(rounds, visits, index rounds, index visits) of one verbose call with indices in a child process."""
  env = dict(os.environ, EDT_B200_VERBOSE="1")
  r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", name, "--n", str(n)], env=env,
                     capture_output=True, text=True)
  m = re.search(r"distances [\d.]+ ms \(rounds (\d+), tile visits (\d+)\)\s+indices [\d.]+ ms \(rounds (\d+), "
                r"tile visits (\d+)\)", r.stderr)
  return tuple(int(v) for v in m.groups()) if m else ("?",) * 4


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--n_host", type=int, default=96)
  ap.add_argument("--steps", type=int, default=3)
  ap.add_argument("--warmup", type=int, default=1)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--out", default=None)
  ap.add_argument("--child", default=None)
  a = ap.parse_args()
  if a.child:
    t, s, w = volume(a.child, a.n)
    edt.geodesic_distance(t, s, w, return_indices=True)
    torch.cuda.synchronize()
    return
  say("geodesic_bench: %s, power limit %s, max SM clock %s" % (smi("name"), smi("power.limit"), smi("clocks.max.sm")))
  say("n=%d, steps=%d warmup=%d rounds=%d; ms per call (median round); rounds and tile visits of the distance and "
      "index phases; MiB of device memory beyond inputs and outputs (with indices); reached: finite voxels per "
      "labelled voxel" % (a.n, a.steps, a.warmup, a.rounds))
  say("%-14s %9s %9s %7s %9s %7s %9s %7s %8s" % ("workload", "dist", "indices", "rounds", "visits", "irounds",
                                                 "ivisits", "MiB", "reached"))
  for name in WORKLOADS:
    t, s, w = volume(name, a.n)
    d = edt.geodesic_distance(t, s, w)
    frac = float(torch.isfinite(d).sum()) / max(1.0, float((t != 0).sum()))
    del d
    dist_ms = timed(lambda: edt.geodesic_distance(t, s, w), a.steps, a.warmup, a.rounds)
    idx_ms = timed(lambda: edt.geodesic_distance(t, s, w, return_indices=True), a.steps, a.warmup, a.rounds)
    mib = extra_bytes(lambda: edt.geodesic_distance(t, s, w, return_indices=True)) / 2**20
    del t, s
    torch.cuda.empty_cache()
    r, v, ir, iv = counts(name, a.n)
    say("%-14s %9.2f %9.2f %7s %9s %7s %9s %7.0f %8.4f" % (name, dist_ms, idx_ms, r, v, ir, iv, mib, frac))
  import numpy as np
  import geodesic_cases as gc
  say()
  say("scipy.sparse.csgraph.dijkstra (and the tight-edge indices) on one host thread against the GPU call with "
      "indices, n_host=%d" % a.n_host)
  say("%-14s %12s %10s %8s %s" % ("workload", "scipy s", "GPU ms", "x", "equal"))
  for name in WORKLOADS:
    t, s, w = volume(name, a.n_host)
    gpu_ms = timed(lambda: edt.geodesic_distance(t, s, w, return_indices=True), a.steps, a.warmup, a.rounds)
    dist, idx = edt.geodesic_distance(t, s, w, return_indices=True)
    dist, idx = dist.cpu().numpy(), idx.cpu().numpy()
    host, hs = t.cpu().numpy(), s.cpu().numpy()
    t0 = time.perf_counter()
    want, S = gc.restate(host, hs, w)
    sec = time.perf_counter() - t0
    same = (np.array_equal(dist.view(np.uint32), want.view(np.uint32))
            and np.array_equal(idx, gc.index_planes(S, host.shape)))
    say("%-14s %12.2f %10.3f %8.0f %s" % (name, sec, gpu_ms, sec * 1e3 / gpu_ms, "yes" if same else "NO"))
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
      fh.write("\n".join(LINES) + "\n")


if __name__ == "__main__":
  main()
