#!/usr/bin/env python
"""watershed on one GPU: ms per phase, the rounds and tile visits each phase took, device memory, the
geodesic split users reach for today on the same volumes, and the CPU restatement for scale.

  python tools/watershed_bench.py [--n 512] [--n_host 96] [--steps 3] [--warmup 1] [--rounds 3] [--out FILE]

Device-resident n^3 inputs, (z, y, x) C order:
  balls     64 random balls (radii 0.03 n .. 0.11 n) as an 8-bit mask, image -edt(mask), a marker (int32) at
            each ball's centre
  voronoi   32-bit Voronoi cells of 200 sites as labels, image -edt(cells), one marker per cell at its site
  noise     a ball mask (radius 0.45 n) as labels, a uniform random float32 image, 1000 random markers
  maze      an 8-bit serpentine maze: walls of label 0 across every 8th y row, open at alternate ends, extruded
            along z; a uniform random image; markers at two far corners
For each (CUDA events around each round of `steps` calls, after warm-up; the median round):
  ws        edt.watershed(image, markers, labels) in ms per call
  levels / labels / store   the device ms of the level phase, the label phase and the store, and the rounds
            and tile visits of both phases, from one EDT_B200_VERBOSE=1 call in a child process (tile visits:
            the tiles relaxed, summed over the rounds)
  MiB       device memory taken beyond the inputs and the outputs (the drop in free device memory over one
            call with everything released first)
  geodesic  edt.geodesic_distance(labels, markers != 0, return_indices=True), the geodesic split
Then the restatement of tests/watershed_cases.py (heapq minimax Dijkstra and BFS) on one host thread at
n_host^3 against the GPU call at that size, with W and the level compared bit for bit.  The card's name,
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
WORKLOADS = ("balls", "voronoi", "noise", "maze")


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
  """(image, markers, labels) on the device, (z, y, x) C order."""
  g = torch.Generator(device="cuda")
  g.manual_seed(0)
  markers = torch.zeros((n, n, n), dtype=torch.int32, device="cuda")
  ax = torch.arange(n, device="cuda", dtype=torch.float32)
  if name == "balls":
    mask = torch.zeros((n, n, n), dtype=torch.bool, device="cuda")
    centres = (torch.rand((64, 3), device="cuda", generator=g) * 0.8 + 0.1) * n
    radii = (torch.rand(64, device="cuda", generator=g) * 0.08 + 0.03) * n
    for k in range(64):
      c, r = centres[k].tolist(), float(radii[k])
      lo = [max(0, int(ci - r)) for ci in c]
      hi = [min(n, int(ci + r) + 2) for ci in c]
      z, y, x = (ax[lo[i]:hi[i]] - c[i] for i in range(3))
      mask[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] |= (z.view(-1, 1, 1) ** 2 + y.view(1, -1, 1) ** 2
                                                      + x.view(1, 1, -1) ** 2) <= r * r
    at = centres.long().clamp(0, n - 1)
    markers[at[:, 0], at[:, 1], at[:, 2]] = torch.arange(1, 65, dtype=torch.int32, device="cuda")
    mask = mask.to(torch.uint8)
    return -edt.edt(mask), markers, mask
  if name == "voronoi":
    z, y, x = ax.view(n, 1, 1), ax.view(1, n, 1), ax.view(1, 1, n)
    c = torch.rand((200, 3), device="cuda", generator=g) * n
    best = torch.full((n, n, n), float("inf"), device="cuda")
    lab = torch.zeros((n, n, n), dtype=torch.int32, device="cuda")
    for k in range(200):
      d = (z - c[k, 0]) ** 2 + (y - c[k, 1]) ** 2 + (x - c[k, 2]) ** 2
      m = d < best
      best = torch.where(m, d, best)
      lab = torch.where(m, torch.full_like(lab, k + 1), lab)
    del best
    at = c.long().clamp(0, n - 1)
    markers[at[:, 0], at[:, 1], at[:, 2]] = torch.arange(1, 201, dtype=torch.int32, device="cuda")
    return -edt.edt(lab), markers, lab
  image = torch.rand((n, n, n), device="cuda", generator=g)
  if name == "noise":
    c = ax - (n - 1) / 2
    lab = ((c.view(-1, 1, 1) ** 2 + c.view(1, -1, 1) ** 2 + c.view(1, 1, -1) ** 2) <= (0.45 * n) ** 2).to(torch.uint8)
    at = ((torch.rand((1000, 3), device="cuda", generator=g) - 0.5) * 0.5 * n + n / 2).long().clamp(0, n - 1)
    markers[at[:, 0], at[:, 1], at[:, 2]] = torch.arange(1, 1001, dtype=torch.int32, device="cuda")
    return image, markers, lab
  # the serpentine maze
  lab = torch.ones((n, n, n), dtype=torch.uint8, device="cuda")
  for j, y in enumerate(range(7, n - 1, 8)):
    lab[:, y, :] = 0
    lab[:, y, n - 1 if j % 2 == 0 else 0] = 1
  markers[0, 0, 0] = 1
  markers[n - 1, n - 1, n - 1] = 2
  return image, markers, lab


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
  """(levels ms, rounds, visits, labels ms, rounds, visits, store ms) of one verbose call in a child process."""
  env = dict(os.environ, EDT_B200_VERBOSE="1")
  r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", name, "--n", str(n)], env=env,
                     capture_output=True, text=True)
  m = re.search(r"levels ([\d.]+) ms \(rounds (\d+), tile visits (\d+)\)\s+labels ([\d.]+) ms \(rounds (\d+), "
                r"tile visits (\d+)\)\s+store ([\d.]+) ms", r.stderr)
  return tuple(m.groups()) if m else ("?",) * 7


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
    img, mk, lab = volume(a.child, a.n)
    torch.cuda.synchronize()
    edt.watershed(img, mk, lab)
    torch.cuda.synchronize()
    return
  say("watershed_bench: %s, power limit %s, max SM clock %s" % (smi("name"), smi("power.limit"),
                                                                smi("clocks.max.sm")))
  say("n=%d, steps=%d warmup=%d rounds=%d; ms per call (median round); device ms and rounds / tile visits of the "
      "level and label phases (one verbose call); MiB of device memory beyond inputs and outputs; geodesic: "
      "geodesic_distance(labels, markers != 0, return_indices=True) in ms" % (a.n, a.steps, a.warmup, a.rounds))
  say("%-8s %8s %8s %6s %8s %8s %6s %8s %7s %6s %9s" % ("workload", "ws", "levels", "rounds", "visits", "labels",
                                                      "rounds", "visits", "store", "MiB", "geodesic"))
  for name in WORKLOADS:
    img, mk, lab = volume(name, a.n)
    ws_ms = timed(lambda: edt.watershed(img, mk, lab), a.steps, a.warmup, a.rounds)
    mib = extra_bytes(lambda: edt.watershed(img, mk, lab)) / 2**20
    seeds = mk != 0
    geo_ms = timed(lambda: edt.geodesic_distance(lab, seeds, return_indices=True), 1, 1, a.rounds)
    del img, mk, lab, seeds
    edt.release()
    torch.cuda.empty_cache()
    lm, lr, lv, wm, wr, wv, sm = counts(name, a.n)
    say("%-8s %8.2f %8s %6s %8s %8s %6s %8s %7s %6.0f %9.2f" % (name, ws_ms, lm, lr, lv, wm, wr, wv, sm, mib, geo_ms))
  import numpy as np
  import watershed_cases as wc
  say()
  say("the restatement (heapq minimax Dijkstra, then BFS per marker) on one host thread against the GPU call with "
      "the level, n_host=%d" % a.n_host)
  say("%-8s %10s %10s %8s %s" % ("workload", "host s", "GPU ms", "x", "equal"))
  for name in WORKLOADS:
    img, mk, lab = volume(name, a.n_host)
    gpu_ms = timed(lambda: edt.watershed(img, mk, lab, return_level=True), a.steps, a.warmup, a.rounds)
    W, L = edt.watershed(img, mk, lab, return_level=True)
    W, L = W.cpu().numpy(), L.cpu().numpy()
    hi, hm, hl = img.cpu().numpy(), mk.cpu().numpy(), lab.cpu().numpy()
    t0 = time.perf_counter()
    want_w, want_l = wc.restate(hi, hm, hl)
    sec = time.perf_counter() - t0
    same = np.array_equal(W, want_w) and np.array_equal(L.view(np.uint32), want_l.view(np.uint32))
    say("%-8s %10.2f %10.3f %8.0f %s" % (name, sec, gpu_ms, sec * 1e3 / gpu_ms, "yes" if same else "NO"))
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
      fh.write("\n".join(LINES) + "\n")


if __name__ == "__main__":
  main()
