"""Chunked voxel-graph transform (edtb200_transform_voxel_graph_chunked) against the one-shot call.

  python tools/voxel_graph_chunked_bench.py [--n 512] [--big 1024] [--out FILE]

Part 1 times edtsq under a random graph on an --n^3 uint32 volume (about 10% background voxels, 5% of
graph bytes random), one-shot and chunked (budget 0, and a budget forced to about 8 phase-1 chunks),
from pinned and from pageable host buffers.  Every chunked result is compared with the one-shot result
byte for byte.  Time is the host clock around the call (it returns once the result has landed), the
median of 3 after one warm-up; bytes are what the call moves over PCIe: (L + 5) N one-shot,
(2L + 10) N up and 12 N down chunked.

Part 2 runs a --big^3 uint32 volume with a graph (1024^3 by default), if the host has the memory for
it.  It records what edtb200_transform_voxel_graph returns (EDTB200_ENOMEM on an 80 GB card) and the
time of the chunked call with budget 0 from pageable buffers.  Part 3 checks that result exactly at
10^6 sampled voxels: the labels are 1 everywhere but 10^4 seeded zeros, 10^4 seeded voxels forbid one
of their +x / +y / +z edges, there is no black border and the anisotropy is (1, 1, 1).  The doubled
grid's background cells are then the 8 cells of every zero voxel and one edge cell per forbidden edge;
a voxel's squared distance is a quarter of the squared doubled-grid distance from its even cell to the
nearest background cell (scipy.spatial.cKDTree), a multiple of 1/4 below 2^24 and so exact in float32.
"""
import argparse
import ctypes
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import edt_b200 as edt  # noqa: E402

ENOMEM = -3
LINES = []


def say(msg=""):
  print(msg, flush=True)
  LINES.append(msg)


def meminfo():
  vals = {}
  with open("/proc/meminfo") as f:
    for line in f:
      k, v = line.split(":")
      vals[k] = int(v.split()[0]) * 1024
  return vals


def card():
  try:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
  except Exception as e:                     # reported, not hidden
    return "nvidia-smi unavailable (%s)" % e


class Host:
  """A host buffer of nbytes: pinned (edtb200_host_alloc) or pageable (numpy), faulted in."""

  def __init__(self, nbytes, pinned):
    self.lib = edt._lib()
    self.ptr = None
    if pinned:
      self.ptr = self.lib.edtb200_host_alloc(ctypes.c_size_t(nbytes))
      if not self.ptr:
        raise MemoryError("edtb200_host_alloc(%d) failed" % nbytes)
      self.arr = np.frombuffer((ctypes.c_char * nbytes).from_address(self.ptr), np.uint8, count=nbytes)
    else:
      self.arr = np.empty(nbytes, np.uint8)
    self.arr.fill(0)

  def free(self):
    if self.ptr:
      self.lib.edtb200_host_free(ctypes.c_void_p(self.ptr))
      self.ptr = None


def timed(fn, reps=3):
  fn()                                       # warm-up
  ts = []
  for _ in range(reps):
    t0 = time.perf_counter()
    fn()
    ts.append(time.perf_counter() - t0)
  return float(np.median(ts))


def check(rc, what):
  if rc != 0:
    raise RuntimeError("%s failed (%d): %s" % (what, rc, edt._lib().edtb200_last_error().decode()))


def part1(n):
  lib = edt._lib()
  rng = np.random.default_rng(1)
  N, L = n ** 3, 4
  labels = (rng.integers(1, 4, N, dtype=np.uint32) * (rng.random(N, np.float32) < 0.9)).astype(np.uint32)
  graph = np.where(rng.random(N, np.float32) < 0.95, 63, rng.integers(0, 64, N)).astype(np.uint8)
  say("## part 1: %d^3 uint32 edtsq under a random graph, one-shot vs chunked, host buffers" % n)
  say("%-8s %-22s %8s %10s %9s %8s" % ("buffers", "method", "chunks", "ms", "GB moved", "GB/s"))
  ref = None
  for pinned in (True, False):
    lab, gr, out = Host(N * L, pinned), Host(N, pinned), Host(4 * N, pinned)
    lab.arr[:] = labels.view(np.uint8)
    gr.arr[:] = graph
    args = (lab.arr.ctypes.data, L, gr.arr.ctypes.data, 3, n, n, n, 1.0, 1.0, 1.0, 0, 0, out.arr.ctypes.data, 0)
    tag = "pinned" if pinned else "pageable"
    t = timed(lambda: check(lib.edtb200_transform_voxel_graph(*args, None), "edtb200_transform_voxel_graph"))
    moved = (L + 5) * N
    say("%-8s %-22s %8s %10.1f %9.2f %8.2f" % (tag, "one-shot", "-", t * 1e3, moved / 1e9, moved / t / 1e9))
    if ref is None:
      ref = out.arr.copy()
    slice1 = n * n * (L + 49)                # one phase-1 slice of the plan (tile kernels)
    for budget in (0, 2 * (-(-n // 8)) * slice1):
      chunks = (ctypes.c_int64 * 2)()
      out.arr.fill(0xA5)
      t = timed(lambda: check(lib.edtb200_transform_voxel_graph_chunked(*args, ctypes.c_size_t(budget), chunks),
                              "edtb200_transform_voxel_graph_chunked"))
      if not np.array_equal(out.arr, ref):
        raise AssertionError("%s: chunked result differs from the one-shot voxel-graph transform" % tag)
      moved = (2 * L + 10) * N + 12 * N
      method = "chunked budget 0" if budget == 0 else "chunked %.2f GiB" % (budget / 2 ** 30)
      say("%-8s %-22s %8s %10.1f %9.2f %8.2f" % (tag, method, "%d+%d" % tuple(chunks), t * 1e3, moved / 1e9,
                                                 moved / t / 1e9))
    for h in (lab, gr, out):
      h.free()
  say("every chunked result above equals the one-shot result byte for byte")


def part2_and_3(n):
  lib = edt._lib()
  N = n ** 3
  need = 13 * N + (8 << 30)                  # labels, graph, result, the call's scratch, headroom
  mem = meminfo()
  say("## part 2: %d^3 uint32 with a graph, pageable buffers (%.1f GB), host MemAvailable %.1f GB"
      % (n, 9 * N / 1e9, mem["MemAvailable"] / 1e9))
  if mem["MemAvailable"] < need:
    say("not run: needs %.1f GB of host memory" % (need / 1e9))
    return
  rng = np.random.default_rng(2)
  labels = np.ones((n, n, n), np.uint32)                              # C order: (z, y, x)
  zeros = np.unique(rng.integers(0, N, 10 ** 4))
  labels.reshape(-1)[zeros] = 0
  graph = np.full((n, n, n), 63, np.uint8)
  cut = np.unique(rng.integers(0, N, 10 ** 4))
  cut_bit = rng.choice(np.array([1, 4, 16], np.uint8), cut.size)      # the +x, +y or +z edge
  graph.reshape(-1)[cut] = 63 & ~cut_bit
  out = np.empty(N, np.float32)
  args = (labels.ctypes.data, 4, graph.ctypes.data, 3, n, n, n, 1.0, 1.0, 1.0, 0, 0, out.ctypes.data, 0)
  t0 = time.perf_counter()
  rc = lib.edtb200_transform_voxel_graph(*args, None)
  msg = lib.edtb200_last_error().decode()
  say("edtb200_transform_voxel_graph: rc %d after %.1f s (%s)" % (rc, time.perf_counter() - t0, msg if rc else "ok"))
  if rc != ENOMEM:
    say("the one-shot call did not run out of device memory: the oversized case shows nothing")
  chunks = (ctypes.c_int64 * 2)()
  t0 = time.perf_counter()
  check(lib.edtb200_transform_voxel_graph_chunked(*args, ctypes.c_size_t(0), chunks),
        "edtb200_transform_voxel_graph_chunked")
  t = time.perf_counter() - t0
  moved = 18 * N + 12 * N
  say("edtb200_transform_voxel_graph_chunked, budget 0, pageable buffers: chunks %d+%d, %.1f s, %.1f GB moved, "
      "%.2f GB/s" % (chunks[0], chunks[1], t, moved / 1e9, moved / t / 1e9))

  from scipy.spatial import cKDTree
  say("## part 3: exact check of part 2 at 10^6 sampled voxels against cKDTree (%d zero voxels, %d forbidden "
      "edges)" % (zeros.size, cut.size))
  cells = []
  zz, zy, zx = np.unravel_index(zeros, labels.shape)
  for a in (0, 1):
    for b in (0, 1):
      for c in (0, 1):
        cells.append(np.stack([2 * zx + a, 2 * zy + b, 2 * zz + c], 1))
  cz, cy, cx = np.unravel_index(cut, labels.shape)
  fg = labels.reshape(-1)[cut] != 0                                   # a zero voxel's cells are all background
  step = np.stack([cut_bit == 1, cut_bit == 4, cut_bit == 16], 1).astype(np.int64)
  cells.append((np.stack([2 * cx, 2 * cy, 2 * cz], 1) + step)[fg])
  cells = np.concatenate(cells).astype(np.int64)
  tree = cKDTree(cells)
  S = 10 ** 6
  q = rng.integers(0, N, S)
  pz, py, px = np.unravel_index(q, labels.shape)
  p2 = np.stack([2 * px, 2 * py, 2 * pz], 1).astype(np.int64)
  _, j = tree.query(p2)
  want = ((cells[j] - p2) ** 2).sum(1) / 4.0
  got = out[q].astype(np.float64)
  bad = int((got != want).sum())
  say("max squared distance %.2f; mismatches: %d of %d" % (want.max(), bad, S))
  if bad:
    raise AssertionError("the oversized chunked voxel-graph transform differs from the KD-tree")


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--big", type=int, default=1024)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if edt.device_count() == 0:
    raise SystemExit("no CUDA device: this benchmark measures the GPU path only")
  mem = meminfo()
  say("# edtb200_transform_voxel_graph_chunked vs edtb200_transform_voxel_graph")
  say("GPU (name, power limit): %s" % card())
  say("host: %d CPUs, MemTotal %.1f GB" % (os.cpu_count(), mem["MemTotal"] / 1e9))
  if args.n:
    part1(args.n)
  if args.big:
    part2_and_3(args.big)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
      f.write("\n".join(LINES) + "\n")


if __name__ == "__main__":
  main()
