"""Chunked host feature transform (edtb200_feature_transform_chunked) against the one-shot call.

  python tools/feature_chunked_bench.py [--n 512] [--big 1400] [--out FILE]

Part 1 times the feature transform of the 512^3 volumes of tools/feature_bench.py (workloads.py:
cfg2, cfg2b, cfg3, balls, voronoi), with distances, one-shot and chunked with budgets forced to about
4 and 16 phase-2 chunks, from pinned and from pageable host buffers.  Every chunked result (distances
and the three index planes) is compared with the one-shot result byte for byte.  Time is the host
clock around the call (it returns once the result has landed), the median of 3 after one warm-up;
bytes are what the call moves over PCIe: (L + 16) N one-shot, (2L + 12) N up and 28 N down chunked.

Part 2 runs a volume the one-shot call cannot hold on an 80 GB card, if the host has the memory for
it: --big^3 uint8 (1400^3 by default: 37 bytes per voxel, about 101 GB, in one shot), indices only
(about 36 GB of host memory).  It shows that edtb200_feature_transform returns EDTB200_ENOMEM and that
the chunked call with budget 0 succeeds.  Part 3 checks that result exactly at 10^6 seeded voxels: the
labels are 1 everywhere but 10^4 seeded zeros, the weights integers, no black border, so every
voxel's site must be a zero voxel whose exact squared distance (float64) is the nearest seed's
distance found by scipy.spatial.cKDTree.
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
SQRT = 1
WORKLOADS = ("cfg2", "cfg2b", "cfg3", "balls", "voronoi")
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
  import torch
  from edt_b200 import workloads
  lib = edt._lib()
  say("## part 1: %d^3 feature transform with distances, one-shot vs chunked, host buffers" % n)
  say("%-8s %-8s %-18s %8s %10s %9s %8s" % ("volume", "buffers", "method", "chunks", "ms", "GB moved", "GB/s"))
  for name in WORKLOADS:
    lab_t, an, bb = workloads.generate(name, n, "cuda")
    labels = edt._label_view(np.ascontiguousarray(lab_t.cpu().numpy()))
    del lab_t
    torch.cuda.empty_cache()
    N, L = labels.size, labels.dtype.itemsize
    (sx, sy, sz), (wx, wy, wz) = edt._x_fastest(labels.shape, an, False)
    ref = None
    for pinned in (True, False):
      lab = Host(N * L, pinned)
      out = Host(16 * N, pinned)              # distances, then the x, y, z planes
      lab.arr[:] = labels.reshape(-1).view(np.uint8)
      base = out.arr.ctypes.data
      planes = (ctypes.c_void_p * 3)(*[base + 4 * N * (k + 1) for k in range(3)])
      args = (lab.arr.ctypes.data, L, 3, sx, sy, sz, wx, wy, wz, int(bb), SQRT, base, planes, 0)
      tag = "pinned" if pinned else "pageable"
      t = timed(lambda: check(lib.edtb200_feature_transform(*args, None), "edtb200_feature_transform"))
      moved = (L + 16) * N
      say("%-8s %-8s %-18s %8s %10.1f %9.2f %8.2f" % (name, tag, "one-shot", "-", t * 1e3, moved / 1e9,
                                                      moved / t / 1e9))
      if ref is None:
        ref = out.arr.copy()
      slice2 = sx * sz * (L + 28)             # one phase-2 slice of the plan
      for per_phase in (4, 16):
        budget = 2 * (-(-sy // per_phase)) * slice2
        chunks = (ctypes.c_int64 * 2)()
        out.arr.fill(0xA5)
        t = timed(lambda: check(lib.edtb200_feature_transform_chunked(*args, ctypes.c_size_t(budget), chunks),
                                "edtb200_feature_transform_chunked"))
        if not np.array_equal(out.arr, ref):
          raise AssertionError("%s %s: chunked result differs from the one-shot feature transform" % (name, tag))
        moved = (2 * L + 12) * N + 28 * N
        say("%-8s %-8s %-18s %8s %10.1f %9.2f %8.2f" % (name, tag, "chunked %.2f GiB" % (budget / 2 ** 30),
                                                        "%d+%d" % tuple(chunks), t * 1e3, moved / 1e9,
                                                        moved / t / 1e9))
      lab.free()
      out.free()
  say("every chunked result above equals the one-shot result byte for byte (distances and index planes)")


def part2_and_3(n):
  lib = edt._lib()
  N = n ** 3
  need = 13 * N + (8 << 30)                  # labels + three index planes + headroom
  mem = meminfo()
  say("## part 2: %d^3 uint8, indices only (%.1f GB of host buffers), host MemAvailable %.1f GB"
      % (n, 13 * N / 1e9, mem["MemAvailable"] / 1e9))
  if mem["MemAvailable"] < need:
    say("not run: needs %.1f GB of host memory" % (need / 1e9))
    return
  rng = np.random.default_rng(2)
  labels = np.ones((n, n, n), np.uint8)                               # C order: (z, y, x)
  seeds = np.unique(rng.integers(0, N, 10 ** 4))
  labels.reshape(-1)[seeds] = 0
  planes = np.empty((3, N), np.int32)                                  # x, y, z (x fastest)
  w = (1.0, 2.0, 3.0)                                                  # wx, wy, wz
  ptrs = (ctypes.c_void_p * 3)(*[planes[k].ctypes.data for k in range(3)])
  args = (labels.ctypes.data, 1, 3, n, n, n, *w, 0, SQRT, None, ptrs, 0)
  t0 = time.perf_counter()
  rc = lib.edtb200_feature_transform(*args, None)
  msg = lib.edtb200_last_error().decode()
  say("edtb200_feature_transform: rc %d after %.1f s (%s)" % (rc, time.perf_counter() - t0, msg if rc else "ok"))
  if rc != ENOMEM:
    say("the one-shot call did not run out of device memory: the oversized case shows nothing")
  chunks = (ctypes.c_int64 * 2)()
  t0 = time.perf_counter()
  check(lib.edtb200_feature_transform_chunked(*args, ctypes.c_size_t(0), chunks),
        "edtb200_feature_transform_chunked")
  t = time.perf_counter() - t0
  moved = 14 * N + 24 * N                                              # no distances: 24 bytes down
  say("edtb200_feature_transform_chunked, budget 0, pageable buffers: chunks %d+%d, %.1f s, %.1f GB moved, "
      "%.2f GB/s" % (chunks[0], chunks[1], t, moved / 1e9, moved / t / 1e9))

  from scipy.spatial import cKDTree
  say("## part 3: exact check of part 2 at 10^6 seeded voxels against cKDTree (%d seeded zeros)" % seeds.size)
  sz_, sy_, sx_ = np.unravel_index(seeds, labels.shape)
  W = np.array(w)
  tree = cKDTree(np.stack([sx_, sy_, sz_], 1) * W)
  S = 10 ** 6
  q = rng.integers(0, N, S)
  pz, py, px = np.unravel_index(q, labels.shape)
  site = np.stack([planes[k][q] for k in range(3)], 1).astype(np.int64)        # x, y, z
  p = np.stack([px, py, pz], 1).astype(np.int64)
  inside = ((site >= 0) & (site < n)).all(1)
  ours = (((site - p) * W) ** 2).sum(1)
  _, j = tree.query(p * W)
  nearest = np.stack([sx_[j], sy_[j], sz_[j]], 1).astype(np.int64)
  want = (((nearest - p) * W) ** 2).sum(1)
  zero = np.zeros(S, bool)
  zero[inside] = labels[site[inside, 2], site[inside, 1], site[inside, 0]] == 0
  bad = int((~inside | ~zero | (ours != want)).sum())
  say("sites outside the volume or not a seeded zero: %d; squared distance differs from the nearest seed: %d; "
      "mismatches in total: %d of %d" % (int((~inside | ~zero).sum()), int((inside & (ours != want)).sum()), bad, S))
  if bad:
    raise AssertionError("the oversized chunked feature transform differs from the KD-tree")


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--big", type=int, default=1400)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if edt.device_count() == 0:
    raise SystemExit("no CUDA device: this benchmark measures the GPU path only")
  mem = meminfo()
  say("# edtb200_feature_transform_chunked vs edtb200_feature_transform")
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
