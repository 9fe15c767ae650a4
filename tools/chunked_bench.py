"""Chunked host transform (edtb200_transform_chunked) against the one-shot host transform.

  python tools/chunked_bench.py [--n 512] [--big 1792] [--out FILE]

Part 1 times 512^3 volumes (iid uint32, 32^3 blocks uint32, BASELINE configs[2]: all ones uint8,
(6, 6, 30), black border) with the one-shot host transform and chunked with budgets forced to about
4 and 16 chunks per phase, from pinned and from pageable host buffers.  Every chunked result is
compared with the one-shot result bit for bit.  Time is the host clock around the call (it returns
once the result has landed), the median of 3 after one warm-up; bytes are what the call moves over
PCIe: (L + 4) N for the one-shot transform, (2L + 4) N up and 8 N down chunked.

Part 2 runs one volume the one-shot transform cannot hold (--big^3 uint32, 1792^3 by default: the
long-line Z pass needs 16 bytes per voxel on the device), if the host has the memory for it: it shows
that edtb200_transform returns EDTB200_ENOMEM and that the chunked call with budget 0 succeeds, and
checks the result at 10^7 seeded voxels against a closed form.  The labels are 32^3 blocks labelled
1 + (bx & 1) + 2 (by & 1) + 4 (bz & 1), so every face neighbour of a block has another label; with a
black border and weights w, edtsq = min_a (w_a min(c_a - start_a + 1, end_a - c_a))^2 exactly, with
[start_a, end_a) the block's extent clipped to the volume.
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


def volume(kind, n):
  """(C-ordered labels (z, y, x), (wx, wy, wz), black_border)."""
  rng = np.random.default_rng(0)
  if kind == "iid":
    return rng.integers(0, 256, (n, n, n), dtype=np.uint32), (1.0, 1.0, 1.0), False
  if kind == "blocks32":
    k = -(-n // 32)
    small = rng.integers(0, 256, (k, k, k), dtype=np.uint32)
    big = np.repeat(np.repeat(np.repeat(small, 32, 0), 32, 1), 32, 2)
    return np.ascontiguousarray(big[:n, :n, :n]), (1.0, 1.0, 1.0), False
  if kind == "cfg3":
    return np.ones((n, n, n), np.uint8), (6.0, 6.0, 30.0), True
  raise ValueError(kind)


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
  say("## part 1: %d^3, one-shot vs chunked, host buffers" % n)
  say("%-9s %-8s %-18s %12s %10s %9s %8s" % ("volume", "buffers", "method", "chunks", "ms", "GB moved", "GB/s"))
  for kind in ("iid", "blocks32", "cfg3"):
    labels, w, border = volume(kind, n)
    N, L = labels.size, labels.dtype.itemsize
    dims = (n, n, n)
    ref = None
    for pinned in (True, False):
      lab = Host(N * L, pinned)
      out = Host(N * 4, pinned)
      lab.arr[:] = labels.reshape(-1).view(np.uint8)
      args = (lab.arr.ctypes.data, L, 3, *dims, *w, int(border), 0, out.arr.ctypes.data, 0)
      tag = "pinned" if pinned else "pageable"
      t = timed(lambda: check(lib.edtb200_transform(*args, None), "edtb200_transform"))
      moved = (L + 4) * N
      say("%-9s %-8s %-18s %12s %10.1f %9.2f %8.2f" % (kind, tag, "one-shot", "-", t * 1e3, moved / 1e9, moved / t / 1e9))
      if ref is None:
        ref = out.arr.copy()
      slice_bytes = n * n * (L + 4)           # both phases: n x n voxels per slice, tile kernels
      for per_phase in (4, 16):
        budget = 2 * (-(-n // per_phase)) * slice_bytes
        chunks = (ctypes.c_int64 * 2)()
        t = timed(lambda: check(lib.edtb200_transform_chunked(*args, ctypes.c_size_t(budget), chunks),
                                "edtb200_transform_chunked"))
        if not np.array_equal(out.arr, ref):
          raise AssertionError("%s %s: chunked result differs from the one-shot transform" % (kind, tag))
        moved = (2 * L + 4) * N + 8 * N
        say("%-9s %-8s %-18s %12s %10.1f %9.2f %8.2f" % (kind, tag, "chunked %.2f GiB" % (budget / 2 ** 30),
                                                          "%d+%d" % tuple(chunks), t * 1e3, moved / 1e9,
                                                          moved / t / 1e9))
      lab.free()
      out.free()
  say("every chunked result above equals the one-shot result bit for bit")


def part2(n):
  lib = edt._lib()
  N = n ** 3
  need = 8 * N + (8 << 30)                   # labels + result + headroom for this process
  mem = meminfo()
  say("## part 2: %d^3 uint32 (%.2f GB labels + %.2f GB result), host MemTotal %.1f GB, MemAvailable %.1f GB"
      % (n, 4 * N / 1e9, 4 * N / 1e9, mem["MemTotal"] / 1e9, mem["MemAvailable"] / 1e9))
  if mem["MemAvailable"] < need:
    say("not run: needs %.1f GB of host memory" % (need / 1e9))
    return
  t0 = time.perf_counter()
  labels = np.empty((n, n, n), np.uint32)
  b = (np.arange(n) // 32) & 1
  plane = (1 + b[None, :] + 2 * b[:, None]).astype(np.uint32)          # x fastest: bx, by
  for z in range(n):
    labels[z] = plane + np.uint32(4 * b[z])
  out = np.empty(N, np.float32)
  out.fill(0)
  say("labels generated in %.1f s" % (time.perf_counter() - t0))
  w = (1.0, 2.0, 3.0)
  args = (labels.ctypes.data, 4, 3, n, n, n, *w, 1, 0, out.ctypes.data, 0)
  t0 = time.perf_counter()
  rc = lib.edtb200_transform(*args, None)
  msg = lib.edtb200_last_error().decode()
  say("edtb200_transform: rc %d after %.1f s (%s)" % (rc, time.perf_counter() - t0, msg if rc else "ok"))
  if rc != ENOMEM:
    say("the one-shot transform did not run out of device memory: the oversized case shows nothing")
  chunks = (ctypes.c_int64 * 2)()
  t0 = time.perf_counter()
  check(lib.edtb200_transform_chunked(*args, ctypes.c_size_t(0), chunks), "edtb200_transform_chunked")
  t = time.perf_counter() - t0
  moved = 12 * N + 8 * N
  say("edtb200_transform_chunked, budget 0, pageable buffers: chunks %d+%d, %.1f s, %.1f GB moved, %.2f GB/s"
      % (chunks[0], chunks[1], t, moved / 1e9, moved / t / 1e9))
  rng = np.random.default_rng(1)
  S = 10 ** 7
  c = [rng.integers(0, n, S) for _ in range(3)]                         # x, y, z
  best = np.full(S, np.inf)
  for a in range(3):
    start = (c[a] // 32) * 32
    end = np.minimum(start + 32, n)
    d = np.minimum(c[a] - start + 1, end - c[a]) * w[a]
    best = np.minimum(best, d * d)
  got = out[(c[2] * n + c[1]) * n + c[0]]
  bad = int((got != best.astype(np.float32)).sum())
  say("closed-form check at %d seeded voxels: %d differ" % (S, bad))
  if bad:
    raise AssertionError("the oversized chunked result differs from the closed form")


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--big", type=int, default=1792)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if edt.device_count() == 0:
    raise SystemExit("no CUDA device: this benchmark measures the GPU path only")
  mem = meminfo()
  say("# edtb200_transform_chunked vs edtb200_transform")
  say("GPU: %s" % card())
  say("host: %d CPUs, MemTotal %.1f GB" % (os.cpu_count(), mem["MemTotal"] / 1e9))
  part1(args.n)
  if args.big:
    part2(args.big)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
      f.write("\n".join(LINES) + "\n")


if __name__ == "__main__":
  main()
