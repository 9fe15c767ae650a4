#!/usr/bin/env python
"""Per-pass device times of the 512^3 uint32 label-noise edtsq with planted unsettled voxels, for
settled-tile skipping (DESIGN.md section 4.1):

  python tools/settled_bench.py [--reps N]        (EDTB200_LIBRARY=... to time another build)

Volumes: iid labels 1..2^20 (every voxel ends the X pass at f = 1, so nothing is unsettled), then with
x-runs of three planted (the middle voxel ends the X pass at f = 4 > w2 = 1) at densities 3e-5, 1e-3
and 1e-2 of the voxels, and at one per 32-voxel x-segment of every row, where no tile can be skipped.
Each volume is transformed twice before timing, so that the run statistic predicts label noise.  The
card's name and power limit are read in the same run."""
import argparse
import ctypes
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import edt_b200 as edt  # noqa: E402
import torch  # noqa: E402

N = 512


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                          "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    return out or "unknown"
  except Exception as e:          # no nvidia-smi: say so rather than guess
    return "unknown (%s)" % e


def volume(density, rng):
  """C order (z, y, x): iid labels with x-runs of three planted at `density` of the voxels, or
  (density = "segment") one in every 32-voxel x-segment of every row."""
  lab = rng.integers(1, 1 << 20, (N, N, N), dtype=np.uint32)
  fresh = np.arange(1 << 21, (1 << 21) + N * N * (N // 32), dtype=np.uint32)
  if density == "segment":
    x0 = np.arange(0, N, 32)[None, None, :] + rng.integers(0, 30, (N, N, N // 32))
    z, y, _ = np.indices(x0.shape)
    for d in range(3):
      lab[z, y, x0 + d] = fresh[:x0.size].reshape(x0.shape)
  elif density > 0:
    k = int(density * N ** 3)
    z, y, x0 = rng.integers(0, N, k), rng.integers(0, N, k), rng.integers(0, N - 2, k)
    for d in range(3):
      lab[z, y, x0 + d] = fresh[:k]
  return lab


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=20)
  args = ap.parse_args()
  lib = edt._lib()
  buf3 = (ctypes.c_float * 3)()
  print("card:", card())
  print("library:", os.path.relpath(edt.library_path(), ROOT))
  rng = np.random.default_rng(0)
  print("%-10s %8s %8s %8s %8s  %s" % ("density", "x ms", "y ms", "z ms", "total", "settled"))
  for density in (0, 3e-5, 1e-3, 1e-2, "segment"):
    lab = torch.from_numpy(volume(density, rng)).cuda()
    out = torch.empty(lab.shape, dtype=torch.float32, device="cuda")
    for _ in range(3):
      edt.edt_cuda(lab, out=out)
    torch.cuda.synchronize()
    lib.edtb200_profile_passes(1)
    for _ in range(args.reps):
      edt.edt_cuda(lab, out=out)
    torch.cuda.synchronize()
    lib.edtb200_profile_passes(0)
    ms = []
    for back in range(args.reps):
      if lib.edtb200_pass_ms(back, ctypes.cast(buf3, ctypes.c_void_p)) != 0:
        raise RuntimeError("edtb200_pass_ms failed")
      ms.append(list(buf3))
    x, y, z = (statistics.median(m[i] for m in ms) for i in range(3))
    settled = edt.last_later_launch().get("settled", "-")
    print("%-10s %8.3f %8.3f %8.3f %8.3f  %s" % (density, x, y, z, x + y + z, settled), flush=True)
    del lab, out
    torch.cuda.empty_cache()


if __name__ == "__main__":
  main()
