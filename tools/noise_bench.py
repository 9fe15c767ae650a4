#!/usr/bin/env python
"""Device times of the 512^3 label-noise edtsq (iid labels 0..255, anisotropy (1, 1, 1), no black
border: the bench.py workload) for labels of 4 and 8 bytes, whole transform and per pass (GPU only):

  python tools/noise_bench.py [--size 512] [--steps 20] [--reps 3] [--anisotropy 1,0.7,1] [--image 262144,512]
                              (EDTB200_LIBRARY=... for another build)

--image SY,SX times an SY x SX image of the same label noise instead (the Z pass time reads 0).

--anisotropy (array order) picks other weights: with a non-integer one the later passes read their
run-start planes without skipping settled tiles.

Each label width is transformed twice before timing, so that the run statistic predicts label noise
and the X pass writes the run-start planes.  A rep times `steps` transforms between two CUDA events,
then the same steps again with the library's per-pass events (which keep a pass from starting under
the previous one's tail, so they are not part of the whole-transform time).  The card's name, power
limit and clocks are read in the same run.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import edt_b200 as edt  # noqa: E402


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                          "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    return out or "unknown"
  except Exception as e:          # no nvidia-smi: say so rather than guess
    return "unknown (%s)" % e


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--size", type=int, default=512)
  ap.add_argument("--steps", type=int, default=20)
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--anisotropy", type=lambda v: tuple(float(x) for x in v.split(",")), default=None)
  ap.add_argument("--image", type=lambda v: tuple(int(x) for x in v.split(",")), default=None,
                  help="SY,SX: a 2-D image instead of the 3-D volume")
  args = ap.parse_args()
  shape = args.image or (args.size,) * 3
  w = args.anisotropy or (1.0,) * len(shape)
  dev = torch.device("cuda", 0)
  lib = edt._lib()
  g = torch.Generator(device=dev)
  g.manual_seed(0)
  base = torch.randint(0, 256, shape, dtype=torch.int32, device=dev, generator=g)
  print(json.dumps({"card": card(), "library": os.path.basename(edt.library_path())}), flush=True)
  for dtype in (torch.int32, torch.int64):
    lab = base.to(dtype)
    out = torch.empty(lab.shape, dtype=torch.float32, device=dev)
    for _ in range(2):
      edt.edt_cuda(lab, w, False, out=out)
    torch.cuda.synchronize()
    totals, passes = [], []
    for _ in range(args.reps):
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(args.steps):
        edt.edt_cuda(lab, w, False, out=out)
      e1.record()
      torch.cuda.synchronize()
      totals.append(e0.elapsed_time(e1) / args.steps)
      lib.edtb200_profile_passes(1)
      for _ in range(args.steps):
        edt.edt_cuda(lab, w, False, out=out)
      torch.cuda.synchronize()
      lib.edtb200_profile_passes(0)
      buf = (ctypes.c_float * 3)()
      smp = []
      for back in range(args.steps):
        if lib.edtb200_pass_ms(back, ctypes.cast(buf, ctypes.c_void_p)) != 0:
          raise RuntimeError("edtb200_pass_ms failed")
        smp.append([float(v) for v in buf])
      passes.append([statistics.mean(s[i] for s in smp) for i in range(3)])
    print(json.dumps({"label_bytes": lab.element_size(), "shape": list(shape), "anisotropy": w, "steps": args.steps,
                      "ms": [round(t, 4) for t in totals], "ms_median": round(statistics.median(totals), 4),
                      "pass_ms_xyz": [[round(v, 4) for v in p] for p in passes], "clocks": card()}), flush=True)
    del lab, out
    torch.cuda.empty_cache()


if __name__ == "__main__":
  main()
