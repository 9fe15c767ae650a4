#!/usr/bin/env python
"""Device-resident timing of the transform over a matrix of synthetic workloads (GPU only).

  python tools/perf_matrix.py [--size 512] [--only cfg2,cfg2b] [--steps 5]

Prints one JSON line per workload: ms per transform, Mvoxels/s, algorithmic GB/s.
Labels are generated on the GPU with torch (seeded); C-contiguous (z, y, x) tensors, i.e.
x fastest, which is the layout the kernels work in.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import edt_b200  # noqa: E402


from edt_b200 import workloads  # noqa: E402


def gen(name, n, dev):
  return workloads.generate(name, n, dev)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--size", type=int, default=512)
  ap.add_argument("--only", default="cfg2,cfg2b,blocks8,cfg3,balls,voronoi,ones_nobb")
  ap.add_argument("--steps", type=int, default=5)
  ap.add_argument("--sqrt", action="store_true")
  ap.add_argument("--aniso", default=None, help="w_z,w_y,w_x overriding the workload's anisotropy (e.g. a "
                  "non-integer one, which takes the double-precision hull tests)")
  args = ap.parse_args()
  dev = torch.device("cuda", 0)
  for name in args.only.split(","):
    lab, an, bb = gen(name, args.size, dev)
    if args.aniso:
      an = tuple(float(v) for v in args.aniso.split(","))
    out = torch.empty(lab.shape, dtype=torch.float32, device=dev)
    for _ in range(2):
      edt_b200.edt_cuda(lab, an, bb, sqrt=args.sqrt, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
      edt_b200.edt_cuda(lab, an, bb, sqrt=args.sqrt, out=out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    nvox = lab.numel()
    L = lab.element_size()
    print(json.dumps({"workload": name, "size": args.size, "label_bytes": L, "ms": round(ms, 4),
                      "Mvox_s": round(nvox / ms / 1e3, 1),
                      "alg_GBps": round((3 * L + 20) * nvox / ms / 1e6, 1),
                      "finite_max": float(out[torch.isfinite(out)].max().item()) if torch.isfinite(out).any() else None}),
          flush=True)
    del lab, out
    torch.cuda.empty_cache()


if __name__ == "__main__":
  main()
