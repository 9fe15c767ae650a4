#!/usr/bin/env python
"""medial_axis on one GPU against the composition of public calls it replaces.

  python tools/medial_axis_bench.py [--n 512] [--n2 8192] [--steps 5] [--warmup 2] [--rounds 3] [--out FILE]

Device-resident inputs: n^3 8-bit balls and 32-bit Voronoi cells (200 seeds) (workloads.py), 32-bit labels in
32^3 blocks, an 8-bit single mask (one ball), and one n2^2 2-D 8-bit mask (one disc).  Two arms, alternating
round by round in this one command (CUDA events around each round of `steps` calls, after warm-up; the
median round is printed):
  native    edt.medial_axis(labels)
  composed  what a user writes without it: d2 = edtsq(labels); _, idx = parabolic_dilate(d2,
            return_indices=True); mask[tuple(i[labels != 0] for i in idx)] = True
For each: ms per call; the device memory taken beyond the input and the output (the drop in free device
memory over one call with everything released first: the library keeps its scratch pool's high-water mark,
EDTB200_POOL_KEEP_MB, and torch keeps what its caching allocator took); the medial voxels as a fraction of
the labelled voxels; and whether the two masks are byte-equal.  The card's name, power limit and maximum SM
clock are read in the same run.
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


def say(line=""):
  print(line, flush=True)
  LINES.append(line)


def smi(fields):
  try:
    return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + fields, "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or "unknown"
  except Exception as e:
    return "unknown (%s)" % e


def volumes(n, n2):
  yield "balls8", workloads.generate("balls", n, "cuda")[0]
  yield "voronoi32", workloads.generate("voronoi", n, "cuda")[0]
  g = torch.Generator(device="cuda")
  g.manual_seed(5)
  k = 32
  small = torch.randint(0, 1 << 20, (-(-n // k),) * 3, dtype=torch.int32, device="cuda", generator=g)
  blocks = small.repeat_interleave(k, 0).repeat_interleave(k, 1).repeat_interleave(k, 2)[:n, :n, :n].contiguous()
  del small
  yield "blocks32", blocks
  del blocks
  c = torch.arange(n, device="cuda", dtype=torch.float32) - (n - 1) / 2
  d2 = c.view(-1, 1, 1) ** 2 + c.view(1, -1, 1) ** 2 + c.view(1, 1, -1) ** 2
  mask = (d2 <= (0.4 * n) ** 2).to(torch.uint8)
  del d2
  yield "mask8", mask
  del mask
  c = torch.arange(n2, device="cuda", dtype=torch.float32) - (n2 - 1) / 2
  yield "disc8_2d", ((c.view(-1, 1) ** 2 + c.view(1, -1) ** 2) <= (0.4 * n2) ** 2).to(torch.uint8)


def native(t):
  return edt.medial_axis(t)


def composed(t):
  d2 = edt.edtsq(t)
  _, idx = edt.parabolic_dilate(d2, return_indices=True)
  mask = torch.zeros(t.shape, dtype=torch.bool, device=t.device)
  fg = t != 0
  mask[tuple(i[fg] for i in idx)] = True
  return mask


def timed_pair(fa, fb, steps, warmup, rounds):
  """Median per-call ms of fa and fb, alternating round by round."""
  for _ in range(warmup):
    fa(); fb()
  torch.cuda.synchronize()
  ta, tb = [], []
  for _ in range(rounds):
    for f, acc in ((fa, ta), (fb, tb)):
      s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      s.record()
      for _ in range(steps):
        f()
      e.record()
      e.synchronize()
      acc.append(s.elapsed_time(e) / steps)
  return sorted(ta)[len(ta) // 2], sorted(tb)[len(tb) // 2]


def extra_bytes(f):
  """Device memory one call takes beyond its input and output (its output kept alive)."""
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


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--n2", type=int, default=8192)
  ap.add_argument("--steps", type=int, default=5)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  say("medial_axis_bench: %s, power limit %s, max SM clock %s" % (smi("name"), smi("power.limit"),
                                                                  smi("clocks.max.sm")))
  say("n=%d (3-D), n2=%d (2-D), steps=%d warmup=%d rounds=%d; ms per call (median round); MiB of device memory "
      "beyond input and output; medial voxels per labelled voxel" % (a.n, a.n2, a.steps, a.warmup, a.rounds))
  say("%-9s %10s %10s %6s %9s %9s %9s %s" % ("workload", "composed", "native", "x", "MiB comp", "MiB nat",
                                             "medial", "equal"))
  for name, t in volumes(a.n, a.n2):
    got, exp = native(t), composed(t)
    ok = got.dtype == exp.dtype and torch.equal(got, exp)
    frac = float(got.sum()) / max(1.0, float((t != 0).sum()))
    del got, exp
    t_comp, t_nat = timed_pair(lambda: composed(t), lambda: native(t), a.steps, a.warmup, a.rounds)
    m_comp = extra_bytes(lambda: composed(t))
    m_nat = extra_bytes(lambda: native(t))
    say("%-9s %10.3f %10.3f %6.2f %9.0f %9.0f %9.5f %s" % (name, t_comp, t_nat, t_comp / t_nat, m_comp / 2**20,
                                                          m_nat / 2**20, frac, "yes" if ok else "NO"))
    del t
    torch.cuda.empty_cache()
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
      fh.write("\n".join(LINES) + "\n")


if __name__ == "__main__":
  main()
