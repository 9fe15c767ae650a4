#!/usr/bin/env python
"""fill_holes and dust on one GPU: ms per call, device ms per phase, against the composition of public calls
each one replaces (outputs asserted equal), and scipy on one host thread for scale.

  python tools/holes_bench.py [--n 512] [--n_host 128] [--steps 3] [--warmup 1] [--rounds 3] [--out FILE]

Device-resident n^3 inputs, (z, y, x) C order, connectivity 1:
  fill_holes of
    balls     64 random uint8 balls (labels 1..64), each with a random spherical cavity
    voronoi   int32 Voronoi cells of 200 random sites with 2000 random spherical cavities
    porous    a bool mask: smoothed noise thresholded at 0.5 (blind pores and open pore space)
    noise     int32 label noise 0..3: about a quarter background, the worst case for the tally
  dust of
    noise     int32 label noise 0..3 at thresholds 2, 8 and 64
    voronoi   the Voronoi cells with 20000 fragments of 1..4 voxels of other labels, threshold 64
The composition each call replaces (its output must equal the native call's; a difference is reported with
whether each side repeats itself, and fails the run):
  fill_holes  comp = connected_components(labels == 0); per component torch scatter-reductions of the faces
              (amax), the sizes (bincount) and the least and largest bordering label over every neighbour
              offset (amin / amax); then a gather of the fill label.
  dust        comp = connected_components(labels); sizes = bincount(comp); a gather of sizes[comp] >= threshold.
ms per call: CUDA events around rounds of `steps` calls after warm-up, the median round.  Phase ms: one
EDT_B200_VERBOSE=1 call of each workload in a child process.  scipy: binary_fill_holes per label value
(fill_holes) and ndimage.label per label value with bincount (dust) at n_host^3 on one host thread, against
the GPU call, outputs compared.  The card's name and power limit are read in the same run.
"""
import argparse
import os
import re
import subprocess
import sys
import time

for var in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):
  os.environ.setdefault(var, "1")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import edt_b200 as edt  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

LINES = []
FILL_WORK = ("balls", "voronoi", "porous", "noise")
DUST_WORK = (("noise", 2), ("noise", 8), ("noise", 64), ("voronoi_fragments", 64))


def say(line=""):
  print(line, flush=True)
  LINES.append(line)


def smi():
  try:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except Exception as e:  # noqa: BLE001
    return "nvidia-smi unavailable (%s)" % e


def _grid(n, dev):
  z = torch.arange(n, device=dev, dtype=torch.float32)
  return z.view(n, 1, 1), z.view(1, n, 1), z.view(1, 1, n)


def _spheres(lab, centres, radii, value):
  """lab[|p - c| <= r] = value for each sphere, each written within its bounding box."""
  n = lab.shape[0]
  for (cz, cy, cx), r in zip(centres.tolist(), radii.tolist()):
    lo = [max(int(c - r), 0) for c in (cz, cy, cx)]
    hi = [min(int(c + r) + 1, n) for c in (cz, cy, cx)]
    z, y, x = (torch.arange(a, b, device=lab.device, dtype=torch.float32) for a, b in zip(lo, hi))
    m = (z.view(-1, 1, 1) - cz) ** 2 + (y.view(1, -1, 1) - cy) ** 2 + (x.view(1, 1, -1) - cx) ** 2 <= r * r
    box = lab[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]]
    box[m] = value if not callable(value) else value(box[m])


def voronoi(n, dev, g):
  sites = torch.rand((200, 3), generator=g, device=dev) * n
  lab = torch.empty((n, n, n), dtype=torch.int32, device=dev)
  z, y, x = _grid(n, dev)
  for z0 in range(0, n, 8):
    zz = z[z0:z0 + 8]
    best = torch.full((zz.shape[0], n, n), float("inf"), device=dev)
    for k in range(200):
      d = (zz - sites[k, 0]) ** 2 + (y - sites[k, 1]) ** 2 + (x - sites[k, 2]) ** 2
      take = d < best
      best = torch.where(take, d, best)
      lab[z0:z0 + 8][take] = k + 1
  return lab


def make(name, n, dev):
  g = torch.Generator(device=dev)
  g.manual_seed(7)
  if name == "balls":
    lab = torch.zeros((n, n, n), dtype=torch.uint8, device=dev)
    centres = torch.rand((64, 3), generator=g, device=dev) * n
    radii = (0.03 + 0.08 * torch.rand(64, generator=g, device=dev)) * n
    for k in range(64):
      _spheres(lab, centres[k:k + 1], radii[k:k + 1], k + 1)
    off = (torch.rand((64, 3), generator=g, device=dev) - 0.5) * radii.view(-1, 1) * 0.5
    _spheres(lab, centres + off, radii * 0.4, 0)
    return lab
  if name in ("voronoi", "voronoi_fragments"):
    lab = voronoi(n, dev, g)
    if name == "voronoi":
      _spheres(lab, torch.rand((2000, 3), generator=g, device=dev) * n,
               1 + 6 * torch.rand(2000, generator=g, device=dev), 0)
      return lab
    idx = torch.randint(0, n ** 3 - 4, (20000,), generator=g, device=dev)
    flat = lab.view(-1)
    for k in range(4):                                           # fragments of 1..4 voxels along x
      keep = torch.rand(20000, generator=g, device=dev) * 4 >= k
      flat[idx[keep] + k] = 201 + (idx[keep] % 50).to(torch.int32)
    return lab
  if name == "porous":
    small = torch.rand((1, 1, n // 8, n // 8, n // 8), generator=g, device=dev)
    smooth = torch.nn.functional.interpolate(small, size=(n, n, n), mode="trilinear", align_corners=False)[0, 0]
    return smooth > 0.5
  if name == "noise":
    return torch.randint(0, 4, (n, n, n), generator=g, device=dev, dtype=torch.int32)
  raise ValueError(name)


def _offsets(nd):
  return [d for d in np.ndindex(*(3,) * nd) if sum(abs(k - 1) for k in d) == 1]


def _shift(a, d, fill):
  out = torch.full_like(a, fill)
  n = a.shape
  src = tuple(slice(max(k - 1, 0), n[i] + min(k - 1, 0)) for i, k in enumerate(d))
  dst = tuple(slice(max(1 - k, 0), n[i] + min(1 - k, 0)) for i, k in enumerate(d))
  out[dst] = a[src]
  return out


def fill_composed(lab):
  """fill_holes at connectivity 1 from public calls: the components of the background, the face, size and
  bordering-label reductions per component, and a gather."""
  comp = edt.connected_components(lab == 0).to(torch.int64)
  m = int(comp.max()) + 1
  face = torch.zeros_like(comp, dtype=torch.bool)
  face[0], face[-1], face[:, 0], face[:, -1], face[:, :, 0], face[:, :, -1] = (True,) * 6
  is_open = torch.zeros(m, dtype=torch.int64, device=lab.device).scatter_reduce(
    0, comp[face], torch.ones_like(comp[face]), "amax")
  sizes = torch.bincount(comp.view(-1), minlength=m)
  wide = lab.to(torch.int64)
  lo = torch.full((m,), 1 << 62, dtype=torch.int64, device=lab.device)
  hi = torch.full((m,), -1, dtype=torch.int64, device=lab.device)
  for d in _offsets(3):
    nb = _shift(wide, d, 0)
    hit = (comp > 0) & (nb != 0)
    lo.scatter_reduce_(0, comp[hit], nb[hit], "amin")
    hi.scatter_reduce_(0, comp[hit], nb[hit], "amax")
  fill = (is_open == 0) & (hi >= 0) & (lo == hi) & (sizes > 0)
  fill[0] = False
  return torch.where(fill[comp], hi[comp], wide).to(lab.dtype)


def dust_composed(lab, threshold):
  comp = edt.connected_components(lab).to(torch.int64)
  sizes = torch.bincount(comp.view(-1))
  keep = (sizes[comp] >= threshold) & (comp > 0)
  return torch.where(keep, lab, torch.zeros_like(lab))


MISMATCHES = []


def check_equal(what, native, composed, again_native, again_composed):
  """Records a mismatch between the native call and its composition, with whether each side repeats itself
  (both sides run union-find whose races must not change the result)."""
  if torch.equal(native, composed):
    return
  n = int((native != composed).sum())
  a, b = again_native(), again_composed()
  MISMATCHES.append(what)
  say("MISMATCH %s: %d voxels differ; native repeats itself: %s, composition repeats itself: %s, "
      "second native == second composition: %s" % (what, n, torch.equal(native, a), torch.equal(composed, b),
                                                     torch.equal(a, b)))


def timed(fn, steps, warmup, rounds):
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  times = []
  for _ in range(rounds):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
      fn()
    b.record()
    b.synchronize()
    times.append(a.elapsed_time(b) / steps)
  return sorted(times)[len(times) // 2]


def phases(n):
  """One verbose call of each workload (run in a child with EDT_B200_VERBOSE=1)."""
  for name in FILL_WORK:
    edt.fill_holes(make(name, n, "cuda"))
    torch.cuda.synchronize()
  for name, threshold in DUST_WORK:
    edt.dust(make(name, n, "cuda"), threshold)
    torch.cuda.synchronize()


def scipy_side(n_host):
  import scipy.ndimage as ndi
  import holes_cases as hc
  say("scipy on one host thread at %d^3 (outputs equal to the GPU's):" % n_host)
  for name in FILL_WORK:
    lab = make(name, n_host, "cuda")
    host = lab.cpu().numpy()
    t = time.perf_counter()
    want = host.copy()
    for L in np.unique(host[host != 0]):
      want[ndi.binary_fill_holes(host == L) & (host == 0)] = L
    t = time.perf_counter() - t
    # scipy fills per label: equal to the GPU where no gap borders two labels
    ms = timed(lambda: edt.fill_holes(lab), 3, 1, 3)
    got = edt.fill_holes(lab).cpu().numpy()
    assert np.array_equal(got, hc.restate_fill(host)[0])
    say("  fill_holes %-8s scipy per label %9.1f ms   GPU %7.3f ms   (%.0fx)" % (name, t * 1e3, ms, t * 1e3 / ms))
  for name, threshold in DUST_WORK:
    lab = make(name, n_host, "cuda")
    host = lab.cpu().numpy()
    t = time.perf_counter()
    want = hc.restate_dust(host, threshold, how="scipy")
    t = time.perf_counter() - t
    ms = timed(lambda: edt.dust(lab, threshold), 3, 1, 3)
    got = edt.dust(lab, threshold).cpu().numpy()
    assert np.array_equal(got, want)
    say("  dust %-18s t=%-3d scipy %9.1f ms   GPU %7.3f ms   (%.0fx)" % (name, threshold, t * 1e3, ms, t * 1e3 / ms))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--n_host", type=int, default=128)
  ap.add_argument("--steps", type=int, default=3)
  ap.add_argument("--warmup", type=int, default=1)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--out")
  ap.add_argument("--phases", action="store_true", help=argparse.SUPPRESS)
  args = ap.parse_args()
  if args.phases:
    phases(args.n)
    return
  if not torch.cuda.is_available():
    sys.exit("holes_bench: no CUDA device: nothing here is measured without one")
  say("holes_bench: %d^3 device-resident, connectivity 1; GPU: %s" % (args.n, smi()))
  say("%-28s %10s %12s %8s" % ("workload", "native ms", "composed ms", "ratio"))
  for name in FILL_WORK:
    lab = make(name, args.n, "cuda")
    native = edt.fill_holes(lab)
    check_equal("fill_holes " + name, native, fill_composed(lab), lambda: edt.fill_holes(lab), lambda: fill_composed(lab))
    del native
    a = timed(lambda: edt.fill_holes(lab), args.steps, args.warmup, args.rounds)
    b = timed(lambda: fill_composed(lab), args.steps, args.warmup, args.rounds)
    say("%-28s %10.3f %12.3f %8.2f" % ("fill_holes " + name, a, b, b / a))
    del lab
    torch.cuda.empty_cache()
  for name, threshold in DUST_WORK:
    lab = make(name, args.n, "cuda")
    native = edt.dust(lab, threshold)
    check_equal("dust %s t=%d" % (name, threshold), native, dust_composed(lab, threshold),
                lambda: edt.dust(lab, threshold), lambda: dust_composed(lab, threshold))
    del native
    a = timed(lambda: edt.dust(lab, threshold), args.steps, args.warmup, args.rounds)
    b = timed(lambda: dust_composed(lab, threshold), args.steps, args.warmup, args.rounds)
    say("%-28s %10.3f %12.3f %8.2f" % ("dust %s t=%d" % (name, threshold), a, b, b / a))
    del lab
    torch.cuda.empty_cache()
  say("device ms per phase (one EDT_B200_VERBOSE=1 call each):")
  env = dict(os.environ, EDT_B200_VERBOSE="1")
  res = subprocess.run([sys.executable, os.path.abspath(__file__), "--phases", "--n", str(args.n)], env=env,
                       capture_output=True, text=True, timeout=1800)
  for line in res.stderr.splitlines():
    if re.search(r"\] (fill_holes|dust) ", line):
      say("  " + line.split("] ", 1)[1])
  if res.returncode:
    say("  phase run failed: " + res.stderr[-500:])
  scipy_side(args.n_host)
  if args.out:
    with open(args.out, "w") as f:
      f.write("\n".join(LINES) + "\n")
  if MISMATCHES:
    sys.exit("holes_bench: the native calls and their compositions differ on: " + ", ".join(MISMATCHES))


if __name__ == "__main__":
  main()
