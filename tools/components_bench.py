#!/usr/bin/env python
"""connected_components and extended_maxima on one GPU: ms per call, device ms per phase, the bytes each
phase must move and their share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), and the scipy
restatement on one host thread for scale.

  python tools/components_bench.py [--n 512] [--n_host 128] [--steps 3] [--warmup 1] [--rounds 3] [--out FILE]

Device-resident n^3 inputs, (z, y, x) C order, at connectivity 1 and 3:
  connected_components of
    noise     uint32 label noise: labels 0..9 uniformly at random (about one component per 2-3 voxels)
    blocks    uint32 32^3 blocks, one label each
    voronoi   int32 Voronoi cells of 200 random sites
    balls     64 random balls (radii 0.03 n .. 0.11 n), uint8
    ones      an all-ones uint8 volume: one component
    maze      a uint8 serpentine maze: walls of label 0 across every 8th y row, open at alternate ends
  extended_maxima of
    edt(balls) at h = 0, 1 and 2 (labels: the balls)
    random    a uniform random float32 image, h = 0 (no labels)
  split       dist = edt(balls); markers = extended_maxima(dist, 1, balls); watershed(-dist, markers, balls)
For each: ms per call (CUDA events around rounds of `steps` calls after warm-up, the median round), the
device ms of each phase from one EDT_B200_VERBOSE=1 call (all of them in one child process), and GB/s and share of
3.35 TB/s of the whole call for the bytes it must move at least (read the inputs once, write the result once:
label bytes + 4 per voxel, + 4 for an image).  The phase model (bytes per voxel, B the label width, O = 4 the
output width): union B + 4 (labels in, parents out; the border pass re-reads only face voxels), flatten
4 + 4 + O (parents in and out, flags out; plus mark: B + 4 for R and labels), numbering 4 O + 4 (cub's
in-place scan reads and writes out, the number pass reads parents and out and writes out).
Then scipy.ndimage.label per label value (connected_components) and components_cases.restate_em (extended
maxima) on one host thread at n_host^3 against the GPU call, outputs compared.  The card's name and power
limit are read in the same run.
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

PEAK = 3.35e12
LINES = []
CC_WORK = ("noise", "blocks", "voronoi", "balls", "ones", "maze")
EM_WORK = (("balls", 0.0), ("balls", 1.0), ("balls", 2.0), ("random", 0.0))


def say(line=""):
  print(line, flush=True)
  LINES.append(line)


def smi(fields):
  try:
    return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + fields, "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip() or "unknown"
  except Exception as e:
    return "unknown (%s)" % e


def labels_of(name, n):
  g = torch.Generator(device="cuda")
  g.manual_seed(0)
  ax = torch.arange(n, device="cuda", dtype=torch.float32)
  if name == "noise":
    return torch.randint(0, 10, (n, n, n), device="cuda", generator=g, dtype=torch.int32).to(torch.uint32)
  if name == "blocks":
    b = (torch.arange(n, device="cuda") // 32).to(torch.int32)
    nb = (n + 31) // 32
    return ((b.view(-1, 1, 1) * nb + b.view(1, -1, 1)) * nb + b.view(1, 1, -1) + 1).to(torch.uint32)
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
    return lab
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
    return mask.to(torch.uint8)
  if name == "ones":
    return torch.ones((n, n, n), dtype=torch.uint8, device="cuda")
  lab = torch.ones((n, n, n), dtype=torch.uint8, device="cuda")       # the maze
  for j, y in enumerate(range(7, n - 1, 8)):
    lab[:, y, :] = 0
    lab[:, y, n - 1 if j % 2 == 0 else 0] = 1
  return lab


def em_inputs(name, n):
  if name == "random":
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    return torch.rand((n, n, n), device="cuda", generator=g), None
  lab = labels_of("balls", n)
  return edt.edt(lab), lab


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


PHASES = re.compile(r"reconstruction ([\d.]+) ms \(rounds (\d+), tile visits (\d+)\)\s+union ([\d.]+) ms\s+"
                    r"flatten(?: and mark)? ([\d.]+) ms\s+numbering ([\d.]+) ms")


def configs():
  """Every (kind, name, connectivity, h) the tables time, in their order."""
  return ([("cc", name, conn, 0.0) for name in CC_WORK for conn in (1, 3)]
          + [("em", name, conn, h) for name, h in EM_WORK for conn in (1, 3)])


def phases(n):
  """{config: (reconstruction ms, rounds, union ms, flatten ms, numbering ms)} from one EDT_B200_VERBOSE=1 call
  of each config, all in one child process (the library reads the variable once)."""
  env = dict(os.environ, EDT_B200_VERBOSE="1")
  r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--n", str(n)], env=env,
                     capture_output=True, text=True)
  found = [(m.group(1), m.group(2), m.group(4), m.group(5), m.group(6)) for m in PHASES.finditer(r.stderr)]
  out = {}
  for k, c in enumerate(configs()):
    out[c] = found[k] if k < len(found) else ("?",) * 5
  return out


def share(nbytes, ms):
  return "%7.0f %5.1f%%" % (nbytes / ms / 1e6, 100.0 * nbytes / (ms * 1e-3) / PEAK)


def phase_shares(vox, label_bytes, mark, times):
  """The shares of 3.35 TB/s of the union, flatten (and mark) and numbering phases for the bytes the phase
  model of the docstring says each must move, from their device ms."""
  model = (label_bytes + 4, 12 + (label_bytes + 4 if mark else 0), 4 * 4 + 4)
  out = []
  for b, t in zip(model, times):
    try:
      out.append("%5.1f%%" % (100.0 * b * vox / (float(t) * 1e-3) / PEAK))
    except (ValueError, ZeroDivisionError):
      out.append("    ?")
  return " ".join(out)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=512)
  ap.add_argument("--n_host", type=int, default=128)
  ap.add_argument("--steps", type=int, default=3)
  ap.add_argument("--warmup", type=int, default=1)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--out", default=None)
  ap.add_argument("--child", action="store_true")
  a = ap.parse_args()
  if a.child:
    inputs = {}
    for kind, name, conn, h in configs():
      if (kind, name) not in inputs:
        inputs.clear()
        inputs[(kind, name)] = (labels_of(name, a.n), None) if kind == "cc" else em_inputs(name, a.n)
      x, lab = inputs[(kind, name)]
      torch.cuda.synchronize()
      if kind == "cc":
        edt.connected_components(x, connectivity=conn)
      else:
        edt.extended_maxima(x, h, lab, connectivity=conn)
      torch.cuda.synchronize()
    return
  say("components_bench: %s, power limit %s, max SM clock %s" % (smi("name"), smi("power.limit"),
                                                                 smi("clocks.max.sm")))
  say("n=%d, steps=%d warmup=%d rounds=%d; ms per call (median round); device ms per phase (one verbose call); "
      "GB/s and share of the 3.35 TB/s data-sheet bandwidth for the bytes the call must move at least"
      % (a.n, a.steps, a.warmup, a.rounds))
  vox = a.n ** 3
  ph = phases(a.n)
  say()
  say("connected_components")
  say("%-8s %2s %6s %9s %8s %8s %9s %14s  %s" % ("workload", "c", "comps", "ms", "union", "flatten", "numbering",
                                                 "GB/s    share", "phase shares (union flatten numbering)"))
  for name in CC_WORK:
    lab = labels_of(name, a.n)
    nbytes = vox * (lab.element_size() + 4)
    for conn in (1, 3):
      ms = timed(lambda: edt.connected_components(lab, connectivity=conn), a.steps, a.warmup, a.rounds)
      comps = int(edt.connected_components(lab, connectivity=conn).max())
      _, _, un, fl, nu = ph[("cc", name, conn, 0.0)]
      say("%-8s %2d %6d %9.2f %8s %8s %9s %s  %s" % (name, conn, comps, ms, un, fl, nu, share(nbytes, ms),
                                                    phase_shares(vox, lab.element_size(), False, (un, fl, nu))))
    del lab
    edt.release()
    torch.cuda.empty_cache()
  say()
  say("extended_maxima (rec: the reconstruction for h > 0, with its rounds)")
  say("%-8s %4s %2s %6s %9s %8s %6s %8s %8s %9s %14s  %s" % ("image", "h", "c", "maxima", "ms", "rec", "rounds",
                                                           "union", "flat+mk", "numbering", "GB/s    share",
                                                           "phase shares (union flatten+mark numbering)"))
  for name, h in EM_WORK:
    img, lab = em_inputs(name, a.n)
    nbytes = vox * (4 + 4 + (0 if lab is None else lab.element_size()))
    for conn in (1, 3):
      ms = timed(lambda: edt.extended_maxima(img, h, lab, connectivity=conn), a.steps, a.warmup, a.rounds)
      nmax = int(edt.extended_maxima(img, h, lab, connectivity=conn).max())
      rec, rounds, un, fl, nu = ph[("em", name, conn, h)]
      lb = 4 + (0 if lab is None else lab.element_size())                    # the key: R and the label
      say("%-8s %4.1f %2d %6d %9.2f %8s %6s %8s %8s %9s %s  %s" % (name, h, conn, nmax, ms, rec, rounds, un, fl, nu,
                                                                  share(nbytes, ms),
                                                                  phase_shares(vox, lb, True, (un, fl, nu))))
    del img, lab
    edt.release()
    torch.cuda.empty_cache()
  say()
  lab = labels_of("balls", a.n)

  def split():
    dist = edt.edt(lab)
    return edt.watershed(-dist, edt.extended_maxima(dist, 1.0, lab), lab)
  t_edt = timed(lambda: edt.edt(lab), a.steps, a.warmup, a.rounds)
  dist = edt.edt(lab)
  t_em = timed(lambda: edt.extended_maxima(dist, 1.0, lab), a.steps, a.warmup, a.rounds)
  markers = edt.extended_maxima(dist, 1.0, lab)
  t_ws = timed(lambda: edt.watershed(-dist, markers, lab), a.steps, a.warmup, a.rounds)
  t_all = timed(split, a.steps, a.warmup, a.rounds)
  say("split of the 64 balls: edt %.2f ms + extended_maxima(h=1) %.2f ms (%d markers) + watershed %.2f ms; "
      "the whole pipeline %.2f ms per call" % (t_edt, t_em, int(markers.max()), t_ws, t_all))
  del lab, dist, markers
  edt.release()
  torch.cuda.empty_cache()

  import numpy as np
  import scipy.ndimage
  import components_cases as cc
  say()
  say("scipy on one host thread against the GPU call at n_host=%d (connectivity 1), outputs compared" % a.n_host)
  say("%-22s %10s %10s %8s %s" % ("workload", "host s", "GPU ms", "x", "equal"))
  for name in CC_WORK:
    lab = labels_of(name, a.n_host)
    gpu_ms = timed(lambda: edt.connected_components(lab), a.steps, a.warmup, a.rounds)
    got = edt.connected_components(lab).cpu().numpy()
    h_lab = lab.cpu().numpy()
    t0 = time.perf_counter()
    want = cc.restate_cc(h_lab, 1, how="scipy")
    sec = time.perf_counter() - t0
    say("%-22s %10.2f %10.3f %8.0f %s" % ("cc " + name, sec, gpu_ms, sec * 1e3 / gpu_ms,
                                          "yes" if np.array_equal(got, want) else "NO"))
  for name, h in EM_WORK:
    img, lab = em_inputs(name, a.n_host)
    gpu_ms = timed(lambda: edt.extended_maxima(img, h, lab), a.steps, a.warmup, a.rounds)
    got = edt.extended_maxima(img, h, lab).cpu().numpy()
    h_img, h_lab = img.cpu().numpy(), None if lab is None else lab.cpu().numpy()
    t0 = time.perf_counter()
    want = cc.restate_em(h_img, h, h_lab, 1)
    sec = time.perf_counter() - t0
    say("%-22s %10.2f %10.3f %8.0f %s" % ("em %s h=%g" % (name, h), sec, gpu_ms, sec * 1e3 / gpu_ms,
                                          "yes" if np.array_equal(got, want) else "NO"))
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
      fh.write("\n".join(LINES) + "\n")


if __name__ == "__main__":
  main()
