"""GPU tests: edtb200_transform_chunked equals edtb200_transform bit for bit.

Every case runs the one-shot host transform and the chunked one on the same labels and compares the
float32 results bit for bit (NaN-free: +inf compares equal).  Budgets are forced small so that the
phases run in many chunks: one slice per chunk, uneven chunks, and the budget 0 (what the device has
free).  Where the kernel of a phase's later pass is known, the reported chunk counts must equal the
plan documented in include/edt_b200.h, restated by `plan` below.
"""
import ctypes
import os
import subprocess
import threading

import numpy as np
import pytest

from cases import random_case

pytestmark = pytest.mark.gpu

SQRT, SIGNED = 1, 2
ENOMEM = -3
FLAG_SETS = [0, SQRT, SIGNED, SQRT | SIGNED]          # edtsq, edt, sdfsq, sdf


# ---- the documented plan ------------------------------------------------------------------------

def phase_chunks(extent, slice_vox, L, cap, s, budget):
  slice_bytes = slice_vox * (L + 4 + s)
  if extent <= cap and extent * slice_bytes <= budget:
    return 1
  c = min(cap, budget // (2 * slice_bytes))
  assert c > 0
  return -(-extent // c)


def plan(ndim, dims, L, budget, s1, s2):
  """(phase-1 chunks, phase-2 chunks) of the header's plan; s1 / s2: 8 where that phase's later
  pass takes the long-line kernel."""
  sx, sy, sz = dims
  if ndim == 3:
    cap2 = max(1, (2 ** 32 - 65) // (sx * sz))
    return phase_chunks(sz, sx * sy, L, sz, s1, budget), phase_chunks(sy, sx * sz, L, cap2, s2, budget)
  cap2 = max(1, (2 ** 32 - 65) // sy)
  return phase_chunks(sy, sx, L, sy, 0, budget), phase_chunks(sx, sy, L, cap2, s2, budget)


def slices(ndim, dims, L, s1=0, s2=0):
  sx, sy, sz = dims
  if ndim == 3:
    return sx * sy * (L + 4 + s1), sx * sz * (L + 4 + s2)
  return sx * (L + 4), sy * (L + 4 + s2)


def least_budget(ndim, dims, L, s1=0, s2=0):
  """min(extent, 2) slices of each phase, the larger of the two."""
  sx, sy, sz = dims
  e1, e2 = (sz, sy) if ndim == 3 else (sy, sx)
  b1, b2 = slices(ndim, dims, L, s1, s2)
  return max(min(e1, 2) * b1, min(e2, 2) * b2)


# ---- calls ------------------------------------------------------------------------------------------

class Volume:
  """A host array as the C ABI sees it: raw label bits, x-fastest dims and weights."""

  def __init__(self, edt, data, anisotropy):
    self.shape = data.shape
    self.order = "F" if data.flags.f_contiguous else "C"
    if not (data.flags.c_contiguous or data.flags.f_contiguous):
      data = np.ascontiguousarray(data)
      self.order = "C"
    self.labels = edt._label_view(data)
    self.ndim = data.ndim
    an = (anisotropy,) * data.ndim if np.ndim(anisotropy) == 0 else tuple(anisotropy)
    self.dims, self.w = edt._x_fastest(data.shape, an, self.order == "F")
    self.L = self.labels.dtype.itemsize
    self.size = data.size


def host_buffer(edt, nbytes, pinned):
  """(numpy uint8 view, keep-alive): page-locked memory from the library, or plain numpy memory."""
  if not pinned:
    return np.zeros(nbytes, np.uint8), None
  lib = edt._lib()
  ptr = lib.edtb200_host_alloc(ctypes.c_size_t(nbytes))
  assert ptr
  block = (ctypes.c_char * nbytes).from_address(ptr)
  arr = np.frombuffer(block, dtype=np.uint8, count=nbytes)
  return arr, ptr


def oneshot(edt, v, flags, border):
  out = np.empty(v.size, np.float32)
  rc = edt._lib().edtb200_transform(v.labels.ctypes.data, v.L, v.ndim, *v.dims, *v.w, int(border), flags,
                                    out.ctypes.data, 0, None)
  edt._check(rc)
  return out


def chunked(edt, v, flags, border, budget, pinned_labels=False, pinned_out=False):
  """-> (result, [phase-1 chunks, phase-2 chunks], rc)."""
  lib = edt._lib()
  lab, lab_keep = host_buffer(edt, v.labels.nbytes, pinned_labels)
  out, out_keep = host_buffer(edt, v.size * 4, pinned_out)
  try:
    lab[:] = np.ravel(v.labels, order="K").view(np.uint8)
    chunks = (ctypes.c_int64 * 2)()
    rc = lib.edtb200_transform_chunked(lab.ctypes.data, v.L, v.ndim, *v.dims, *v.w, int(border), flags,
                                       out.ctypes.data, 0, ctypes.c_size_t(budget), chunks)
    return out.view(np.float32).copy(), list(chunks), rc
  finally:
    for p in (lab_keep, out_keep):
      if p:
        lib.edtb200_host_free(ctypes.c_void_p(p))


def assert_bit_equal(got, want):
  assert got.shape == want.shape
  bad = got.view(np.uint32) != want.view(np.uint32)
  assert not bad.any(), "%d of %d voxels differ, first at %d: %r vs %r" % (
    int(bad.sum()), bad.size, int(np.argmax(bad)), got[np.argmax(bad)], want[np.argmax(bad)])


def later_kernel(edt):
  return edt.last_later_launch()["kernel"]


# ---- random cases: every dtype, both orders, odd sizes, singleton axes ---------------------------

def _random_cases():
  out = []
  for seed in range(400):
    labels, kw = random_case(seed)
    if labels.ndim >= 2 and labels.size > 1:
      out.append(seed)
    if len(out) == 36:
      break
  return out


@pytest.mark.parametrize("seed", _random_cases())
def test_random_cases_bit_equal(edt, seed):
  labels, kw = random_case(seed)
  v = Volume(edt, labels, kw["anisotropy"])
  border = kw["black_border"]
  for flags in FLAG_SETS:
    want = oneshot(edt, v, flags, border)
    # the long-line kernel may take either phase's later pass here: the least budget covers both
    tight = least_budget(v.ndim, v.dims, v.L, 8, 8)
    for budget in (tight, 3 * tight - 1, 0):
      got, chunks, rc = chunked(edt, v, flags, border, budget)
      assert rc == 0, edt._lib().edtb200_last_error()
      assert_bit_equal(got, want)
      lo = plan(v.ndim, v.dims, v.L, budget or (1 << 40), 0, 0)
      hi = plan(v.ndim, v.dims, v.L, budget or (1 << 40), 8, 8)
      assert all(l <= c <= h for l, c, h in zip(lo, chunks, hi)), (chunks, lo, hi)


def test_singleton_and_thin_axes(edt):
  rng = np.random.default_rng(5)
  for shape in [(1, 1, 1), (1, 7, 1), (5, 1, 9), (1, 1, 13), (2, 2), (1, 9), (9, 1), (3, 1, 1)]:
    labels = rng.integers(0, 3, shape).astype(np.uint16)
    for order in ("C", "F"):
      v = Volume(edt, np.asarray(labels, order=order), (1.0,) * len(shape))
      for border in (False, True):
        for flags in FLAG_SETS:
          want = oneshot(edt, v, flags, border)
          for budget in (least_budget(v.ndim, v.dims, v.L), 0):
            got, chunks, rc = chunked(edt, v, flags, border, budget)
            assert rc == 0, edt._lib().edtb200_last_error()
            assert_bit_equal(got, want)
            assert chunks == list(plan(v.ndim, v.dims, v.L, budget or (1 << 40), 0, 0)), (shape, budget, chunks)


# ---- workloads, weights ------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["cfg2", "cfg2b", "blocks8", "cfg3", "balls", "voronoi", "ones_nobb"])
def test_workloads_bit_equal(edt, name):
  from edt_b200 import workloads
  lab, an, bb = workloads.generate(name, 48, "cuda", nz=37)
  labels = lab.cpu().numpy()
  v = Volume(edt, labels, an)
  for flags in FLAG_SETS:
    for border in (bb, not bb):
      want = oneshot(edt, v, flags, border)
      if name == "ones_nobb" and not border:
        assert np.isinf(want).all()
      for budget in (least_budget(3, v.dims, v.L), 5 * slices(3, v.dims, v.L)[0] + 17, 0):
        got, chunks, rc = chunked(edt, v, flags, border, budget)
        assert rc == 0, edt._lib().edtb200_last_error()
        assert_bit_equal(got, want)
        assert chunks == list(plan(3, v.dims, v.L, budget or (1 << 40), 0, 0)), (budget, chunks)


@pytest.mark.parametrize("anisotropy", [(1.0, 2.0, 3.0), (4.0, 4.0, 40.0), (0.7, 1.3, 2.9), (2.9, 0.7, 1.3),
                                        (1e-7, 1.0, 1e8), (1e8, 1e-7, 3.0), (1e-7, 1e-7, 1e-7), (1e8, 1e8, 1e8)])
@pytest.mark.parametrize("ndim", [2, 3])
def test_weights_bit_equal(edt, anisotropy, ndim):
  rng = np.random.default_rng(11)
  shape = (21, 34, 27)[:ndim]
  labels = rng.integers(0, 4, shape).astype(np.uint32)
  labels[labels == 3] = 1                       # longer runs than iid
  v = Volume(edt, labels, anisotropy[:ndim])
  for flags in FLAG_SETS:
    for border in (False, True):
      want = oneshot(edt, v, flags, border)
      for budget in (least_budget(ndim, v.dims, v.L, 8, 8), 0):
        got, chunks, rc = chunked(edt, v, flags, border, budget)
        assert rc == 0, edt._lib().edtb200_last_error()
        assert_bit_equal(got, want)


def test_budget_formula_one_slice_and_uneven(edt):
  """Integer weights and short lines: every later pass takes the tile kernel (s = 0)."""
  rng = np.random.default_rng(3)
  for shape in [(13, 17, 19), (40, 31, 9), (20, 20, 15), (23, 29)]:
    labels = rng.integers(0, 5, shape).astype(np.uint8)
    v = Volume(edt, labels, (1.0,) * len(shape))
    s1, s2 = slices(v.ndim, v.dims, v.L)
    want = oneshot(edt, v, SQRT, True)
    budgets = [least_budget(v.ndim, v.dims, v.L),            # one slice per chunk in the larger phase
               2 * s1, 2 * s2, 2 * max(s1, s2),
               3 * 2 * max(s1, s2) + 1,                      # three slices: uneven chunks
               7 * 2 * max(s1, s2) - 1,
               10 ** 12, 0]
    for budget in budgets:
      if budget and budget < least_budget(v.ndim, v.dims, v.L):
        continue
      got, chunks, rc = chunked(edt, v, SQRT, True, budget)
      assert rc == 0, edt._lib().edtb200_last_error()
      assert_bit_equal(got, want)
      assert later_kernel(edt) == "tile"
      assert chunks == list(plan(v.ndim, v.dims, v.L, budget or (1 << 40), 0, 0)), (shape, budget, chunks)
    if s1 == s2:                                 # (20, 20, 15): one slice per chunk in both phases
      got, chunks, _ = chunked(edt, v, SQRT, True, 2 * s1)
      assert chunks == [v.dims[2], v.dims[1]]
      assert_bit_equal(got, want)


# ---- the long-line kernel in phase 2 ------------------------------------------------------------

def test_long_lines_phase2(edt):
  """sz > 4096: the Z pass takes the long-line kernel in the one-shot transform and in every chunk."""
  rng = np.random.default_rng(8)
  labels = np.asfortranarray(rng.integers(0, 2, (8, 8, 5000)).astype(np.uint32))
  labels[:, :, 1000:4500] = 1
  v = Volume(edt, labels, (1.0, 2.0, 1.0))
  assert v.dims == [8, 8, 5000]
  for flags in (0, SQRT | SIGNED):
    for border in (False, True):
      want = oneshot(edt, v, flags, border)
      assert later_kernel(edt) == "long"
      tight = least_budget(3, v.dims, v.L, 0, 8)
      for budget in (tight, 3 * tight + 5, 0):
        got, chunks, rc = chunked(edt, v, flags, border, budget)
        assert rc == 0, edt._lib().edtb200_last_error()
        assert later_kernel(edt) == "long"
        assert_bit_equal(got, want)
        assert chunks == list(plan(3, v.dims, v.L, budget or (1 << 40), 0, 8)), (budget, chunks)


def test_inexact_sums_phase2(edt):
  """Weights whose candidate sums are not exact in double: the last pass forms them in double on the
  long-line kernel, chunked as in one shot (2-D: phase 1 has no later pass, so only s2 is 8)."""
  rng = np.random.default_rng(9)
  labels = rng.integers(0, 3, (300, 257)).astype(np.uint64)
  v = Volume(edt, labels, (1e8, 1e-7))                 # wx = 1e-7, wy = 1e8
  for flags in FLAG_SETS:
    want = oneshot(edt, v, flags, False)
    info = edt.last_later_launch()
    assert info["kernel"] == "long" and info["all_double"] == 1
    tight = least_budget(2, v.dims, v.L, 0, 8)
    for budget in (tight, 4 * tight + 3, 0):
      got, chunks, rc = chunked(edt, v, flags, False, budget)
      assert rc == 0, edt._lib().edtb200_last_error()
      assert edt.last_later_launch()["all_double"] == 1
      assert_bit_equal(got, want)
      assert chunks == list(plan(2, v.dims, v.L, budget or (1 << 40), 0, 8)), (budget, chunks)


# ---- host buffers ---------------------------------------------------------------------------------

@pytest.mark.parametrize("pinned_labels,pinned_out", [(False, False), (True, False), (False, True), (True, True)])
def test_pinned_and_pageable(edt, pinned_labels, pinned_out):
  rng = np.random.default_rng(12)
  small = rng.integers(0, 9, (12, 30, 40)).astype(np.uint32)
  labels = np.repeat(np.repeat(np.repeat(small, 8, 0), 8, 1), 8, 2)[:90, :231, :317]    # 6.6 M voxels
  v = Volume(edt, labels, (1.0, 1.0, 2.0))
  want = oneshot(edt, v, SQRT | SIGNED, True)
  # chunks of a few slices (copied directly), of 30 slices (8.8 MB: staged, pitched in phase 2), one
  for budget in (least_budget(3, v.dims, v.L), 13 * slices(3, v.dims, v.L)[0], 60 * slices(3, v.dims, v.L)[0], 0):
    got, chunks, rc = chunked(edt, v, SQRT | SIGNED, True, budget, pinned_labels, pinned_out)
    assert rc == 0, edt._lib().edtb200_last_error()
    assert_bit_equal(got, want)
    assert chunks == list(plan(3, v.dims, v.L, budget or (1 << 40), 0, 0))


@pytest.mark.parametrize("pinned", [False, True])
def test_pitched_rows_longer_than_a_staging_buffer(edt, pinned):
  """(4, 1500, 17000) uint8 in three phase-2 chunks of 500 y rows: each of the 4 pitched distance
  rows is 34 MB, more than one 32 MiB staging buffer."""
  rng = np.random.default_rng(13)
  labels = np.repeat(rng.integers(0, 3, (4, 1500, 17000 // 8)).astype(np.uint8), 8, axis=2)
  v = Volume(edt, labels, (1.0, 1.0, 1.0))
  assert v.dims == [17000, 1500, 4]
  budget = 2 * 500 * 17000 * 4 * 5
  assert 500 * 17000 * 4 > 32 << 20
  want = oneshot(edt, v, 0, False)
  got, chunks, rc = chunked(edt, v, 0, False, budget, pinned, pinned)
  assert rc == 0, edt._lib().edtb200_last_error()
  assert chunks == [4, 3]
  assert_bit_equal(got, want)


# ---- errors ---------------------------------------------------------------------------------------

def test_budget_below_one_chunk_is_enomem(edt):
  rng = np.random.default_rng(14)
  for shape in [(10, 20, 30), (30, 20, 10), (17, 40)]:
    v = Volume(edt, rng.integers(0, 3, shape).astype(np.uint16), (1.0,) * len(shape))
    need = least_budget(v.ndim, v.dims, v.L)
    got, chunks, rc = chunked(edt, v, 0, False, need - 1)
    assert rc == ENOMEM
    msg = edt._lib().edtb200_last_error().decode()
    assert "needs at least %d bytes" % need in msg, msg
    got, chunks, rc = chunked(edt, v, 0, False, need)
    assert rc == 0
    assert_bit_equal(got, oneshot(edt, v, 0, False))


# ---- concurrency ----------------------------------------------------------------------------------

def test_two_threads_and_a_oneshot_call(edt):
  rng = np.random.default_rng(15)
  vols = [Volume(edt, rng.integers(0, 4, (60, 70, 80)).astype(np.uint32), (1.0, 2.0, 3.0)),
          Volume(edt, np.asfortranarray(rng.integers(0, 2, (50, 90, 40)).astype(np.uint8)), (2.0, 1.0, 1.0))]
  want = [oneshot(edt, v, SQRT | SIGNED, True) for v in vols]
  budgets = [3 * least_budget(3, v.dims, v.L) + 1 for v in vols]
  results = {}

  def work(name, fn):
    try:
      results[name] = [fn() for _ in range(4)]
    except Exception as e:                  # reported below
      results[name] = e

  jobs = [("chunked0", lambda: chunked(edt, vols[0], SQRT | SIGNED, True, budgets[0])),
          ("chunked1", lambda: chunked(edt, vols[1], SQRT | SIGNED, True, budgets[1])),
          ("oneshot0", lambda: (oneshot(edt, vols[0], SQRT | SIGNED, True), None, 0))]
  threads = [threading.Thread(target=work, args=job) for job in jobs]
  for t in threads:
    t.start()
  for t in threads:
    t.join()
  for name, idx in (("chunked0", 0), ("chunked1", 1), ("oneshot0", 0)):
    runs = results[name]
    assert not isinstance(runs, Exception), runs
    for got, _, rc in runs:
      assert rc == 0
      assert_bit_equal(got, want[idx])


# ---- fallbacks ------------------------------------------------------------------------------------

def test_python_falls_back_on_enomem(edt, monkeypatch):
  rng = np.random.default_rng(16)
  x = rng.integers(0, 5, (33, 45, 27)).astype(np.int32)
  x2 = x[0]
  want3, want2 = edt.sdf(x, anisotropy=(1.0, 2.0, 3.0)), edt.edtsq(x2, black_border=True)
  calls = []
  lib = edt._lib()

  def out_of_memory(*args):
    calls.append(args)
    return ENOMEM

  monkeypatch.setattr(lib, "edtb200_transform", out_of_memory)
  assert_bit_equal(edt.sdf(x, anisotropy=(1.0, 2.0, 3.0)).reshape(-1), want3.reshape(-1))
  assert_bit_equal(edt.edtsq(x2, black_border=True).reshape(-1), want2.reshape(-1))
  assert len(calls) == 2
  with pytest.raises(edt.EDTError) as info:                  # 1-D has no chunked path
    edt.edt(x[0, 0])
  assert info.value.code == ENOMEM


def test_python_max_device_bytes(edt):
  rng = np.random.default_rng(17)
  x = np.asfortranarray(rng.integers(0, 5, (40, 33, 21)).astype(np.uint16))
  for fn in (edt.edt, edt.edtsq, edt.sdf, edt.sdfsq, edt.edt3d, edt.edt3dsq):
    want = fn(x, black_border=True)
    got = fn(x, black_border=True, max_device_bytes=3 * least_budget(3, [40, 33, 21], 2))
    assert got.flags.f_contiguous and got.shape == x.shape
    assert_bit_equal(np.ravel(got, order="K"), np.ravel(want, order="K"))
  y = x[:, :, 0].copy()
  for fn in (edt.edt2d, edt.edt2dsq, edt.edt):
    assert_bit_equal(fn(y, max_device_bytes=0).reshape(-1), fn(y).reshape(-1))
  with pytest.raises(edt.EDTError) as info:
    edt.edtsq(x, max_device_bytes=1000)
  assert info.value.code == ENOMEM
  import torch
  with pytest.raises(ValueError, match="device-resident"):
    edt.edt(torch.ones((4, 4, 4), dtype=torch.uint8, device="cuda"), max_device_bytes=1 << 20)


CPP_PROGRAM = r"""
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "edt.hpp"

static int wrapped = 0;
extern "C" int __wrap_edtb200_transform(const void*, int, int, int64_t, int64_t, int64_t, float, float, float,
                                        int, int, float*, int, void*) {
  ++wrapped;
  return EDTB200_ENOMEM;
}

int main(int argc, char** argv) {
  const int sx = 37, sy = 29, sz = 23;
  std::vector<uint32_t> labels((size_t)sx * sy * sz);
  FILE* f = fopen(argv[1], "rb");
  if (!f || fread(labels.data(), 4, labels.size(), f) != labels.size()) return 2;
  fclose(f);
  float* dt = edt::edt<uint32_t>(labels.data(), sx, sy, sz, 1.0f, 2.0f, 3.0f, true);
  f = fopen(argv[2], "wb");
  fwrite(dt, 4, labels.size(), f);
  fclose(f);
  delete[] dt;
  printf("wrapped %d\n", wrapped);
  return 0;
}
"""


def test_cpp_shim_falls_back_on_enomem(edt, tmp_path):
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  libdir = os.path.dirname(edt.library_path())
  src = tmp_path / "shim.cpp"
  src.write_text(CPP_PROGRAM)
  exe = tmp_path / "shim"
  subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), str(src), "-o", str(exe),
                  "-L" + libdir, "-ledt_b200", "-Wl,-rpath," + libdir, "-Wl,--wrap=edtb200_transform"],
                 check=True)
  rng = np.random.default_rng(18)
  labels = rng.integers(0, 4, (23, 29, 37)).astype(np.uint32)          # C order: x = 37 fastest
  (tmp_path / "labels.bin").write_bytes(labels.tobytes())
  res = subprocess.run([str(exe), str(tmp_path / "labels.bin"), str(tmp_path / "out.bin")], capture_output=True,
                       text=True)
  assert res.returncode == 0, res.stderr
  assert "wrapped 1" in res.stdout
  got = np.frombuffer((tmp_path / "out.bin").read_bytes(), np.float32)
  want = edt.edt(labels, anisotropy=(3.0, 2.0, 1.0), black_border=True)
  assert_bit_equal(got, want.reshape(-1))
