"""GPU tests: edtb200_transform_voxel_graph_chunked equals edtb200_transform_voxel_graph bit for bit.

Every case runs the one-shot graph transform and the chunked one on the same labels and graph and
compares the float32 results as uint32 (+inf compares equal).  Budgets are forced small so that the
phases run in many chunks: one slice per chunk, uneven chunks, and the budget 0 (what the device has
free).  Where the kernel of a phase's later pass is known, the reported chunk counts must equal the
plan documented in include/edt_b200.h, restated by `plan` below.  A few cases also go against the
oracle, so the check is not only one of self-consistency.
"""
import ctypes
import os
import subprocess
import threading

import numpy as np
import pytest

from cases import random_graph_case

pytestmark = pytest.mark.gpu

SQRT, LABELS_FLOAT = 1, 16
ECUDA, ENOMEM = -2, -3
BIG = 1 << 50


# ---- the documented plan ------------------------------------------------------------------------

def phase_chunks(extent, slice_bytes, cap, budget):
  if extent <= cap and extent * slice_bytes <= budget:
    return 1
  c = min(cap, budget // (2 * slice_bytes))
  assert c > 0
  return -(-extent // c)


def slices(ndim, dims, L, long1=False, long2=False):
  """Device bytes of one phase-1 slice and one phase-2 slice; long1 / long2: that phase's later pass
  takes the long-line kernel (its two scratch volumes of doubled cells)."""
  sx, sy, sz = dims
  s2 = L + 21 + (16 if long2 else 0)
  if ndim == 3:
    return sx * sy * (L + 49 + (64 if long1 else 0)), sx * sz * s2
  return sx * (L + 29), sy * s2


def plan(ndim, dims, L, budget, long1=False, long2=False):
  """(phase-1 chunks, phase-2 chunks) of the header's plan."""
  sx, sy, sz = dims
  s1, s2 = slices(ndim, dims, L, long1, long2)
  if ndim == 3:
    cap2 = max(1, (2 ** 32 - 65) // (2 * sx * sz))
    return phase_chunks(sz, s1, sz, budget), phase_chunks(sy, s2, cap2, budget)
  cap2 = max(1, (2 ** 32 - 65) // (2 * sy))
  return phase_chunks(sy, s1, sy, budget), phase_chunks(sx, s2, cap2, budget)


def least_budget(ndim, dims, L, long1=False, long2=False):
  """min(extent, 2) slices of each phase, the larger of the two."""
  sx, sy, sz = dims
  e1, e2 = (sz, sy) if ndim == 3 else (sy, sx)
  s1, s2 = slices(ndim, dims, L, long1, long2)
  return max(min(e1, 2) * s1, min(e2, 2) * s2)


# ---- calls ------------------------------------------------------------------------------------------

class Volume:
  """Labels and graph as the C ABI sees them: raw label bits (LABELS_FLOAT for floats), the graph
  bytes in the labels' memory order, x-fastest dims and weights."""

  def __init__(self, edt, data, graph, anisotropy):
    self.shape = data.shape
    self.order = "F" if data.flags.f_contiguous else "C"
    if not (data.flags.c_contiguous or data.flags.f_contiguous):
      data = np.ascontiguousarray(data)
      self.order = "C"
    self.graph = edt._graph_bytes(graph, self.order)
    self.flags = 0
    if data.dtype == np.bool_:
      self.labels = data.view(np.uint8)
    elif data.dtype.kind == "f":
      self.labels, self.flags = data, LABELS_FLOAT
    else:
      self.labels = data.view(np.dtype("u%d" % data.dtype.itemsize))
    self.ndim = data.ndim
    an = (anisotropy,) * data.ndim if np.ndim(anisotropy) == 0 else tuple(anisotropy)
    self.dims, self.w = edt._x_fastest(data.shape, an, self.order == "F")
    self.L = self.labels.dtype.itemsize
    self.size = data.size

  def reshape(self, flat):
    return flat.reshape(self.shape, order=self.order)


def host_buffer(edt, nbytes, pinned):
  """(numpy uint8 view, keep-alive): page-locked memory from the library, or plain numpy memory."""
  if not pinned:
    return np.zeros(nbytes, np.uint8), None
  ptr = edt._lib().edtb200_host_alloc(ctypes.c_size_t(nbytes))
  assert ptr
  block = (ctypes.c_char * nbytes).from_address(ptr)
  return np.frombuffer(block, dtype=np.uint8, count=nbytes), ptr


def oneshot(edt, v, flags, border):
  out = np.empty(v.size, np.float32)
  rc = edt._lib().edtb200_transform_voxel_graph(v.labels.ctypes.data, v.L, v.graph.ctypes.data, v.ndim, *v.dims,
                                                *v.w, int(border), flags | v.flags, out.ctypes.data, 0, None)
  edt._check(rc)
  return out


def chunked(edt, v, flags, border, budget, pinned=False):
  """-> (result, [phase-1 chunks, phase-2 chunks], rc)."""
  lib = edt._lib()
  lab, lab_keep = host_buffer(edt, v.labels.nbytes, pinned)
  gr, gr_keep = host_buffer(edt, v.graph.nbytes, pinned)
  out, out_keep = host_buffer(edt, v.size * 4, pinned)
  try:
    lab[:] = np.ravel(v.labels, order="K").view(np.uint8)
    gr[:] = np.ravel(v.graph, order="K")
    chunks = (ctypes.c_int64 * 2)()
    rc = lib.edtb200_transform_voxel_graph_chunked(lab.ctypes.data, v.L, gr.ctypes.data, v.ndim, *v.dims, *v.w,
                                                   int(border), flags | v.flags, out.ctypes.data, 0,
                                                   ctypes.c_size_t(budget), chunks)
    return out.view(np.float32).copy(), list(chunks), rc
  finally:
    for p in (lab_keep, gr_keep, out_keep):
      if p:
        lib.edtb200_host_free(ctypes.c_void_p(p))


def assert_bit_equal(got, want, what=""):
  assert got.shape == want.shape
  bad = got.view(np.uint32) != want.view(np.uint32)
  assert not bad.any(), "%s: %d of %d voxels differ, first at %d: %r vs %r" % (
    what, int(bad.sum()), bad.size, int(np.argmax(bad)), got[np.argmax(bad)], want[np.argmax(bad)])


def later_kernel(edt):
  return edt.last_later_launch()["kernel"]


def run_ok(edt, v, flags, border, budget, pinned=False):
  got, chunks, rc = chunked(edt, v, flags, border, budget, pinned)
  assert rc == 0, edt._lib().edtb200_last_error()
  return got, chunks


# ---- random cases: every dtype, both orders, border and sqrt, odd sizes ------------------------------

@pytest.mark.parametrize("seed", range(44))
def test_random_graph_cases_bit_equal(edt, seed):
  labels, graph, kw = random_graph_case(seed)
  v = Volume(edt, labels, graph, kw["anisotropy"])
  border = kw["black_border"]
  for flags in (0, SQRT):
    want = oneshot(edt, v, flags, border)
    # inexact weights may send either phase's later pass to the long-line kernel: the least budget
    # with both scratch volumes covers every plan
    tight = least_budget(v.ndim, v.dims, v.L, True, True)
    for budget in (tight, 3 * tight - 1, 0):
      got, chunks = run_ok(edt, v, flags, border, budget)
      assert_bit_equal(got, want, (seed, flags, budget))
      lo = plan(v.ndim, v.dims, v.L, budget or BIG)
      hi = plan(v.ndim, v.dims, v.L, budget or BIG, True, True)
      assert all(l <= c <= h for l, c, h in zip(lo, chunks, hi)), (chunks, lo, hi)


def test_singleton_and_odd_extents(edt):
  rng = np.random.default_rng(21)
  for shape in [(1, 1, 1), (1, 7, 1), (5, 1, 9), (1, 1, 13), (3, 1, 1), (7, 5, 3), (2, 2), (1, 9), (9, 1), (1, 1),
                (13, 11)]:
    labels = (rng.random(shape) < 0.8).astype(np.uint16) * 3
    graph = np.where(rng.random(shape) < 0.6, 63, rng.integers(0, 64, shape)).astype(np.uint8)
    for order in ("C", "F"):
      v = Volume(edt, np.asarray(labels, order=order), np.asarray(graph, order=order), (1.0,) * len(shape))
      for border in (False, True):
        for flags in (0, SQRT):
          want = oneshot(edt, v, flags, border)
          for budget in (least_budget(v.ndim, v.dims, v.L), 0):
            got, chunks = run_ok(edt, v, flags, border, budget)
            assert_bit_equal(got, want, (shape, order, border, flags, budget))
            assert chunks == list(plan(v.ndim, v.dims, v.L, budget or BIG)), (shape, budget, chunks)


# ---- budgets and the plan --------------------------------------------------------------------------

def test_budget_formula_one_slice_and_uneven(edt):
  """Unit weights and short lines: every later pass takes the tile kernel."""
  rng = np.random.default_rng(22)
  for shape, dtype in [((13, 17, 19), np.uint8), ((40, 31, 9), np.uint32), ((20, 20, 15), np.uint64),
                       ((23, 29), np.uint16), ((57, 8), np.uint8)]:
    labels = (rng.random(shape) < 0.9).astype(dtype)
    graph = np.where(rng.random(shape) < 0.7, 63, rng.integers(0, 64, shape)).astype(np.uint8)
    v = Volume(edt, labels, graph, (1.0,) * len(shape))
    s1, s2 = slices(v.ndim, v.dims, v.L)
    least = least_budget(v.ndim, v.dims, v.L)
    want = oneshot(edt, v, SQRT, True)
    budgets = [least,                                        # one slice per chunk in the larger phase
               2 * s1, 2 * s2, 2 * max(s1, s2),
               3 * 2 * max(s1, s2) + 1,                      # three slices: uneven chunks
               7 * 2 * max(s1, s2) - 1,
               10 ** 12, 0]
    for budget in budgets:
      if budget and budget < least:
        continue
      got, chunks = run_ok(edt, v, SQRT, True, budget)
      assert_bit_equal(got, want, (shape, budget))
      assert later_kernel(edt) == "tile"
      assert chunks == list(plan(v.ndim, v.dims, v.L, budget or BIG)), (shape, budget, chunks)
    got, chunks = run_ok(edt, v, SQRT, True, least)
    e1, e2 = (v.dims[2], v.dims[1]) if v.ndim == 3 else (v.dims[1], v.dims[0])
    assert chunks[0] == e1 or chunks[1] == e2                # one slice per chunk somewhere
    assert_bit_equal(got, want)


def test_budget_below_one_chunk_is_enomem(edt):
  rng = np.random.default_rng(23)
  for shape in [(10, 20, 30), (30, 20, 10), (17, 40), (40, 17)]:
    labels = rng.integers(0, 3, shape).astype(np.uint16)
    v = Volume(edt, labels, np.full(shape, 63, np.uint8), (1.0,) * len(shape))
    need = least_budget(v.ndim, v.dims, v.L)
    got, chunks, rc = chunked(edt, v, 0, False, need - 1)
    assert rc == ENOMEM and chunks == [0, 0]
    msg = edt._lib().edtb200_last_error().decode()
    assert "needs at least %d bytes" % need in msg, msg
    got, chunks = run_ok(edt, v, 0, False, need)
    assert_bit_equal(got, oneshot(edt, v, 0, False))


# ---- the long-line kernel -----------------------------------------------------------------------

def _thin(rng, shape, dtype=np.uint32):
  labels = (rng.random(shape) < 0.97).astype(dtype)
  graph = np.where(rng.random(shape) < 0.9, 63, rng.integers(0, 64, shape)).astype(np.uint8)
  return labels, graph


def test_long_lines_y_phase(edt):
  """sy = 2100: the doubled Y lines (4200 cells) take the long-line kernel in phase 1."""
  rng = np.random.default_rng(24)
  labels, graph = _thin(rng, (3, 2100, 5))
  v = Volume(edt, labels, graph, (1.0, 1.0, 1.0))
  assert v.dims == [5, 2100, 3]
  for border in (False, True):
    want = oneshot(edt, v, SQRT, border)
    tight = least_budget(3, v.dims, v.L, True, False)
    for budget in (tight, 2 * tight + 7, 0):
      got, chunks = run_ok(edt, v, SQRT, border, budget)
      assert_bit_equal(got, want, (border, budget))
      assert later_kernel(edt) == "tile"                      # the Z lines are short
      assert chunks == list(plan(3, v.dims, v.L, budget or BIG, True, False)), (budget, chunks)


@pytest.mark.parametrize("ndim", [2, 3])
def test_long_lines_last_phase(edt, ndim):
  """The last axis 2100 long: its doubled lines take the long-line kernel in phase 2."""
  rng = np.random.default_rng(25)
  shape = (2100, 6, 4) if ndim == 3 else (2100, 7)
  labels, graph = _thin(rng, shape, np.uint8)
  v = Volume(edt, labels, graph, (1.0,) * ndim)
  assert v.dims[ndim - 1] == 2100
  for border in (False, True):
    want = oneshot(edt, v, 0, border)
    assert later_kernel(edt) == "long"
    tight = least_budget(ndim, v.dims, v.L, False, True)
    for budget in (tight, 3 * tight + 5, 0):
      got, chunks = run_ok(edt, v, 0, border, budget)
      assert later_kernel(edt) == "long"
      assert_bit_equal(got, want, (border, budget))
      assert chunks == list(plan(ndim, v.dims, v.L, budget or BIG, False, True)), (budget, chunks)


def test_past_the_tile_volume_limit(edt):
  """1024 x 1024 x 513 voxels: just past 2^32 / 8, so the one-shot Z pass over the doubled volume
  takes the long-line kernel, while every phase-2 chunk holds fewer than 2^32 - 64 doubled cells and
  takes the tile kernel."""
  import torch
  free, _ = torch.cuda.mem_get_info(0)
  n = 1024 * 1024 * 513
  assert 8 * n + 64 >= 1 << 32
  if free < 115 * n:                         # one-shot: inputs, mask, distances, long-line scratch
    pytest.skip("the device lacks the room for the one-shot transform")
  rng = np.random.default_rng(26)
  labels = np.ones((513, 1024, 1024), np.uint8)
  labels.reshape(-1)[rng.integers(0, n, 20000)] = 0
  graph = np.full(labels.shape, 63, np.uint8)
  graph.reshape(-1)[rng.integers(0, n, 200000)] = rng.integers(0, 64, 200000).astype(np.uint8)
  v = Volume(edt, labels, graph, (1.0, 1.0, 1.0))
  want = oneshot(edt, v, 0, True)
  assert later_kernel(edt) == "long"
  got, chunks = run_ok(edt, v, 0, True, 0)
  assert later_kernel(edt) == "tile"
  assert_bit_equal(got, want)


# ---- host buffers ---------------------------------------------------------------------------------

@pytest.mark.parametrize("pinned", [False, True])
def test_pinned_and_pageable(edt, pinned):
  rng = np.random.default_rng(27)
  small = (rng.random((12, 30, 40)) < 0.9).astype(np.uint32) * 7
  labels = np.repeat(np.repeat(np.repeat(small, 8, 0), 8, 1), 8, 2)[:90, :231, :317]    # 6.6 M voxels
  graph = np.where(rng.random(labels.shape) < 0.95, 63, rng.integers(0, 64, labels.shape)).astype(np.uint8)
  v = Volume(edt, labels, graph, (1.0, 1.0, 2.0))
  want = oneshot(edt, v, SQRT, True)
  s1 = slices(3, v.dims, v.L)[0]
  for budget in (least_budget(3, v.dims, v.L), 13 * s1, 60 * s1, 0):
    got, chunks = run_ok(edt, v, SQRT, True, budget, pinned)
    assert_bit_equal(got, want, budget)
    assert chunks == list(plan(3, v.dims, v.L, budget or BIG))


@pytest.mark.parametrize("pinned", [False, True])
def test_pitched_rows_longer_than_a_staging_buffer(edt, pinned):
  """(6, 1600, 17000) uint8 under a budget of two phase-1 slices: phase 2 in three chunks of 533 or
  534 y rows, each of whose 6 pitched rows of either cell is 36 MB, more than one 32 MiB staging
  buffer."""
  rng = np.random.default_rng(28)
  labels = np.repeat((rng.random((6, 1600, 17000 // 8)) < 0.95).astype(np.uint8), 8, axis=2)
  graph = np.where(rng.random(labels.shape) < 0.99, 63, 0b101011).astype(np.uint8)
  v = Volume(edt, labels, graph, (1.0, 1.0, 1.0))
  assert v.dims == [17000, 1600, 6]
  budget = 2 * slices(3, v.dims, v.L)[0]
  chunks_want = plan(3, v.dims, v.L, budget)
  assert chunks_want == (6, 3)
  assert 533 * 17000 * 4 > 32 << 20
  want = oneshot(edt, v, 0, False)
  got, chunks = run_ok(edt, v, 0, False, budget, pinned)
  assert chunks == list(chunks_want)
  assert_bit_equal(got, want)


# ---- concurrency ----------------------------------------------------------------------------------

def test_concurrent_oneshot_call(edt):
  rng = np.random.default_rng(29)
  vols = []
  for shape, dtype, order in [((60, 70, 80), np.uint32, "C"), ((50, 90, 40), np.uint8, "F")]:
    labels = np.asarray((rng.random(shape) < 0.9).astype(dtype), order=order)
    graph = np.asarray(np.where(rng.random(shape) < 0.8, 63, rng.integers(0, 64, shape)).astype(np.uint8), order=order)
    vols.append(Volume(edt, labels, graph, (1.0, 2.0, 3.0)))
  want = [oneshot(edt, v, SQRT, True) for v in vols]
  budget = 3 * least_budget(3, vols[0].dims, vols[0].L, True, True) + 1
  results = {}

  def work(name, fn):
    try:
      results[name] = [fn() for _ in range(4)]
    except Exception as e:                  # reported below
      results[name] = e

  jobs = [("chunked", lambda: run_ok(edt, vols[0], SQRT, True, budget)[0]),
          ("oneshot", lambda: oneshot(edt, vols[1], SQRT, True))]
  threads = [threading.Thread(target=work, args=job) for job in jobs]
  for t in threads:
    t.start()
  for t in threads:
    t.join()
  for name, idx in (("chunked", 0), ("oneshot", 1)):
    runs = results[name]
    assert not isinstance(runs, Exception), runs
    for got in runs:
      assert_bit_equal(got, want[idx], name)


# ---- against the oracle ---------------------------------------------------------------------------

@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_chunked_against_oracle(edt, oracle, seed):
  rng = np.random.default_rng(30 + seed)
  shape = [(41, 37, 29), (64, 53), (23, 50, 31), (90, 77)][seed]
  labels = (rng.random(shape) < 0.93).astype([np.uint8, np.uint32, np.float32, np.uint16][seed])
  graph = np.where(rng.random(shape) < 0.85, 63, rng.integers(0, 64, shape)).astype(np.uint8)
  an = [(1.0, 2.0, 3.0), (0.5, 1.5), (4.0, 4.0, 40.0), (1.0, 1.0)][seed]
  border = seed % 2 == 0
  v = Volume(edt, labels, graph, an)
  budget = least_budget(v.ndim, v.dims, v.L, True, True)
  got, _ = run_ok(edt, v, 0, border, budget)
  want = oracle.edtsq(labels, anisotropy=an, black_border=border, voxel_graph=graph)
  assert np.array_equal(v.reshape(got), want), seed
  got, _ = run_ok(edt, v, SQRT, border, budget)
  want = oracle.edt(labels, anisotropy=an, black_border=border, voxel_graph=graph)
  assert np.array_equal(v.reshape(got), want), seed


# ---- fallbacks ------------------------------------------------------------------------------------

def test_python_falls_back_on_enomem(edt, monkeypatch):
  rng = np.random.default_rng(31)
  x = (rng.integers(0, 5, (33, 45, 27)) * (rng.random((33, 45, 27)) < 0.9)).astype(np.int32)
  g = np.where(rng.random(x.shape) < 0.8, 63, rng.integers(0, 64, x.shape)).astype(np.uint8)
  x2, g2 = x[0], g[0]
  want_edt = edt.edt(x, anisotropy=(1.0, 2.0, 3.0), voxel_graph=g)
  want_sdf = edt.sdf(x, anisotropy=(1.0, 2.0, 3.0), voxel_graph=g, black_border=True)
  want_2d = edt.edt2dsq(x2, voxel_graph=g2)
  calls = []
  lib = edt._lib()

  def out_of_memory(*args):
    calls.append(args)
    return ENOMEM

  monkeypatch.setattr(lib, "edtb200_transform_voxel_graph", out_of_memory)
  assert_bit_equal(edt.edt(x, anisotropy=(1.0, 2.0, 3.0), voxel_graph=g).reshape(-1), want_edt.reshape(-1))
  assert len(calls) == 1
  assert_bit_equal(edt.sdf(x, anisotropy=(1.0, 2.0, 3.0), voxel_graph=g, black_border=True).reshape(-1),
                   want_sdf.reshape(-1))
  assert len(calls) == 3                                     # sdf is two transforms, each retried
  assert_bit_equal(edt.edt2dsq(x2, voxel_graph=g2).reshape(-1), want_2d.reshape(-1))
  assert len(calls) == 4


def test_python_does_not_retry_other_errors(edt, monkeypatch):
  lib = edt._lib()
  retried = []
  monkeypatch.setattr(lib, "edtb200_transform_voxel_graph", lambda *args: ECUDA)
  monkeypatch.setattr(lib, "edtb200_transform_voxel_graph_chunked", lambda *args: retried.append(args) or 0)
  with pytest.raises(edt.EDTError) as info:
    edt.edt(np.ones((4, 5, 6), np.uint8), voxel_graph=np.full((4, 5, 6), 63, np.uint8))
  assert info.value.code == ECUDA and not retried


CPP_PROGRAM = r"""
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "edt_voxel_graph.hpp"

static int wrapped = 0;
extern "C" int __wrap_edtb200_transform_voxel_graph(const void*, int, const unsigned char*, int, int64_t, int64_t,
                                                    int64_t, float, float, float, int, int, float*, int, void*) {
  ++wrapped;
  return EDTB200_ENOMEM;
}

int main(int argc, char** argv) {
  const int sx = 37, sy = 29, sz = 23;
  const size_t n = (size_t)sx * sy * sz;
  std::vector<uint32_t> labels(n);
  std::vector<uint8_t> graph(n);
  FILE* f = fopen(argv[1], "rb");
  if (!f || fread(labels.data(), 4, n, f) != n || fread(graph.data(), 1, n, f) != n) return 2;
  fclose(f);
  float* dt = pyedt::_edt3d_voxel_graph<uint32_t, uint8_t>(labels.data(), graph.data(), sx, sy, sz, 1.0f, 2.0f, 3.0f,
                                                           true);
  f = fopen(argv[2], "wb");
  fwrite(dt, 4, n, f);
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
                  "-L" + libdir, "-ledt_b200", "-Wl,-rpath," + libdir, "-Wl,--wrap=edtb200_transform_voxel_graph"],
                 check=True)
  rng = np.random.default_rng(32)
  labels = (rng.random((23, 29, 37)) < 0.9).astype(np.uint32)         # C order: x = 37 fastest
  graph = np.where(rng.random(labels.shape) < 0.8, 63, rng.integers(0, 64, labels.shape)).astype(np.uint8)
  (tmp_path / "in.bin").write_bytes(labels.tobytes() + graph.tobytes())
  res = subprocess.run([str(exe), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True,
                       text=True)
  assert res.returncode == 0, res.stderr
  assert "wrapped 1" in res.stdout
  got = np.frombuffer((tmp_path / "out.bin").read_bytes(), np.float32)
  want = edt.edt(labels, anisotropy=(3.0, 2.0, 1.0), black_border=True, voxel_graph=graph)
  assert_bit_equal(got, want.reshape(-1))
