"""GPU tests (-m gpu) of the first-axis pass alone: edtb200_pass_first on device tensors against the
oracle (tests/first_axis_cases.py), bit for bit, in every kernel instance launch_first can pick, at
the row lengths where its vector blocks and boundary words begin and end; its step tables under
retirement, many streams and many threads; and the run statistic it leaves for the later passes.

Which instance ran follows from launch_first's selection rule, restated in first_variant; the
variants reached are collected in HIT and the last test fails if a reachable one was never run.
"""
import ctypes
import threading

import numpy as np
import pytest

import envelope_cases as ec
import first_axis_cases as fc

pytestmark = pytest.mark.gpu

SQRT, SIGNED = fc.SQRT, fc.SIGNED
LENGTHS = (1, 2, 3, 4, 5, 31, 32, 33, 124, 127, 128, 129, 132, 252, 256, 257, 260, 508, 512, 513, 516, 1020,
           1023, 1024, 1025, 1028, 1056, 2048, 4096, 4097, 46342)
TORCH_VIEW = {1: np.uint8, 2: np.int16, 4: np.int32, 8: np.int64}   # same bits, a dtype torch takes
HIT = set()          # (label bytes, "vec", K, Plain) or (label bytes, "generic", 0, False)


def first_variant(nbytes, sx, lab_ptr, f_ptr, flags):
  """The kernel launch_first (csrc/edt_passes.cuh) runs for these arguments: the vector kernel with K
  128-voxel blocks per lane when rows are short, divisible by 4 and both pointers aligned, Plain when
  the kernel flags are 0 (no sqrt, background not a label); the generic kernel otherwise."""
  if sx % 4 == 0 and sx <= 1024 and lab_ptr % (4 * nbytes) == 0 and f_ptr % 16 == 0:
    k = 1 if sx <= 128 else 2 if sx <= 256 else 4 if sx <= 512 else 8
    return (nbytes, "vec", k, (flags & (SQRT | SIGNED)) == 0)
  return (nbytes, "generic", 0, False)


def reachable():
  return ({(b, "vec", k, plain) for b in fc.WIDTHS for k in (1, 2, 4, 8) for plain in (True, False)} |
          {(b, "generic", 0, False) for b in fc.WIDTHS})


def generic_limit():
  """The longest row the generic kernel takes: one warp's boundary words (16 bytes per 32 voxels) in
  one block's opt-in shared memory (launch_first_generic)."""
  import torch
  smem = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
  return (smem // 16 - 1) * 32 + 31


def to_device(lab, offset=0):
  """Labels as a flat device tensor that starts `offset` elements into its allocation."""
  import torch
  flat = np.ascontiguousarray(lab).reshape(-1)
  src = torch.from_numpy(flat.view(TORCH_VIEW[flat.dtype.itemsize]))
  buf = torch.empty(flat.size + offset, dtype=src.dtype, device="cuda")
  buf[offset:].copy_(src)
  return buf[offset:]


def device_floats(count, offset=0):
  import torch
  return torch.empty(count + offset, dtype=torch.float32, device="cuda")[offset:]


def launch(edt, lab_t, nbytes, sx, nlines, w, border, flags, f_t, stream=None):
  """edtb200_pass_first over nlines rows of sx voxels, queued on `stream` (a torch stream, None = NULL)."""
  lib = edt._lib()
  s = ctypes.c_void_p(stream.cuda_stream if stream is not None else None)
  rc = lib.edtb200_pass_first(lab_t.data_ptr(), nbytes, sx, nlines, 1, float(w), int(border), flags,
                              f_t.data_ptr(), 0, s)
  assert rc == 0, lib.edtb200_last_error()
  HIT.add(first_variant(nbytes, sx, lab_t.data_ptr(), f_t.data_ptr(), flags))


def run(edt, lab_t, nbytes, sx, nlines, w, border, flags, f_t):
  import torch
  f_t.fill_(float("nan"))                      # every voxel must be written
  torch.cuda.synchronize()
  launch(edt, lab_t, nbytes, sx, nlines, w, border, flags, f_t)
  torch.cuda.synchronize()
  return f_t[:sx * nlines].cpu().numpy().reshape(nlines, sx)


def assert_same(got, want, what):
  if not np.array_equal(got, want):
    bad = np.argwhere(~(got == want))
    first = tuple(bad[0])
    raise AssertionError("%s: %d voxels differ; first at %s: got %r want %r" % (
      what, len(bad), first, got[first], want[first]))


@pytest.mark.parametrize("nbytes", sorted(fc.WIDTHS))
def test_rows_vs_oracle(edt, oracle, nbytes):
  """Every labeling at every row length up to the generic kernel's longest: every weight, both
  borders, all four flag sets on all rows at once (a partial CTA of eight rows); each call again
  through a label pointer one element off, an output one float off, or both (the generic kernel),
  bit-equal to the aligned call; and one and seven of the rows on their own."""
  rng = np.random.default_rng(200 + nbytes)
  for n in LENGTHS + (generic_limit(),):
    lab = np.concatenate([fc.rows(rng, n, nbytes), fc.rows(rng, n, nbytes)])
    rows = lab.shape[0]
    relabelled = fc.relabel_background(lab)      # no background left: flags 0 on it is SIGNED
    lab_a, lab_o = to_device(lab), to_device(lab, 1)
    f_a, f_o = device_floats(lab.size), device_floats(lab.size, 1)
    k = 0
    for w in fc.WEIGHTS:
      for border in (0, 1):
        plain = fc.expected_first(oracle, lab, w, border, 0)
        signed = fc.expected_first(oracle, relabelled, w, border, 0)
        for flags in fc.FLAG_SETS:
          want = signed if flags & SIGNED else plain
          if flags & SQRT:
            want = np.sqrt(want)
          what = (nbytes, n, w, border, flags)
          got = run(edt, lab_a, nbytes, n, rows, w, border, flags, f_a)
          assert_same(got, want, what)
          la, fa = ((lab_o, f_a), (lab_a, f_o), (lab_o, f_o))[k % 3]
          assert_same(run(edt, la, nbytes, n, rows, w, border, flags, fa), got, what + ("offset", k % 3))
          if k % 7 == 0:
            first, count = (k // 7) % (rows - 6), (1, 7)[(k // 7) % 2]
            part = slice(first * n, (first + count) * n)
            got = run(edt, lab_a[part], nbytes, n, count, w, border, flags, f_a[part])
            assert_same(got, want[first:first + count], what + ("lines", first, count))
          k += 1


def test_row_longer_than_the_generic_kernel_takes(edt, oracle):
  """One voxel past generic_limit() the pass refuses the row (EDTB200_ELIMIT), after it has taken its
  step table; the next pass with that weight is exact."""
  n = generic_limit() + 1
  lab_t, f_t = to_device(np.ones(n, np.uint8)), device_floats(n)
  lib = edt._lib()
  rc = lib.edtb200_pass_first(lab_t.data_ptr(), 1, n, 1, 1, 0.3, 1, 0, f_t.data_ptr(), 0, ctypes.c_void_p(None))
  assert rc == -4, (rc, lib.edtb200_last_error())                  # EDTB200_ELIMIT
  lab = fc.rows(np.random.default_rng(5), 1000, 1)
  got = run(edt, to_device(lab), 1, 1000, lab.shape[0], 0.3, 1, 0, device_floats(lab.size))
  assert_same(got, fc.expected_first(oracle, lab, 0.3, 1, 0), "after the refused row")


@pytest.mark.parametrize("nbytes", sorted(fc.WIDTHS))
def test_more_lines_than_the_grid(edt, oracle, nbytes):
  """More lines than either kernel's capped grid holds warps, so that every warp loops over lines:
  4- and 1024-voxel rows on the vector kernel (and the 4-voxel rows through an offset label pointer),
  33- and 1025-voxel rows on the generic kernel."""
  import torch
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  rng = np.random.default_rng(300 + nbytes)
  cases = ((4, 40000, 0), (4, 40000, 1), (1024, sms * 12 * 8 + 1000, 0), (33, sms * 16 * 8 + 1000, 0),
           (1025, sms * 16 * 8 + 1000, 0))
  for sx, nlines, offset in cases:
    pool = np.concatenate([fc.rows(rng, sx, nbytes) for _ in range(3)])
    pick = rng.integers(0, len(pool), nlines)
    lab_t = to_device(pool[pick], offset)
    f_t = device_floats(sx * nlines)
    for w, border, flags in ((0.7, 1, 0), (1.333549976348877, 0, SQRT | SIGNED)):
      want = fc.expected_first(oracle, pool, w, border, flags)[pick]
      got = run(edt, lab_t, nbytes, sx, nlines, w, border, flags, f_t)
      assert_same(got, want, (nbytes, sx, nlines, offset, w, border, flags))
    del lab_t, f_t


def test_vector_kernel_beyond_2_31_voxels(edt, oracle):
  """2^21 + 3000 rows of 1024 one-byte labels (more than 2^31 voxels) on the vector kernel, tiled
  from 1000 rows; compared on the device with the oracle's results for those rows."""
  import torch
  free, _ = torch.cuda.mem_get_info()
  if free < (16 << 30):
    pytest.skip("needs 16 GB of free device memory, %.1f GB free" % (free / 2**30))
  rng = np.random.default_rng(31)
  sx, nlines, distinct = 1024, (1 << 21) + 3000, 1000
  pool = np.stack([fc.labeling(rng, fc.LABELINGS[i % len(fc.LABELINGS)], sx, 1) for i in range(distinct)])
  pool_t = torch.from_numpy(pool).cuda()
  lab_t = pool_t.repeat(-(-nlines // distinct), 1)[:nlines].reshape(-1)
  f_t = device_floats(sx * nlines)
  assert f_t.numel() > 2**31
  assert first_variant(1, sx, lab_t.data_ptr(), f_t.data_ptr(), 0)[1] == "vec"
  f2 = f_t.view(nlines, sx)
  for w, border, flags in ((0.7, 1, 0), (1.333549976348877, 0, SQRT | SIGNED)):
    f_t.fill_(float("nan"))
    torch.cuda.synchronize()
    launch(edt, lab_t, 1, sx, nlines, w, border, flags, f_t)
    torch.cuda.synchronize()
    want = torch.from_numpy(fc.expected_first(oracle, pool, w, border, flags)).cuda()
    step = 100 * distinct
    for start in range(0, nlines, step):
      end = min(nlines, start + step)
      idx = torch.arange(start, end, device="cuda") % distinct
      if not torch.equal(f2[start:end], want[idx]):
        bad = (f2[start:end] != want[idx]).nonzero()[0].tolist()
        raise AssertionError("%s: row %d voxel %d differs" % ((w, border, flags), start + bad[0], bad[1]))
  del lab_t, f_t, f2, pool_t


def test_step_tables_retire_and_rebuild(edt, oracle):
  """40 X weights, more than the 16 cached step tables, on 4500-voxel rows (tables of more than 4096
  entries), queued over the NULL stream and five side streams with no synchronisation between them.
  Weight i is used on 1 + i % 6 streams, so some tables have more user streams than are tracked and
  are retired after a device-wide synchronisation; then the first weights again, whose tables were
  retired meanwhile."""
  import torch
  rng = np.random.default_rng(41)
  sx = 4500
  lab = fc.rows(rng, sx, 4)[:5]
  lab_t = to_device(lab)
  streams = [None] + [torch.cuda.Stream() for _ in range(5)]
  weights = [float(np.float32(0.55 + 0.0173 * i)) for i in range(40)]
  plan = [(w, streams[(i + j) % 6]) for i, w in enumerate(weights) for j in range(1 + i % 6)]
  plan += [(weights[i], streams[(i + 3) % 6]) for i in range(10)]
  outs = [device_floats(lab.size) for _ in plan]
  for f_t in outs:
    f_t.fill_(float("nan"))
  torch.cuda.synchronize()
  lib = edt._lib()
  for (w, s), f_t in zip(plan, outs):
    ptr = ctypes.c_void_p(s.cuda_stream if s is not None else None)
    rc = lib.edtb200_pass_first(lab_t.data_ptr(), 4, sx, lab.shape[0], 1, w, 1, 0, f_t.data_ptr(), 0, ptr)
    assert rc == 0, lib.edtb200_last_error()
  torch.cuda.synchronize()
  want = {w: fc.expected_first(oracle, lab, w, 1, 0) for w in weights}
  for i, ((w, s), f_t) in enumerate(zip(plan, outs)):
    assert_same(f_t.cpu().numpy().reshape(lab.shape), want[w], ("call", i, w))


def test_step_tables_from_eight_threads(edt, oracle):
  """Eight host threads on one device, each on its own stream with five weights of its own (40 in
  all), three rounds each without synchronising: tables are built, used and retired while other
  threads are between taking a table and queueing the kernel that reads it.  Rows of 4500 voxels
  (generic kernel) and 1000 (vector kernel) alternate."""
  import torch
  rng = np.random.default_rng(43)
  shapes = {4500: fc.rows(rng, 4500, 2)[:4], 1000: fc.rows(rng, 1000, 2)[:4]}
  labs = {sx: to_device(lab) for sx, lab in shapes.items()}
  weights = [[float(np.float32(2.05 + 0.0311 * (5 * t + j))) for j in range(5)] for t in range(8)]
  jobs = [[(r, j, (4500, 1000)[(r + j) % 2]) for r in range(3) for j in range(5)] for t in range(8)]
  outs = [[device_floats(shapes[sx].size) for (_, _, sx) in jobs[t]] for t in range(8)]
  streams = [torch.cuda.Stream() for _ in range(8)]
  for row in outs:
    for f_t in row:
      f_t.fill_(float("nan"))
  torch.cuda.synchronize()
  lib = edt._lib()
  errors = []

  def worker(t):
    try:
      ptr = ctypes.c_void_p(streams[t].cuda_stream)
      for (r, j, sx), f_t in zip(jobs[t], outs[t]):
        rc = lib.edtb200_pass_first(labs[sx].data_ptr(), 2, sx, 4, 1, weights[t][j], r % 2, 0, f_t.data_ptr(), 0,
                                    ptr)
        if rc != 0:
          errors.append((t, r, j, lib.edtb200_last_error()))
    except Exception as e:        # reported by the main thread
      errors.append((t, repr(e)))

  threads = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
  for th in threads:
    th.start()
  for th in threads:
    th.join()
  torch.cuda.synchronize()
  assert not errors, errors
  for t in range(8):
    for (r, j, sx), f_t in zip(jobs[t], outs[t]):
      want = fc.expected_first(oracle, shapes[sx], weights[t][j], r % 2, 0)
      assert_same(f_t.cpu().numpy().reshape(want.shape), want, (t, r, j, sx))


def change_rows(rng, sx, nrows, changes):
  """nrows rows of sx voxels (labels 1 and 2) with exactly `changes` label changes each."""
  out = np.empty((nrows, sx), np.uint32)
  for r in range(nrows):
    cut = np.zeros(sx, np.int64)
    cut[1 + rng.choice(sx - 1, changes, replace=False)] = 1
    out[r] = 1 + np.cumsum(cut) % 2
  return out


def later_ctas(edt, oracle, rng):
  """CTAs per SM of a tile/TMA pass_later on a (200, 4, 8) volume: 2 when the run statistic the last
  first-axis pass published says label noise (runs per voxel >= 0.9), else 3."""
  import torch
  shape = (200, 4, 8)
  lab = ec.labels(rng, "runs", shape, 2, np.uint32)
  f = ec.profile(rng, "int_ties", shape)
  lt = to_device(lab)
  ft = torch.from_numpy(f.copy()).cuda()
  lib = edt._lib()
  rc = lib.edtb200_pass_later(lt.data_ptr(), 4, 2, 8, 4, 200, 1.0, 1, 0, 0, ft.data_ptr(), 0, ctypes.c_void_p(None))
  assert rc == 0, lib.edtb200_last_error()
  torch.cuda.synchronize()
  v = edt.last_later_launch()
  assert v["kernel"] == "tile" and v["tx"] == 32 and v["tma"] == 1 and v["wide"] == 0, v
  assert_same(ft.cpu().numpy(), ec.expected_pass(oracle, lab, f, 2, 1.0, 1, 0), "later pass")
  return v["ctas"]


def check_steering(edt, oracle, rng, nrows, what):
  """0.92 and then 0.88 label changes per voxel on both kernels (the vector kernel on aligned 100-voxel
  rows, the generic kernel on the same rows one label off), no border: the later pass must follow."""
  for offset in (0, 1):
    for changes, ctas in ((92, 2), (88, 3)):
      lab = change_rows(rng, 100, nrows, changes)
      lab_t, f_t = to_device(lab, offset), device_floats(lab.size)
      got = run(edt, lab_t, 4, 100, nrows, 1.0, 0, 0, f_t)
      assert first_variant(4, 100, lab_t.data_ptr(), f_t.data_ptr(), 0)[1] == ("generic" if offset else "vec")
      assert_same(got, fc.expected_first(oracle, lab, 1.0, 0, 0), (what, nrows, offset, changes))
      assert later_ctas(edt, oracle, rng) == ctas, (what, nrows, offset, changes)


def test_run_statistic_steers_the_later_pass(edt, oracle):
  """The run statistic each kernel publishes steers the next tile pass between 2 and 3 CTAs per SM;
  it still does after two first-axis passes with different grid sizes ran at the same time on two
  streams (a one-CTA grid next to a grid of whole waves), on grids of one CTA and of eight."""
  import torch
  rng = np.random.default_rng(51)
  for nrows in (8, 64):
    check_steering(edt, oracle, rng, nrows, "alone")
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  big = rng.integers(0, 3, (sms * 12 * 8 * 4, 1024)).astype(np.uint8)
  small = change_rows(rng, 100, 8, 50)
  big_t, small_t = to_device(big), to_device(small)
  fb, fs = device_floats(big.size), device_floats(small.size)
  s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
  fb.fill_(float("nan"))
  fs.fill_(float("nan"))
  torch.cuda.synchronize()
  launch(edt, big_t, 1, 1024, big.shape[0], 1.0, 0, 0, fb, stream=s1)
  launch(edt, small_t, 4, 100, 8, 1.0, 0, 0, fs, stream=s2)
  torch.cuda.synchronize()
  assert_same(fs.cpu().numpy().reshape(small.shape), fc.expected_first(oracle, small, 1.0, 0, 0), "small")
  assert_same(fb.cpu().numpy().reshape(big.shape), fc.expected_first(oracle, big, 1.0, 0, 0), "big")
  for nrows in (8, 64):
    check_steering(edt, oracle, rng, nrows, "after two concurrent passes")


@pytest.fixture(autouse=True)
def _record_run(request):
  yield
  RAN.add(request.node.name)


RAN = set()
PRODUCERS = {"test_rows_vs_oracle[%d]" % b for b in fc.WIDTHS}


def test_every_first_axis_variant_was_run():
  """The first-axis instances the tests above reached, against the 36 launch_first can pick.
  Meaningful only after the row tests have run in this process; skipped otherwise."""
  if not PRODUCERS <= RAN:
    pytest.skip("the variant-producing tests of this file did not run before this one: %s" % sorted(PRODUCERS - RAN))
  want = reachable()
  print("\nfirst-axis variants run (%d of %d reachable):" % (len(HIT & want), len(want)))
  print("  " + " ".join("%8s" % f for f in ("bytes", "kernel", "K", "Plain")))
  for row in sorted(HIT, key=repr):
    print("  " + " ".join("%8s" % v for v in row))
  assert not HIT - want, sorted(HIT - want, key=repr)
  assert not want - HIT, sorted(want - HIT, key=repr)
