"""CPU tests (gloo, world_size 2 and 3) of the slab-split host logic in
euclidean-distance-transform-3d_b200/distributed.py.

There is no GPU here, so the per-axis device entry points are replaced by the oracle's per-axis
passes (test infrastructure) -- what is under test is the decomposition itself: slab geometry,
the Z-slab <-> Y-slab exchange, border flags, uneven and empty slabs.  The same code runs over
NCCL in the `-m gpu` test below and in bench.py --gpus N.
"""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import slab_cases  # noqa: E402
from slab_cases import OraclePasses  # noqa: E402


def _free_port():
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    return s.getsockname()[1]


def _volume(case):
  shape, kind = case[0], case[1]
  rng = np.random.default_rng(1234)
  if kind == "iid":
    vol = rng.integers(0, 4, shape)
  elif kind == "ones":
    vol = np.ones(shape, dtype=np.int64)
    vol[tuple(s // 2 for s in shape)] = 0
  elif kind == "solid":
    vol = np.full(shape, 7, dtype=np.int64)
  elif kind == "tie":
    vol = slab_cases.tie_volume(case[6])[0]
  elif kind == "trap":
    vol = slab_cases.stop_trap(case[6])[0]
  elif kind == "span":
    vol = slab_cases.span_volume(shape)
  elif kind == "stripes":       # z-runs of length 2 starting at odd z (slab faces cut them), some background
    z, y, x = np.meshgrid(*[np.arange(s) for s in shape], indexing="ij")
    vol = 1 + ((z + 1) // 2 + x + 2 * y) % 3
    vol[(x + y) % 4 == 0] = 0
    vol[:, 1, 1] = np.where(np.arange(shape[0]) % 3 == 0, 0, 5)
  else:
    small = rng.integers(0, 3, tuple((s + 4) // 5 for s in shape))
    vol = np.repeat(np.repeat(np.repeat(small, 5, 0), 5, 1), 5, 2)[:shape[0], :shape[1], :shape[2]]
  return np.ascontiguousarray(vol.astype(np.int32))


def _worker(rank, world, port, queue):
  sys.path.insert(0, ROOT)
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    _worker_body(rank, world, queue)
  except Exception as exc:          # surface the failure instead of letting the peers time out
    import traceback
    queue.put(("error", rank, traceback.format_exc()))
    raise
  finally:
    dist.destroy_process_group()


def _worker_body(rank, world, queue):
  if True:
    import edt_b200.distributed as ed
    for idx, case in enumerate(CASES):
      shape, kind, an, bb, sqrt, signed, depths = case
      if depths is not None and len(depths) != world:
        continue
      vol = _volume(case)
      if depths is None:
        parts = ed.split_extent(shape[0], world)
      else:
        starts = np.cumsum([0] + list(depths[:-1]))
        parts = list(zip(starts.tolist(), depths))
      z0, zc = parts[rank]
      local = torch.from_numpy(vol[z0:z0 + zc].copy())
      for halo in (2, 64):            # 2: the halo method where it is exact; 64: always the transpose
        info = {}
        # (odd cases take the transposition without the packed exchange layout)
        out = ed.slab_transform(local, an, bb, sqrt=sqrt, signed=signed, passes=OraclePasses(packed=idx % 2 == 0),
                                halo=halo, info=info)
        queue.put((idx, halo, info["method"], rank, z0, out.numpy()))


CASES = [
  ((12, 9, 7), "iid", (1.0, 1.0, 1.0), False, False, False, None),
  ((12, 9, 7), "iid", (3.0, 2.0, 1.0), True, True, False, None),
  ((11, 5, 6), "blocks", (1.0, 2.0, 3.0), False, False, True, None),
  ((10, 4, 9), "ones", (1.0, 1.0, 1.0), False, False, False, None),       # inf-rich, long z runs
  ((10, 4, 9), "ones", (2.0, 1.0, 1.0), True, True, True, None),
  ((7, 3, 4), "blocks", (1.0, 1.0, 1.0), True, False, False, (7, 0)),     # an empty slab
  ((7, 3, 4), "blocks", (1.0, 1.0, 1.0), False, True, True, (0, 3, 4)),   # an empty first slab
  ((12, 5, 6), "stripes", (1.0, 1.0, 1.0), False, False, False, None),    # halo method applies
  ((12, 5, 6), "stripes", (2.0, 3.0, 1.0), True, True, True, None),
  ((13, 4, 5), "stripes", (0.7, 1.0, 1.3), False, True, False, None),
  # runs far longer than the halo (2 rows): still exact through the halo when the distances at the
  # faces stay within its reach (w_z = 3: reach 6 >= the <= 3 voxels to the x / y borders) ...
  ((16, 5, 7), "solid", (3.0, 1.0, 1.0), True, False, False, None),
  ((16, 5, 7), "solid", (3.0, 1.0, 1.0), True, True, True, None),
  # ... and not when they do not (w_z = 1: reach 2 < 3): the verdict sends it to the transpose
  ((16, 5, 7), "solid", (1.0, 1.0, 1.0), True, False, False, None),
  # ... unless the slabs are deep enough for the next halo depth (2 -> 8 rows: world 2 has 10-row slabs)
  ((20, 5, 7), "solid", (1.0, 1.0, 1.0), True, False, False, None),
  # the fix-up's traps (tests/slab_cases.py): a double-rounding tie three rows behind a face ...
  ((9, 1, 2), "tie", slab_cases.TIE_W, False, False, False, (3, 6)),
  ((12, 1, 2), "tie", slab_cases.TIE_W, False, False, False, (3, 6, 3)),
  # ... a rounded tie more than 4096 rows behind a face with a strictly lower row after it ...
  ((12000, 1, 2), "trap", slab_cases.TRAP_W, False, False, False, (6000, 6000)),
  ((12100, 1, 2), "trap", slab_cases.TRAP_W, False, False, False, (100, 6000, 6000)),
  # ... and a run spanning the middle slab of three, walked from both faces
  ((14, 3, 4), "span", (1.0, 1.0, 1.0), False, False, False, None),
  ((14, 3, 4), "span", (2.0, 1.0, 1.0), False, True, True, None),
]
# method taken when starting with halo=2, per world size
EXPECT_HALO2 = {10: {2: "halo", 3: "halo"}, 11: {2: "halo", 3: "halo"}, 12: {2: "transpose", 3: "transpose"},
                13: {2: "halo", 3: "transpose"}, 14: {2: "halo"}, 15: {3: "halo"}, 16: {2: "halo"}, 17: {3: "halo"},
                18: {2: "transpose", 3: "halo"}, 19: {2: "transpose", 3: "halo"}}
# with halo=64 only slabs deeper than 64 rows can take the halo method
EXPECT_HALO64 = {16: {2: "halo"}, 17: {3: "halo"}}


@pytest.mark.parametrize("world", [2, 3])
def test_slab_split_matches_single_volume(world):
  sys.path.insert(0, ROOT)
  from oracle import oracle
  ctx = mp.get_context("spawn")
  queue = ctx.Queue()
  port = _free_port()
  procs = [ctx.Process(target=_worker, args=(r, world, port, queue)) for r in range(world)]
  for p in procs:
    p.start()
  active = [i for i, c in enumerate(CASES) if c[6] is None or len(c[6]) == world]
  results = []
  for _ in range(2 * world * len(active)):
    item = queue.get(timeout=300)
    assert item[0] != "error", item
    results.append(item)
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  assert len(active) >= 6
  used = set()
  for idx in active:
    case = CASES[idx]
    shape, kind, an, bb, sqrt, signed, _ = case
    fn = {(False, False): oracle.edtsq, (True, False): oracle.edt,
          (False, True): oracle.sdfsq, (True, True): oracle.sdf}[(sqrt, signed)]
    want = fn(_volume(case), anisotropy=an, black_border=bb)    # the same volume, not distributed
    for halo in (2, 64):
      got = np.zeros(shape, dtype=np.float32)
      methods = set()
      for i, h, method, rank, z0, arr in results:
        if i == idx and h == halo:
          got[z0:z0 + arr.shape[0]] = arr
          methods.add(method)
      assert len(methods) == 1, (world, idx, halo, methods)       # every rank took the same path
      if halo == 64:
        assert methods == {EXPECT_HALO64.get(idx, {}).get(world, "transpose")}, (world, idx, methods)
      elif idx in EXPECT_HALO2:
        assert methods == {EXPECT_HALO2[idx][world]}, (world, idx, methods)
      used.add((idx, methods.pop()))
      assert np.array_equal(got, want, equal_nan=True), (world, idx, halo)
  assert any(m == "halo" for _, m in used) and any(m == "transpose" for _, m in used), used


def _deferred_worker(rank, world, port, queue):
  """defer_check=True / "local": verdicts are collected over a batch of steps and read once."""
  sys.path.insert(0, ROOT)
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    import edt_b200.distributed as ed

    def step(idx, mode):
      shape, kind, an, bb, sqrt, signed, _ = CASES[idx]
      z0, zc = ed.split_extent(shape[0], world)[rank]
      local = torch.from_numpy(_volume(CASES[idx])[z0:z0 + zc].copy())
      info = {}
      out = ed.slab_transform(local, an, bb, sqrt=sqrt, signed=signed, passes=OraclePasses(), halo=2, info=info,
                              defer_check=mode)
      assert info["method"] == "halo"
      return idx, z0, out.numpy(), info["verdict"]

    report = {}
    for mode in (True, "local"):
      clean = [step(idx, mode) for idx in (7, 8, 9, 10, 11)]      # the halo is exact for these
      report[("clean", mode)] = ed.check_verdicts([v for *_, v in clean])
      dirty = clean[:2] + [step(12, mode)]                        # ... and one step where it is not
      report[("dirty", mode)] = ed.check_verdicts([v for *_, v in dirty])
      if mode == "local":
        assert all(work is None for *_, (flag, work) in clean)    # no collective inside the steps
        for idx, z0, arr, _ in clean:
          queue.put((idx, rank, z0, arr))
    queue.put(("report", rank, report))
  except Exception:
    import traceback
    queue.put(("error", rank, traceback.format_exc()))
    raise
  finally:
    dist.destroy_process_group()


def test_deferred_verdicts_are_combined_once_per_batch():
  sys.path.insert(0, ROOT)
  from oracle import oracle
  world = 2
  ctx = mp.get_context("spawn")
  queue = ctx.Queue()
  port = _free_port()
  procs = [ctx.Process(target=_deferred_worker, args=(r, world, port, queue)) for r in range(world)]
  for p in procs:
    p.start()
  items = []
  for _ in range(world * 6):
    item = queue.get(timeout=300)
    assert item[0] != "error", item
    items.append(item)
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  reports = [it[2] for it in items if it[0] == "report"]
  assert len(reports) == world
  for rep in reports:                    # every rank reaches the same conclusion
    assert rep == {("clean", True): True, ("dirty", True): False, ("clean", "local"): True, ("dirty", "local"): False}
  for idx in (7, 8, 9, 10, 11):
    shape, kind, an, bb, sqrt, signed, _ = CASES[idx]
    fn = {(False, False): oracle.edtsq, (True, False): oracle.edt,
          (False, True): oracle.sdfsq, (True, True): oracle.sdf}[(sqrt, signed)]
    got = np.zeros(shape, dtype=np.float32)
    for it in items:
      if it[0] == idx:
        got[it[2]:it[2] + it[3].shape[0]] = it[3]
    assert np.array_equal(got, fn(_volume(CASES[idx]), anisotropy=an, black_border=bb), equal_nan=True), idx


@pytest.mark.gpu
def test_slab_pack_kernel_against_slicing():
  """edtb200_slab_pack (one launch, either direction) == slicing the slab per rank and concatenating."""
  sys.path.insert(0, ROOT)
  import edt_b200.distributed as ed
  dev = torch.device("cuda", 0)
  passes = ed.CudaPasses(dev)
  gen = torch.Generator(device="cpu").manual_seed(5)
  for zc, sy, sx, dtype, world in ((7, 20, 64, torch.float32, 3), (5, 9, 33, torch.uint8, 4), (3, 8, 10, torch.int16, 8),
                                   (4, 512, 128, torch.float32, 8), (0, 6, 4, torch.float32, 2), (6, 5, 12, torch.int64, 7)):
    ysplit = ed.split_extent(sy, world)                      # world > sy: some parts are empty
    src = torch.randint(0, 120, (zc, sy, sx), generator=gen).to(dtype).to(dev)
    packed = torch.empty(src.numel(), dtype=dtype, device=dev)
    passes.repartition(src, packed, ysplit)
    want = torch.cat([src[:, s:s + c, :].reshape(-1) for s, c in ysplit]) if src.numel() else packed
    assert torch.equal(packed, want), (zc, sy, sx, dtype, world)
    back = torch.full_like(src, 99)
    passes.repartition(packed, back, ysplit, unpack=True)
    assert torch.equal(back, src), (zc, sy, sx, dtype, world, "unpack")
  with pytest.raises(ed.EDTError):
    passes.repartition(torch.zeros((2, 4, 4), device=dev), torch.zeros(32, device=dev), [(2, 1), (1, 3)])   # not rising from 0


def test_split_extent():
  sys.path.insert(0, ROOT)
  import edt_b200.distributed as ed
  assert ed.split_extent(10, 3) == [(0, 4), (4, 3), (7, 3)]
  assert ed.split_extent(2, 4) == [(0, 1), (1, 1), (2, 0), (2, 0)]
  assert sum(c for _, c in ed.split_extent(4096, 8)) == 4096


def test_halo_ladder():
  """The halos a slab_transform call tries before the transposition (tests/test_slab_ladder.py runs them)."""
  sys.path.insert(0, ROOT)
  import edt_b200.distributed as ed
  ladder = ed._halo_ladder
  assert ladder("auto", 2, 10, 2) == [2, 8]                   # 32 does not fit into 10-row slabs
  assert ladder("auto", 2, 5, 3) == [2]
  assert ladder("auto", 8, 1000, 2) == [8, 32, 128]
  assert ladder("auto", 8, 40, 2) == [8, 32]
  assert ladder("auto", 100, 1000, 2) == [100, 128]
  assert ladder("auto", 128, 1000, 2) == [128]
  assert ladder("auto", 254, 255, 2) == [254]                 # 128 is not deeper than 254
  assert ladder("auto", 64, 64, 2) == []                      # slabs must be deeper than the halo
  assert ladder("halo", 8, 1000, 2) == [8]                    # one attempt, no retry
  assert ladder("halo", 8, 8, 2) == []
  assert ladder("transpose", 8, 1000, 2) == []
  assert ladder("auto", 8, 1000, 1) == ladder("halo", 8, 1000, 1) == []


# ---------------------------------------------------------------------------------------
# the real thing: NCCL over 2 GPUs (skipped unless the box has at least two)
# ---------------------------------------------------------------------------------------

def _nccl_worker(rank, world, port, queue):
  sys.path.insert(0, ROOT)
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  torch.cuda.set_device(rank)
  dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
  try:
    import edt_b200
    import edt_b200.distributed as ed
    rng = np.random.default_rng(99)
    peer_halo, peer_why = ed.make_peer_halo(torch.device("cuda", rank), 54, 70, torch.int32, 32)
    # (a) z-runs of exactly 4 planes plus an iid region: the halo method is exact here
    z, y, x = np.meshgrid(np.arange(143), np.arange(54), np.arange(70), indexing="ij")
    vol_a = (1 + ((z // 4) + (y // 9) * 3 + (x // 10) * 7) % 5).astype(np.int32)
    vol_a[60:90, 10:30, 5:50] = rng.integers(0, 3, (30, 20, 45))
    # (b) big blocks: runs longer than the halo (48 planes), but no voxel is further than 32 w_z from
    # its region's boundary (the plane is 54 x 70), so the halo's reach check passes
    small = rng.integers(0, 2, (3, 6, 7))
    vol_b = np.repeat(np.repeat(np.repeat(small, 48, 0), 9, 1), 10, 2).astype(np.int32)[:143]
    # (c) one label, one background voxel in a corner: the distances at the slab face (~70) are
    # beyond the halo's reach, "auto" must notice and fall back
    vol_c = np.full((143, 54, 70), 3, dtype=np.int32)
    vol_c[0, 0, 0] = 0
    # with the black border and w_z = 3 even (c) is within reach: nothing is further than 27 from a y border
    for vol, expects in ((vol_a, ("halo", "halo")), (vol_b, ("halo", "halo")), (vol_c, ("transpose", "halo"))):
      for expect, (bb, sqrt, signed, an) in zip(expects, ((False, False, False, (1.0, 1.0, 1.0)),
                                                          (True, True, True, (3.0, 1.0, 2.0)))):
        parts = ed.split_extent(vol.shape[0], world)
        z0, zc = parts[rank]
        local = torch.from_numpy(vol[z0:z0 + zc].copy()).cuda()
        whole = edt_b200.edt_cuda(torch.from_numpy(vol).cuda(), an, bb, sqrt=sqrt, signed=signed)
        for method, peer in (("auto", None), ("transpose", None), ("auto", peer_halo), ("auto", "auto")):
          info = {}
          out = ed.slab_transform(local, an, bb, sqrt=sqrt, signed=signed, method=method, info=info,
                                  peer_halo=peer)
          torch.cuda.synchronize()
          want_method = expect if method == "auto" else "transpose"
          bad = int((out != whole[z0:z0 + zc]).sum().item())
          queue.put((rank, bad == 0 and info["method"] == want_method, bad, info["method"], want_method,
                     "nccl" if peer is None else "peer", peer_why))
  finally:
    dist.destroy_process_group()


@pytest.mark.gpu
def test_slab_split_nccl_two_gpus():
  if torch.cuda.device_count() < 2:
    pytest.skip("needs two GPUs")
  ctx = mp.get_context("spawn")
  queue = ctx.Queue()
  port = _free_port()
  procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, queue)) for r in range(2)]
  for p in procs:
    p.start()
  results = [queue.get(timeout=300) for _ in range(48)]
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  assert all(r[1] for r in results), [r for r in results if not r[1]]


# ---------------------------------------------------------------------------------------
# several GPUs behind the boundary: one process, one host volume (edtb200_transform_multi)
# ---------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_transform_multi_devices_in_one_process():
  sys.path.insert(0, ROOT)
  import edt_b200
  from oracle import oracle
  ndev = torch.cuda.device_count()
  if ndev < 2:
    pytest.skip("needs two GPUs")
  rng = np.random.default_rng(5)
  small = rng.integers(0, 5, (9, 7, 11))
  lab = np.asfortranarray(np.repeat(np.repeat(np.repeat(small, 9, 0), 13, 1), 10, 2).astype(np.uint16))  # 81x91x110
  lab[3:70, 5:80, 20:90][rng.uniform(size=(67, 75, 70)) < 0.3] = 0
  devs = list(range(min(ndev, 4)))
  for fn, kw in (("edtsq", dict(anisotropy=(1, 1, 1))), ("edt", dict(anisotropy=(2, 1, 3), black_border=True)),
                 ("sdf", dict(anisotropy=(1.5, 0.5, 2.5)))):
    want = getattr(oracle, fn)(lab, **kw)
    got = getattr(edt_b200, fn)(lab, devices=devs, **kw)
    assert got.flags.f_contiguous and np.array_equal(got, want), fn
    got_c = getattr(edt_b200, fn)(np.ascontiguousarray(lab), devices=devs, **kw)
    assert np.array_equal(got_c, want), (fn, "C order")
  # a volume too thin to split falls back to the first device
  thin = np.asfortranarray(lab[:, :, :1])
  assert np.array_equal(edt_b200.edtsq(thin, devices=devs), oracle.edtsq(thin))


@pytest.mark.gpu
def test_two_threads_on_two_gpus_overlap():
  """Host-buffer transforms on different GPUs from different threads must run concurrently
  (per-device locks, no library-wide mutex).  Page-locked buffers, so that what is measured is
  the library and the two PCIe links, not the host's page-fault path: two calls at once on two
  GPUs must take less than 1.3 x one call alone."""
  sys.path.insert(0, ROOT)
  import ctypes
  import threading
  import time
  import edt_b200
  if torch.cuda.device_count() < 2:
    pytest.skip("needs two GPUs")
  lib = edt_b200._lib()
  n = 384
  gen = torch.Generator().manual_seed(6)
  labs = [torch.randint(0, 256, (n, n, n), dtype=torch.int32, generator=gen).pin_memory() for _ in range(2)]
  outs = [torch.empty((n, n, n), dtype=torch.float32).pin_memory() for _ in range(2)]

  def call(d):
    rc = lib.edtb200_transform(labs[d].data_ptr(), 4, 3, n, n, n, 1.0, 1.0, 1.0, 0, 0, outs[d].data_ptr(), d, None)
    assert rc == 0, lib.edtb200_last_error()

  for d in range(2):
    call(d)                                              # warm-up: buffers, streams, tables
  first = outs[0].clone()
  alone = []
  for _ in range(3):
    t0 = time.perf_counter()
    call(0)
    alone.append(time.perf_counter() - t0)
  both = []
  for _ in range(3):
    threads = [threading.Thread(target=call, args=(d,)) for d in range(2)]
    t0 = time.perf_counter()
    for t in threads:
      t.start()
    for t in threads:
      t.join()
    both.append(time.perf_counter() - t0)
  assert torch.equal(outs[0], first)
  assert min(both) < 1.3 * min(alone), (alone, both)


def _run_slab_check(nproc, extra, timeout):
  import subprocess
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
         "--master-addr", "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "tools", "slab_check.py")] + extra
  res = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=timeout)
  assert res.returncode == 0, res.stdout + res.stderr
  assert "OK" in res.stdout, res.stdout


@pytest.mark.gpu
def test_slab_check_all_gpus_of_the_box():
  """The fused slab step (symmetric-memory staging, flag words) on every GPU of the box against the
  single-GPU transform: edtsq, edt with a border, sdf on 512 x 512 x (64 * N) blocks."""
  n = torch.cuda.device_count()
  if n < 2:
    pytest.skip("needs two GPUs")
  _run_slab_check(n, ["--depth", "64"], 900)


@pytest.mark.gpu
def test_cfg5_512x512x4096_sdf_eight_gpus():
  """BASELINE.json configs[4] as written: 512 x 512 x 4096 uint32 multi-label, Z slabs over 8 GPUs,
  sdf -- every rank's slab bit-equal to the single-GPU sdf of the whole volume."""
  if torch.cuda.device_count() < 8:
    pytest.skip("needs eight GPUs")
  _run_slab_check(8, ["--full"], 1800)
