"""CPU tests (gloo, world sizes 2 and 3) that pin which attempts slab_transform makes for a call, in
which order, and which collectives every rank issues.  Every rank must make the same collective
calls in the same order or the job hangs, so this ladder is part of slab_transform's behaviour:

  * the starting halo is the `halo` argument, else the halo of an explicit PeerHalo, else the depth
    the last clean method="auto" call on the same group and plane shape needed ("auto" only), else
    DEFAULT_HALO;
  * a halo attempt runs only when world > 1 and every slab is deeper than its halo;
  * after a dirty verdict, "auto" tries min(4 * halo, 128) when that is deeper than the halo and the
    slabs are deeper still, and otherwise the transposition; method="halo" raises;
  * a deferred verdict ends the call after its first attempt.

`ScriptedPasses` runs the oracle's per-axis passes but takes every attempt's verdict from a script.
Its slab_step (the fused step, which needs GPUs) records its arguments and writes a scripted
status, and a PeerHalo built without symmetric memory stands in for the staging buffer.
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

PLANE = (2, 3)


def _addr(rank):
  """Address of `rank`'s stand-in staging buffer."""
  return 0x10000 * (rank + 1)


class _Mapped:
  def __init__(self, addr):
    self.addr = addr

  def data_ptr(self):
    return self.addr


class _Handle:
  def get_buffer(self, rank, shape, dtype, offset):
    return _Mapped(_addr(rank))


class ScriptedPasses(slab_cases.OraclePasses):
  """OraclePasses that logs every call.  `dirty`: halos at which the NCCL path's fix-up raises its
  verdict; `status`: {halo: value} that the fused slab_step writes into its status word."""

  def __init__(self, log, dirty=(), status=None):
    super().__init__()
    self.log, self.dirty, self.script = log, set(dirty), dict(status or {})

  def pass_first(self, labels, f, wx, black_border, signed):
    self.log.append(("pass_first", None))
    super().pass_first(labels, f, wx, black_border, signed)

  def face_runs(self, labels, high_face, halo, signed, overflow, out=None):
    self.log.append(("face_runs", halo))
    return super().face_runs(labels, high_face, halo, signed, overflow, out)

  def face_fixup(self, labels, f, high_face, halo, wz, sqrt, signed, nb_label, nb_m, nb_f, inexact):
    self.log.append(("face_fixup", halo))
    if halo in self.dirty:
      inexact[0] = 1

  def slab_step(self, labels, f, w_xyz, black_border, has_lo, has_hi, sqrt, signed, halo, sym_self, sym_lo, sym_hi,
                step, status):
    self.log.append(("slab_step", dict(halo=halo, w_xyz=tuple(w_xyz), has_lo=bool(has_lo), has_hi=bool(has_hi),
                                       sym_self=sym_self, sym_lo=sym_lo, sym_hi=sym_hi, step=step)))
    status[0] = self.script.get(halo, 0)


def attempts(log, world):
  """The call's attempts as (transport, halo): ("fused", h), ("exchange", h), then ("transpose", None)
  (("single", None) for a group of one).  Every attempt but the fused one starts with the X pass,
  and the NCCL exchange computes its face run lengths just before."""
  out, runs = [], None
  for name, arg in log:
    if name == "slab_step":
      out.append(("fused", arg["halo"]))
    elif name == "face_runs":
      runs = arg
    elif name == "pass_first":
      out.append(("exchange", runs) if runs is not None else ("transpose" if world > 1 else "single", None))
      runs = None
  return out


class Caller:
  """Runs one slab_transform call on this rank's slab of a seeded volume and returns what the tests pin."""

  def __init__(self, ed, rank, world):
    self.ed, self.rank, self.world = ed, rank, world
    self.collectives = []
    real_all_reduce, real_batch = dist.all_reduce, dist.batch_isend_irecv

    def all_reduce(*args, **kw):
      self.collectives.append(("all_reduce", bool(kw.get("async_op", False))))
      return real_all_reduce(*args, **kw)

    def batch_isend_irecv(ops):
      self.collectives.append(("batch_isend_irecv", False))
      return real_batch(ops)
    dist.all_reduce, dist.batch_isend_irecv = all_reduce, batch_isend_irecv

  def staging(self, halo, plane=PLANE):
    """A PeerHalo stand-in: the fields slab_transform reads, and stand-in addresses for peer_ptr."""
    ph = object.__new__(self.ed.PeerHalo)
    ph.group, ph.rank, ph.world = dist.group.WORLD, self.rank, self.world
    ph.halo, ph.sy, ph.sx = halo, plane[0], plane[1]
    ph.esz, ph.nbytes = 4, 256
    ph.buf, ph.hdl, ph._peers = _Mapped(_addr(self.rank)), _Handle(), {}
    ph.step = 0
    ph.status = torch.zeros(1, dtype=torch.int32)
    return ph

  def __call__(self, depth=10, plane=PLANE, dirty=(), status=None, info=True, check=False, group=None,
               known_depths=False, **kw):
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    vol = np.random.default_rng(7).integers(0, 4, (depth * world,) + tuple(plane)).astype(np.int32)
    local = torch.from_numpy(vol[rank * depth:(rank + 1) * depth].copy())
    log = []
    passes = ScriptedPasses(log, dirty, status)
    info = {} if info else None
    if known_depths:
      kw["depths"] = [depth] * world
    del self.collectives[:]
    rec = {"raised": None}
    try:
      self.ed.slab_transform(local, (3.0, 2.0, 1.0), False, group=group, passes=passes, info=info, **kw)
    except (ValueError, self.ed.EDTError) as exc:
      rec["raised"] = (type(exc).__name__, str(exc))
    rec.update(attempts=attempts(log, world), collectives=list(self.collectives), hint=sorted(self.ed._HALO_HINT.values()),
               steps=[arg for name, arg in log if name == "slab_step"])
    if info is not None:
      rec.update(method=info.get("method"), halo=info.get("halo"))
      if "verdict" in info:
        rec["deferred"] = "local" if info["verdict"][1] is None else "async"
        if check:
          try:
            rec["clean"] = self.ed.check_verdicts([info["verdict"]], group)
          except self.ed.EDTError as exc:
            rec["clean"] = ("EDTError", str(exc))
    return rec


def ladder(run, groups):
  return {
    "2-8": run(halo=2, dirty={2}),
    "2-thin": run(depth=5, halo=2, dirty={2}),
    "8-32": run(depth=40, halo=8, dirty={8}),
    "8-32-128-transpose": run(depth=130, halo=8, dirty={8, 32, 128}),
    "64-on-64": run(depth=64, halo=64),
    "254": run(depth=255, halo=254, dirty={254}),
    "transpose": run(halo=2, method="transpose"),
  }


def method_halo(run, groups):
  one = groups["single"]
  return {
    "clean": run(halo=2, method="halo"),
    "dirty": run(halo=2, method="halo", dirty={2}),
    "impossible": run(depth=2, halo=2, method="halo"),
    "world1": [run(group=one, method=m, dirty={8}) for m in ("auto", "halo", "transpose")],
    "world1-staging": run(group=one, method="halo", staging=True),
  }


def hint(run, groups):
  return {
    "escalate": run(depth=40, dirty={8}),
    "remembered": run(depth=40),
    "method-halo": run(depth=40, method="halo"),
    "explicit": run(depth=40, halo=8),
    "transposed": run(depth=40, dirty={32}),
    "other-plane-deferred": run(plane=(3, 2), defer_check=True),
    "other-plane-local": run(plane=(3, 2), defer_check="local", dirty={8}),
    "other-plane": run(plane=(3, 2)),
    "other-group": run(group=groups["all"]),
    "staging": run(staging=5),
    "after-staging": run(),
  }


def deferred(run, groups):
  out = {}
  for mode in (True, "local"):
    for staging in (None, 2):
      for dirty in (False, True):
        out[(mode, staging, dirty)] = run(halo=2, defer_check=mode, staging=staging, known_depths=True, check=True,
                                          dirty={2} if dirty else (), status={2: 1} if dirty else None)
    out[(mode, "no info")] = run(halo=2, defer_check=mode, info=False)
  return out


def fused(run, groups):
  out = {"steps": [run(staging="keep") for _ in range(2)]}
  out["mismatch"] = run(staging="keep", halo=8)
  out["step-after-mismatch"] = run.kept.step
  out["dirty"] = run(staging=2, status={2: 1})
  out["dirty-nccl-only"] = run(staging=None, halo=2, dirty={2})
  out["time-out"] = run(staging=5, status={5: 2})
  out["time-out-deferred"] = run(staging=5, status={5: 2}, defer_check="local", check=True)
  return out


SCENARIOS = {"ladder": ladder, "method_halo": method_halo, "hint": hint, "deferred": deferred, "fused": fused}


def _worker(rank, world, port, queue):
  sys.path.insert(0, ROOT)
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    import edt_b200.distributed as ed
    groups = {"single": [dist.new_group([r]) for r in range(world)][rank], "all": dist.new_group(list(range(world)))}
    caller = Caller(ed, rank, world)

    def run(staging="auto", **kw):
      """staging: "auto", None, True (a stand-in of the default halo), a halo (a new stand-in) or
      "keep" (the stand-in of halo 5 that the previous "keep" call used)."""
      if staging == "keep":
        run.kept = getattr(run, "kept", None) or caller.staging(5)
        staging = run.kept
      elif staging is True:
        staging = caller.staging(ed.DEFAULT_HALO)
      elif isinstance(staging, int):
        staging = caller.staging(staging)
      return caller(peer_halo=staging, **kw)

    results = {}
    for name, scenario in SCENARIOS.items():
      ed._HALO_HINT.clear()
      results[name] = scenario(run, groups)
    queue.put(("done", rank, results))
  except Exception:
    import traceback
    queue.put(("error", rank, traceback.format_exc()))
    raise
  finally:
    dist.destroy_process_group()


def _free_port():
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    return s.getsockname()[1]


@pytest.fixture(scope="module", params=[2, 3])
def traced(request):
  """(world, {rank: {scenario: records}}) from one gloo job of `world` ranks."""
  world = request.param
  ctx = mp.get_context("spawn")
  queue = ctx.Queue()
  port = _free_port()
  procs = [ctx.Process(target=_worker, args=(r, world, port, queue)) for r in range(world)]
  for p in procs:
    p.start()
  try:
    items = [queue.get(timeout=300) for _ in range(world)]
  finally:
    for p in procs:
      p.join(timeout=60)
      if p.is_alive():
        p.terminate()
  assert all(it[0] == "done" for it in items), [it for it in items if it[0] != "done"]
  return world, {it[1]: it[2] for it in items}


def _each_rank(traced, name):
  world, by_rank = traced
  return [(rank, by_rank[rank][name]) for rank in range(world)]


def test_attempt_ladder(traced):
  T, X = "transpose", "exchange"
  for _, r in _each_rank(traced, "ladder"):
    assert r["2-8"]["attempts"] == [(X, 2), (X, 8)] and (r["2-8"]["method"], r["2-8"]["halo"]) == ("halo", 8)
    # 8 would not fit into 5-row slabs
    assert r["2-thin"]["attempts"] == [(X, 2), (T, None)] and r["2-thin"]["method"] == T
    assert r["2-thin"]["halo"] is None
    assert r["8-32"]["attempts"] == [(X, 8), (X, 32)] and (r["8-32"]["method"], r["8-32"]["halo"]) == ("halo", 32)
    assert r["8-32-128-transpose"]["attempts"] == [(X, 8), (X, 32), (X, 128), (T, None)]
    assert r["8-32-128-transpose"]["method"] == T
    # a halo attempt needs slabs deeper than the halo
    assert r["64-on-64"]["attempts"] == [(T, None)] and r["64-on-64"]["method"] == T
    # 128 is not deeper than 254
    assert r["254"]["attempts"] == [(X, 254), (T, None)] and r["254"]["method"] == T
    assert r["transpose"]["attempts"] == [(T, None)] and r["transpose"]["method"] == T
    for rec in r.values():
      assert rec["raised"] is None and rec["hint"] == []        # an explicit halo leaves the hint alone


def test_method_halo_raises_or_runs_one_attempt(traced):
  for _, r in _each_rank(traced, "method_halo"):
    assert r["clean"]["attempts"] == [("exchange", 2)] and (r["clean"]["method"], r["clean"]["halo"]) == ("halo", 2)
    assert r["dirty"]["attempts"] == [("exchange", 2)]
    assert r["dirty"]["raised"][0] == "EDTError" and r["dirty"]["raised"][1].startswith("halo method is not exact here")
    assert r["impossible"]["raised"][0] == "EDTError"
    assert r["impossible"]["raised"][1].startswith("halo method needs more than one rank")
    assert all(t == "transpose" for t, _ in r["impossible"]["attempts"])       # no halo attempt
    assert r["impossible"]["collectives"] == [("all_reduce", False)]        # the slab depths only
    # a group of one computes its slab alone, whatever the method and staging
    for rec in r["world1"] + [r["world1-staging"]]:
      assert rec["raised"] is None and rec["method"] == "single" and rec["attempts"] == [("single", None)]
      assert rec["collectives"] == [("all_reduce", False)] and rec["steps"] == []


def test_halo_hint(traced):
  X, T = "exchange", "transpose"
  for _, r in _each_rank(traced, "hint"):
    # halo=None, "auto": starts at DEFAULT_HALO (8) and remembers the halo whose verdict read clean ...
    assert r["escalate"]["attempts"] == [(X, 8), (X, 32)] and r["escalate"]["hint"] == [32]
    # ... where the next such call on the same group and plane shape starts
    assert r["remembered"]["attempts"] == [(X, 32)] and r["remembered"]["hint"] == [32]
    # method="halo" and an explicit halo neither read nor update it
    assert r["method-halo"]["attempts"] == [(X, 8)] and r["method-halo"]["hint"] == [32]
    assert r["explicit"]["attempts"] == [(X, 8)] and r["explicit"]["hint"] == [32]
    # a call that ends in the transposition does not update it
    assert r["transposed"]["attempts"] == [(X, 32), (T, None)] and r["transposed"]["hint"] == [32]
    # another plane shape starts at DEFAULT_HALO; a deferred verdict is not remembered and not retried
    assert r["other-plane-deferred"]["attempts"] == [(X, 8)] and r["other-plane-deferred"]["hint"] == [32]
    assert r["other-plane-local"]["attempts"] == [(X, 8)] and r["other-plane-local"]["hint"] == [32]
    assert r["other-plane"]["attempts"] == [(X, 8)] and r["other-plane"]["hint"] == [8, 32]
    # so does another group
    assert r["other-group"]["attempts"] == [(X, 8)] and r["other-group"]["hint"] == [8, 8, 32]
    # an explicit PeerHalo sets the starting halo ahead of the hint, and a clean verdict is remembered
    assert r["staging"]["attempts"] == [("fused", 5)] and r["staging"]["hint"] == [5, 8, 8]
    assert r["after-staging"]["attempts"] == [(X, 5)]
    for rec in r.values():
      assert rec["raised"] is None


def test_deferred_verdicts(traced):
  for _, r in _each_rank(traced, "deferred"):
    for mode in (True, "local"):
      for staging in (None, 2):
        exchange = [("batch_isend_irecv", False)] if staging is None else []
        for dirty in (False, True):
          rec = r[(mode, staging, dirty)]
          assert rec["raised"] is None and rec["method"] == "halo" and rec["halo"] is None
          assert rec["attempts"] == [("exchange" if staging is None else "fused", 2)]      # no retry
          # True: ONE async all-reduce; "local": no collective at all (besides the NCCL path's exchange)
          assert rec["collectives"] == exchange + ([("all_reduce", True)] if mode is True else [])
          assert rec["deferred"] == ("async" if mode is True else "local")
          assert rec["clean"] is (not dirty)
      assert r[(mode, "no info")]["raised"][0] == "ValueError"


def test_fused_step_orchestration(traced):
  world = traced[0]
  for rank, r in _each_rank(traced, "fused"):
    first, second = r["steps"]
    for n, rec in enumerate((first, second), 1):
      assert rec["raised"] is None and rec["attempts"] == [("fused", 5)] and rec["method"] == "halo"
      assert rec["halo"] == 5 and rec["collectives"] == [("all_reduce", False), ("all_reduce", True)]
      (step,) = rec["steps"]
      assert step == dict(halo=5, w_xyz=(1.0, 2.0, 3.0), has_lo=rank > 0, has_hi=rank < world - 1,
                          sym_self=_addr(rank), sym_lo=_addr(rank - 1) if rank > 0 else 0,
                          sym_hi=_addr(rank + 1) if rank < world - 1 else 0, step=n)
    assert r["mismatch"]["raised"][0] == "ValueError" and r["mismatch"]["steps"] == []
    assert r["step-after-mismatch"] == 2
    # a dirty fused verdict is retried at the deeper halo with "auto" staging: None for CPU slabs
    assert r["dirty"]["attempts"] == [("fused", 2), ("exchange", 8)]
    assert (r["dirty"]["method"], r["dirty"]["halo"]) == ("halo", 8)
    assert r["dirty-nccl-only"]["attempts"] == [("exchange", 2), ("exchange", 8)]
    assert r["time-out"]["raised"][0] == "EDTError" and "never published its faces" in r["time-out"]["raised"][1]
    assert r["time-out"]["attempts"] == [("fused", 5)]
    assert r["time-out-deferred"]["clean"][0] == "EDTError"
