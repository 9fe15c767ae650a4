"""Multi-GPU transform: one process per GPU (torch.distributed), volume split into Z slabs.

Volumes too big (or too slow) for one GPU are split along the slowest axis into contiguous slabs,
one per rank (the reference has no distributed path at all, SURVEY.md section 2.3).

  * X and Y passes couple voxels of one z-slice only (reference src/edt.hpp:430-460 already
    parallelises them over z), so every rank runs them on its own slab with NO communication
    (`edtb200_pass_first`, `edtb200_pass_later(axis=1)`).
  * The Z pass couples slabs, but only through runs of equal labels that cross a slab face.
    Method "halo" (the fast path): every rank runs the Z pass on its own slab with the interior
    faces open, while ONE neighbour exchange ships, per face, the face plane of labels, the
    length of the face-touching run of every (x,y) line and the last/first `halo` planes of the
    Y-pass distances (34 MiB per face at 512 x 512, halo 32).  `edtb200_slab_face_fixup` then
    folds the neighbour's sites into the face-touching runs.  Exact when every face-crossing run
    ends within `halo` rows of the face on the far side, OR goes on but the distances at the
    face do not exceed the halo's reach (value <= (w_z * halo)^2: a site behind the halo is then
    too far away to win).  The fix-up kernel checks the second condition on the values it
    produces and raises a device flag (one int all-reduce after the step).  Method "auto" then
    retries with a four times deeper halo (8 -> 32 -> 128 rows) while every slab is deeper, else:
  * Method "transpose" (exact for any input): one all-to-all turns the Z-slab layout into a
    Y-slab layout (every rank then owns complete z-lines for a range of y), the ordinary Z-pass
    kernel runs with the volume's real border flags, and a second all-to-all brings the result
    back.  Per GPU and step it moves (4 + L) * N/G * (G-1)/G bytes forward and 4 * N/G * (G-1)/G
    back over NVLink (L = label bytes, N = voxels, G = ranks).

For the exchange to overlap with the Z-pass kernel (which fills every SM), create the process
group with a high-priority NCCL stream:
    opts = torch.distributed.ProcessGroupNCCL.Options(is_high_priority_stream=True)
    torch.distributed.init_process_group("nccl", pg_options=opts, ...)

Every rank issues the same collectives in the same order: a call's attempts follow from values all ranks
share (method, halo, slab depths, all-reduced verdicts).  Exchanges are grouped point-to-point operations
(`batch_isend_irecv`), which gloo also implements: the CPU tests run this code with the oracle as kernels.

Array convention: C-contiguous (z, y, x) tensors, x fastest, like `edt_cuda`; `anisotropy` is
given per array axis (w_z, w_y, w_x).
"""
import ctypes

import torch
import torch.distributed as dist

from . import FLAG_SIGNED, FLAG_SQRT, EDTError, _lib, _torch_label_bytes


def split_extent(total, parts):
  """Balanced contiguous split of range(total) into `parts`: list of (start, count)."""
  base, extra = divmod(int(total), int(parts))
  out, start = [], 0
  for r in range(parts):
    count = base + (1 if r < extra else 0)
    out.append((start, count))
    start += count
  return out


class CudaPasses:
  """Per-axis passes on torch CUDA tensors through the C ABI (asynchronous on the current stream)."""

  def __init__(self, device):
    self.device = torch.device(device)
    self.lib = _lib()

  def _stream(self):
    return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

  def _check(self, rc):
    if rc != 0:
      raise EDTError(self.lib.edtb200_last_error().decode("utf-8", "replace"))

  def empty_f32(self, shape):
    return torch.empty(shape, dtype=torch.float32, device=self.device)

  def pass_first(self, labels, f, wx, black_border, signed):
    sz, sy, sx = labels.shape
    nbytes = _torch_label_bytes(torch)[labels.dtype]
    self._check(self.lib.edtb200_pass_first(labels.data_ptr(), nbytes, sx, sy, sz, float(wx),
                                            int(bool(black_border)), FLAG_SIGNED if signed else 0,
                                            f.data_ptr(), self.device.index, self._stream()))

  def pass_later(self, labels, f, axis, w, border_lo, border_hi, sqrt=False, negate=False):
    sz, sy, sx = labels.shape
    nbytes = _torch_label_bytes(torch)[labels.dtype]
    flags = (FLAG_SQRT if sqrt else 0) | (FLAG_SIGNED if negate else 0)
    self._check(self.lib.edtb200_pass_later(labels.data_ptr(), nbytes, int(axis), sx, sy, sz, float(w),
                                            int(bool(border_lo)), int(bool(border_hi)), flags,
                                            f.data_ptr(), self.device.index, self._stream()))

  def slab_step(self, labels, f, w_xyz, black_border, has_lo, has_hi, sqrt, signed, halo, sym_self, sym_lo, sym_hi,
                step, status):
    """One fused slab step (edtb200_slab_step): X, Y, stage faces, Z, fix-up, on the current stream."""
    sz, sy, sx = labels.shape
    nbytes = _torch_label_bytes(torch)[labels.dtype]
    flags = (FLAG_SQRT if sqrt else 0) | (FLAG_SIGNED if signed else 0)
    self._check(self.lib.edtb200_slab_step(labels.data_ptr(), nbytes, sx, sy, sz, float(w_xyz[0]), float(w_xyz[1]),
                                           float(w_xyz[2]), int(bool(black_border)), int(bool(has_lo)),
                                           int(bool(has_hi)), flags, f.data_ptr(), int(halo),
                                           ctypes.c_void_p(sym_self), ctypes.c_void_p(sym_lo or None),
                                           ctypes.c_void_p(sym_hi or None), ctypes.c_uint64(step),
                                           status.data_ptr(), self.device.index, self._stream()))

  def repartition(self, src, dst, ysplit, unpack=False):
    """Z slab (zc, sy, row) <-> the exchange layout of the transposition fallback, ONE launch
    (csrc/edt_slab.cuh: slab_pack_kernel).  `src` / `dst` are contiguous tensors of equal byte size
    whose slab side has shape (zc, sy, row); ysplit = [(y_start, y_count)] per rank."""
    slab = dst if unpack else src
    zc, sy = slab.shape[0], slab.shape[1]
    row_bytes = slab.shape[2] * slab.element_size()
    starts = (ctypes.c_int64 * (len(ysplit) + 1))(*([s for s, _ in ysplit] + [sy]))
    self._check(self.lib.edtb200_slab_pack(src.data_ptr(), dst.data_ptr(), zc, sy, row_bytes, len(ysplit), starts,
                                           1 if unpack else 0, self.device.index, self._stream()))

  def face_runs(self, labels, high_face, halo, signed, overflow, out=None):
    """uint8 (sy, sx) run lengths at one face; raises the device int `overflow` when too long."""
    sz, sy, sx = labels.shape
    nbytes = _torch_label_bytes(torch)[labels.dtype]
    m = out if out is not None else torch.empty((sy, sx), dtype=torch.uint8, device=self.device)
    self._check(self.lib.edtb200_slab_face_runs(labels.data_ptr(), nbytes, sx, sy, sz, int(high_face), int(halo),
                                                FLAG_SIGNED if signed else 0, m.data_ptr(),
                                                overflow.data_ptr(), self.device.index, self._stream()))
    return m

  def face_fixup(self, labels, f, high_face, halo, wz, sqrt, signed, nb_label, nb_m, nb_f, inexact):
    """`inexact` (device int32[1]) is raised when a run continues behind the halo AND the distances
    at the face are larger than the halo reaches, i.e. an unseen site could still win."""
    sz, sy, sx = labels.shape
    nbytes = _torch_label_bytes(torch)[labels.dtype]
    flags = (FLAG_SQRT if sqrt else 0) | (FLAG_SIGNED if signed else 0)
    self._check(self.lib.edtb200_slab_face_fixup(labels.data_ptr(), nbytes, sx, sy, sz, int(high_face),
                                                 int(halo), float(wz), flags, nb_label.data_ptr(),
                                                 nb_m.data_ptr(), nb_f.data_ptr(), f.data_ptr(),
                                                 inexact.data_ptr(), self.device.index, self._stream()))


def _peer(group, r):
  return dist.get_global_rank(group, r) if group is not None else r


def _all_to_all(send_chunks, recv_chunks, group, peers=None):
  """Exchange send_chunks[j] -> rank j / recv_chunks[i] <- rank i (contiguous tensors; the own
  chunk is copied locally).  Empty chunks are skipped on both sides (sizes are symmetric).
  `peers` names the rank of every chunk pair when several arrays travel in one grouped exchange
  (every rank lists its chunks in the same order, so sends and receives match up pair by pair)."""
  rank = dist.get_rank(group)
  ops = []
  for peer, (s, r) in zip(peers if peers is not None else range(len(send_chunks)), zip(send_chunks, recv_chunks)):
    if peer == rank:
      r.copy_(s)
      continue
    gpeer = _peer(group, peer)
    if r.numel():
      ops.append(dist.P2POp(dist.irecv, r, gpeer, group))
    if s.numel():
      ops.append(dist.P2POp(dist.isend, s, gpeer, group))
  if ops:
    for req in dist.batch_isend_irecv(ops):
      req.wait()


class PeerHalo:
  """Face staging buffer in CUDA symmetric memory (torch.distributed._symmetric_memory) for the
  fused slab step `edtb200_slab_step` (csrc/edt_slab.cuh): every rank publishes, per step, its two
  face planes of labels, its face run lengths and its first / last `halo` planes of Y-pass
  distances in its own buffer, raises a flag word in each neighbour's buffer (a remote NVLink
  store), and the neighbours' fix-up kernel READS the staged faces in place over NVLink -- only
  the rows it actually needs (typically one or two planes).  Two staging sets alternate by step
  parity; the flag words order writers and readers across steps, no host call is involved.
  Creating one is a collective call over `group`; reuse it for every transform of the same
  (sy, sx, label width, halo)."""

  def __init__(self, device, sy, sx, label_dtype, halo=8, group=None):
    import torch.distributed._symmetric_memory as symm_mem
    self.group = group if group is not None else dist.group.WORLD
    self.rank = dist.get_rank(group)
    self.world = dist.get_world_size(group)
    self.halo, self.sy, self.sx = int(halo), int(sy), int(sx)
    self.esz = torch.empty((), dtype=label_dtype).element_size()
    lib = _lib()
    self.nbytes = int(lib.edtb200_slab_stage_bytes(self.sx, self.sy, self.esz, self.halo))
    if self.nbytes <= 0:
      raise ValueError("bad staging geometry")
    self.buf = symm_mem.empty(self.nbytes, dtype=torch.uint8, device=device)
    self.buf.zero_()                                   # flag words and the CTA counter start at 0
    torch.cuda.synchronize(device)
    self.hdl = symm_mem.rendezvous(self.buf, self.group)
    dist.barrier(group=self.group)                     # every rank's buffer is zeroed before any step
    self.step = 0
    self._peers = {}
    self.status = torch.zeros(1, dtype=torch.int32, device=device)

  def matches(self, sy, sx, label_dtype, halo):
    esz = torch.empty((), dtype=label_dtype).element_size()
    return (self.sy, self.sx, self.esz, self.halo) == (int(sy), int(sx), esz, int(halo))

  def peer_ptr(self, rank):
    """Device address of `rank`'s staging buffer as mapped into this process (0 if out of range)."""
    if rank < 0 or rank >= self.world:
      return 0
    if rank == self.rank:
      return self.buf.data_ptr()
    if rank not in self._peers:
      self._peers[rank] = self.hdl.get_buffer(rank, (self.nbytes,), torch.uint8, 0)
    return self._peers[rank].data_ptr()


def check_verdicts(verdicts, group=None):
  """True if every deferred halo verdict (info["verdict"] of slab_transform) is clean on every
  rank.  Verdicts deferred with defer_check="local" are still per-rank device flags: they are
  combined here with ONE all-reduce for the whole batch."""
  worst = 0
  local = [flag for flag, work in verdicts if work is None]
  for flag, work in verdicts:
    if work is not None:
      work.wait()
      worst = max(worst, int(flag.item()))
  if local:
    combined = torch.stack([f.reshape(()) for f in local]).max().reshape(1)
    dist.all_reduce(combined, op=dist.ReduceOp.MAX, group=group)
    worst = max(worst, int(combined.item()))
  if worst >= 2:
    raise EDTError("slab step: a neighbouring rank never published its faces (time-out in the fix-up kernel)")
  return worst == 0


def make_peer_halo(device, sy, sx, label_dtype, halo=8, group=None):
  """PeerHalo, or (None, reason) when symmetric memory is unavailable (then slab_transform uses
  the NCCL send/recv exchange).  Collective over `group`; returns (peer_halo, reason)."""
  try:
    return PeerHalo(device, sy, sx, label_dtype, halo, group), None
  except Exception as exc:            # e.g. no P2P access between the GPUs, or an older torch
    return None, "%s: %s" % (type(exc).__name__, exc)


_AUTO_PEER = {}


def _auto_peer_halo(labels_local, sy, sx, halo, group):
  """Cached PeerHalo for this configuration, or None (all ranks agree on which)."""
  if not labels_local.is_cuda:
    return None
  key = (id(group), labels_local.device.index, int(sy), int(sx), labels_local.element_size(), int(halo))
  if key not in _AUTO_PEER:
    ph, _ = make_peer_halo(labels_local.device, sy, sx, labels_local.dtype, halo, group)
    ok = torch.tensor([1 if ph is not None else 0], device=labels_local.device)
    dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
    _AUTO_PEER[key] = ph if int(ok.item()) == 1 else None
  return _AUTO_PEER[key]


_HALO_HINT = {}      # (group, plane shape) -> halo depth that was last needed there
DEFAULT_HALO = 8     # rows of the neighbours' distances staged per face; exact whenever the distances
                     # at the faces stay below 8 * w_z (the fix-up checks it; else see _halo_ladder)


def _halo_ladder(method, halo, min_depth, world):
  """Halos a call tries, in order, before the transposition (none on one rank): `halo`, then for "auto" four
  times deeper up to 128 rows while that is deeper; each only while every slab is deeper than it."""
  halos = []
  while method in ("auto", "halo") and world > 1 and min_depth > halo:
    halos.append(halo)
    deeper = min(4 * halo, 128)
    if method == "halo" or deeper <= halo:
      break
    halo = deeper
  return halos


def _attempt_staging(peer_halo, attempt, labels_local, halo, group):
  """PeerHalo of one halo attempt (the fused step), or None (the NCCL exchange).  A deeper retry takes
  the cached "auto" buffer of its own halo, unless the caller forced NCCL with None."""
  if attempt > 0 and peer_halo is not None:
    peer_halo = "auto"
  _, sy, sx = labels_local.shape
  if isinstance(peer_halo, str):
    return _auto_peer_halo(labels_local, sy, sx, halo, group) if peer_halo == "auto" else None
  if peer_halo is not None and not peer_halo.matches(sy, sx, labels_local.dtype, halo):
    raise ValueError("peer_halo was created for another plane shape / dtype / halo")
  return peer_halo


def _transpose_step(passes, labels_local, f, depths, wz, black_border, sqrt, signed, rank, world, group):
  """Z pass on the X/Y result `f`, exact for any input: Z slabs -> Y slabs (all-to-all), pass, back."""
  zc, sy, sx = labels_local.shape
  sz = sum(depths)
  ysplit = split_extent(sy, world)
  y0, yc = ysplit[rank]
  esz = labels_local.element_size()
  if zc:
    lab_bytes = labels_local.view(torch.uint8).reshape(zc, sy, sx * esz)
  else:
    lab_bytes = torch.empty((0, sy, sx * esz), dtype=torch.uint8, device=labels_local.device)

  f_cols = passes.empty_f32((sz, yc, sx))
  l_cols = torch.empty((sz, yc, sx * esz), dtype=torch.uint8, device=labels_local.device)
  zoff = [sum(depths[:i]) for i in range(world)]
  f_recv = [f_cols[zoff[i]:zoff[i] + depths[i]] for i in range(world)]
  l_recv = [l_cols[zoff[i]:zoff[i] + depths[i]] for i in range(world)]
  packed = hasattr(passes, "repartition") and world <= 64
  if packed:
    # one launch per array packs the slab into per-rank blocks; distances and labels travel in ONE
    # grouped exchange and land in place (contiguous z ranges of the column arrays)
    f_stage = passes.empty_f32((zc * sy * sx,))
    l_stage = torch.empty((zc * sy * sx * esz,), dtype=torch.uint8, device=labels_local.device)
    if zc:
      passes.repartition(f, f_stage, ysplit)
      passes.repartition(lab_bytes, l_stage, ysplit)
    f_send = [f_stage[zc * s * sx:zc * (s + c) * sx].view(zc, c, sx) for (s, c) in ysplit]
    l_send = [l_stage[zc * s * sx * esz:zc * (s + c) * sx * esz].view(zc, c, sx * esz) for (s, c) in ysplit]
    _all_to_all(f_send + l_send, f_recv + l_recv, group, peers=list(range(world)) * 2)
  else:
    f_send = [f[:, s:s + c, :].contiguous() for (s, c) in ysplit]
    l_send = [lab_bytes[:, s:s + c, :].contiguous() for (s, c) in ysplit]
    _all_to_all(f_send, f_recv, group)
    _all_to_all(l_send, l_recv, group)

  if yc and sz:
    labels_cols = l_cols.view(labels_local.dtype).reshape(sz, yc, sx)
    passes.pass_later(labels_cols, f_cols, 2, wz, black_border, black_border, sqrt=sqrt, negate=signed)

  out = passes.empty_f32((zc, sy, sx))
  back_send = [f_cols[zoff[i]:zoff[i] + depths[i]] for i in range(world)]          # contiguous z ranges
  if packed:
    back_recv = f_send                                       # the staging blocks are free again
    _all_to_all(back_send, back_recv, group)
    if zc:
      passes.repartition(f_stage, out, ysplit, unpack=True)
    return out
  back_recv = [passes.empty_f32((zc, c, sx)) for (_, c) in ysplit]
  _all_to_all(back_send, back_recv, group)
  for (s, c), chunk in zip(ysplit, back_recv):
    if c:
      out[:, s:s + c, :] = chunk
  return out


def slab_transform(labels_local, anisotropy=(1.0, 1.0, 1.0), black_border=False, *, sqrt=False,
                   signed=False, group=None, passes=None, halo=None, method="auto", info=None, depths=None,
                   peer_halo="auto", defer_check=False):
  """Distance transform of a volume distributed as Z slabs (axis 0) over the ranks of `group`.

  labels_local : this rank's slab, integer tensor (zc, sy, sx), C-contiguous; slabs are ordered by
                 rank and every rank passes the same sy, sx (zc may differ, 0 is allowed).
  Returns this rank's slab of the result (float32, same shape).  Semantics of edtsq (default),
  edt (sqrt=True), sdfsq (signed=True) and sdf (both) of the reference, on the WHOLE volume.
  method: "auto" (halo exchange; when its verdict says it was not exact for this volume the step
  is repeated with a four times deeper halo, up to 128 rows, then with transpose), "halo" (raise if
  not exact), "transpose".
  halo: rows of the neighbours' distances a rank can see (1..254).  None = an explicit PeerHalo's, else 8
  (DEFAULT_HALO) or the depth the last "auto" call on the same group and plane shape ended up needing.
  `info`, if a dict, receives {"method": ...}, and {"halo": ...} when a halo step was exact.
  depths: slab depth of every rank, if the caller knows them (saves one small all-reduce per call).
  peer_halo: a PeerHalo (symmetric-memory staging); the fix-up then reads the neighbours' faces
  directly over NVLink instead of receiving `halo` planes through NCCL send/recv.  "auto" (the
  default) creates and caches one per (group, plane shape, label width, halo) the first time CUDA
  slabs are transformed -- a collective step, so every rank must make the same first call -- and
  falls back to the NCCL exchange when symmetric memory is not available; None forces NCCL.
  defer_check: the halo method is taken optimistically and its exactness verdict (a device int
  raised by the fix-up kernels, all-reduced) is normally read at the end of the call, which costs
  one host synchronisation.  With defer_check=True the call returns without reading it and puts
  it in info["verdict"] (call `check_verdicts` on a batch of them later); a non-zero verdict means
  the result must be recomputed with a deeper halo or method="transpose".  defer_check="local"
  also skips the all-reduce: the call then contains no collective at all and `check_verdicts`
  combines the ranks' flags once for the whole batch.
  """
  world = dist.get_world_size(group)
  rank = dist.get_rank(group)
  if passes is None:
    passes = CudaPasses(labels_local.device)
  marks = info.get("marks") if isinstance(info, dict) else None      # optional CUDA-event phase marks

  def mark(name):
    if marks is not None:
      ev = torch.cuda.Event(enable_timing=True)
      ev.record()
      marks.append((name, ev))
  mark("start")
  if labels_local.dim() != 3:
    raise TypeError("slab_transform expects a 3-D (z, y, x) slab")
  labels_local = labels_local.contiguous()
  wz, wy, wx = (float(a) for a in anisotropy)
  zc, sy, sx = labels_local.shape

  # slab depths of every rank (needed for the exchange geometry)
  if depths is None:
    dt = torch.zeros(world, dtype=torch.int64, device=labels_local.device)
    dt[rank] = zc
    dist.all_reduce(dt, group=group)
    depths = [int(d) for d in dt.tolist()]
  else:
    depths = [int(d) for d in depths]
    if len(depths) != world or depths[rank] != zc:
      raise ValueError("depths must list the slab depth of every rank")

  hint_key = (id(group), (sy, sx))
  remember = halo is None and method == "auto"
  if halo is None and isinstance(peer_halo, PeerHalo):
    halo = peer_halo.halo                    # an explicit staging buffer fixes the depth
  elif halo is None:
    halo = _HALO_HINT.get(hint_key, DEFAULT_HALO) if remember else DEFAULT_HALO
  halos = _halo_ladder(method, halo, min(depths), world)
  if method == "halo" and world > 1 and not halos:
    raise EDTError("halo method needs more than one rank and slabs deeper than the halo (%d)" % halo)
  if info is None:
    if defer_check and halos:
      raise ValueError("defer_check needs an `info` dict to receive the verdict")
    info = {}

  def xy_passes():
    mark("face_runs")                        # end of the face-run phase (empty outside the NCCL exchange)
    f = passes.empty_f32((zc, sy, sx))
    if zc:
      passes.pass_first(labels_local, f, wx, black_border, signed)
      passes.pass_later(labels_local, f, 1, wy, black_border, black_border)
    mark("x+y passes")
    return f

  def halo_step(staging, halo, inexact):
    if staging is not None:                  # ONE C call: X, Y, publish faces, Z, fix-up (csrc/edt_slab.cuh)
      mark("face_runs")
      f = passes.empty_f32((zc, sy, sx))
      staging.step += 1
      passes.slab_step(labels_local, f, (wx, wy, wz), black_border, rank > 0, rank < world - 1, sqrt, signed, halo,
                       staging.peer_ptr(rank), staging.peer_ptr(rank - 1) if rank > 0 else 0,
                       staging.peer_ptr(rank + 1) if rank < world - 1 else 0, staging.step, inexact)
      mark("fused slab step")
      return f
    overflow = torch.zeros(1, dtype=torch.int32, device=labels_local.device)    # hint only, not reduced
    m_lo = passes.face_runs(labels_local, 0, halo, signed, overflow) if rank > 0 else None
    m_hi = passes.face_runs(labels_local, 1, halo, signed, overflow) if rank < world - 1 else None
    f = xy_passes()
    # ---- one neighbour exchange: face labels, face run lengths, `halo` planes of distances ----
    esz = labels_local.element_size()
    lab_bytes = labels_local.view(torch.uint8).reshape(zc, sy, sx * esz)
    ops, recv = [], {}
    for high_face, nb in ((0, rank - 1), (1, rank + 1)):
      if nb < 0 or nb >= world:
        continue
      face = zc - 1 if high_face else 0
      send_label = lab_bytes[face].contiguous()
      send_m = m_hi if high_face else m_lo
      send_f = (f[zc - halo:] if high_face else f[:halo]).clone()      # the Z pass overwrites f in place
      r_label = torch.empty_like(send_label)
      r_m = torch.empty_like(send_m)
      r_f = passes.empty_f32((halo, sy, sx))
      recv[high_face] = (r_label, r_m, r_f)
      peer = _peer(group, nb)
      for t in (send_label, send_m, send_f):
        ops.append(dist.P2POp(dist.isend, t, peer, group))
      for t in (r_label, r_m, r_f):
        ops.append(dist.P2POp(dist.irecv, t, peer, group))
    reqs = dist.batch_isend_irecv(ops) if ops else []
    mark("halo clone + exchange posted")
    # ---- Z pass on the slab, interior faces open; overlaps with the exchange ----
    passes.pass_later(labels_local, f, 2, wz, black_border and rank == 0, black_border and rank == world - 1,
                      sqrt=sqrt, negate=signed)
    mark("z pass")
    for req in reqs:
      req.wait()
    mark("exchange done")
    for high_face, (r_label, r_m, r_f) in recv.items():
      nb_label = r_label.view(labels_local.dtype).reshape(sy, sx)
      passes.face_fixup(labels_local, f, high_face, halo, wz, sqrt, signed, nb_label, r_m, r_f, inexact)
    mark("face fix-up")
    return f

  # ---- the halo method is taken optimistically; its verdict comes from the fix-up kernels ----
  for attempt, halo in enumerate(halos):
    staging = _attempt_staging(peer_halo, attempt, labels_local, halo, group)
    inexact = torch.zeros(1, dtype=torch.int32, device=labels_local.device)
    info["method"] = "halo"
    f = halo_step(staging, halo, inexact)
    if defer_check == "local":                 # no collective at all in this call
      info["verdict"] = (inexact, None)
      return f
    work = dist.all_reduce(inexact, op=dist.ReduceOp.MAX, group=group, async_op=True)
    if defer_check:
      info["verdict"] = (inexact, work)
      return f
    if check_verdicts([(inexact, work)], group):
      info["halo"] = halo
      if remember:
        _HALO_HINT[hint_key] = halo
      return f
    if method == "halo":
      raise EDTError("halo method is not exact here: a run goes on behind the %d halo rows of a neighbouring "
                     "slab and the distances at that face exceed the halo's reach" % halo)

  info["method"] = "transpose" if world > 1 else "single"
  f = xy_passes()
  if world > 1:
    return _transpose_step(passes, labels_local, f, depths, wz, black_border, sqrt, signed, rank, world, group)
  if zc:
    passes.pass_later(labels_local, f, 2, wz, black_border, black_border, sqrt=sqrt, negate=signed)
  return f
