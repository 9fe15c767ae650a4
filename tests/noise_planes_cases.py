"""A plain restatement, numpy only, of what the plane-writing X pass (first_axis_planes_kernel) writes
on label noise, and of the planes after the Y pass that reads them: the words edtb200_noise_planes
must leave in f and in its planes buffer (include/edt_b200.h).

Labels come as (count, sz, sy, sx) in 3-D or (count, sy, sx) in 2-D, C order, x last.  Every volume
is a stack of slices here: (count * sz, sy, sx) in 3-D, (count, sy, sx) in 2-D, where every image is
a slice of depth 1 and has no z plane.  Rows are numbered slice * sy + y, as the planes are laid out.

  f            the oracle's X pass of each row, then min(f, ty) wherever the voxel's y-run is one row
               long and sy >= 2 (a line end counts as a run end; lines of one row never take it);
               ty = float32(w_y) * float32(w_y), tz likewise
  y plane      bit set iff y == 0 or L[y] != L[y - 1]
  z plane      bit set iff z % sz == 0 or L[z] != L[z - 1] (z within its own volume; 3-D only)
               padding bits past sx in a row's last word are 0
  settled_y    one word per row: bit s set iff every real voxel of x-segment s (32 voxels) has
               f <= ty; padding voxels count as settled, so the segments past sx and bits 16..31 are set
  settled_z    the same with tz (3-D only)

After the Y pass (passes = 2) f is the oracle's Y pass (its sqrt where that pass is the last one and
asked for it), the y plane and settled_y are unchanged, and -- where the Y pass refreshes settled_z --
every Y tile that ran (the x-segment s of one slice: it runs when some row of the slice has bit s of
settled_y clear) and found between 1 and 32 of its rows with bit s of settled_z clear sets each of
those bits iff all the segment's voxels are <= tz after the Y pass (refresh_settled); every other bit
keeps its value.
"""
import numpy as np

SEG = 32                      # voxels per x-segment: one settled bit
PAD_BITS = np.uint32(0xffff0000)
REFRESH_ROWS = 32             # refresh_settled re-reads at most this many rows of a tile


def slices(lab, ndim):
  """The labels as a stack of slices (n, sy, sx) and the depth of each volume (1 in 2-D)."""
  lab = np.ascontiguousarray(lab)
  if ndim == 3:
    return lab.reshape((-1,) + lab.shape[-2:]), lab.shape[-3]
  return lab.reshape((-1,) + lab.shape[-2:]), 1


def square(w):
  """The float32 product w * w that the passes compare with."""
  return np.float32(w) * np.float32(w)


def wpr(sx):
  return (sx + SEG - 1) // SEG


def one_row_runs(vol):
  """(n, sy, sx) bool: the voxel's y-run is one row long (the line ends count as run ends)."""
  sy = vol.shape[1]
  start = np.ones(vol.shape, bool)
  end = np.ones(vol.shape, bool)
  if sy > 1:
    start[:, 1:] = vol[:, 1:] != vol[:, :-1]
    end[:, :-1] = vol[:, :-1] != vol[:, 1:]
  return start & end


def x_pass(oracle, vol, wx, wy, border):
  """f after the plane-writing X pass, (n, sy, sx) float32."""
  f = oracle.pass_first(vol, wx, border)
  if vol.shape[1] >= 2:
    f = np.where(one_row_runs(vol), np.minimum(f, square(wy)), f).astype(np.float32)
  return f


def y_starts(vol):
  out = np.ones(vol.shape, bool)
  out[:, 1:] = vol[:, 1:] != vol[:, :-1]
  return out


def z_starts(vol, depth):
  out = np.ones(vol.shape, bool)
  out[1:] = vol[1:] != vol[:-1]
  out[::depth] = True
  return out


def pack_bits(bits):
  """(n, sy, sx) bool -> (n * sy, wpr) uint32 words, bit x % 32 of word x / 32, zeros past sx."""
  n, sy, sx = bits.shape
  padded = np.zeros((n * sy, wpr(sx) * SEG), bool)
  padded[:, :sx] = bits.reshape(n * sy, sx)
  return np.packbits(padded, axis=1, bitorder="little").view("<u4").astype(np.uint32)


def segments_settled(f, t):
  """(n * sy,) uint32: bit s set iff every voxel of segment s of the row has f <= t; segments past sx
  and bits 16..31 set."""
  n, sy, sx = f.shape
  rows = f.reshape(n * sy, sx)
  words = np.full(n * sy, 0xffffffff, np.uint32)
  for s in range(wpr(sx)):
    open_ = ~np.all(rows[:, s * SEG:(s + 1) * SEG] <= t, axis=1)
    words[open_] &= np.uint32(~(1 << s) & 0xffffffff)
  return words


def restate(oracle, lab, ndim, w, border):
  """What the X pass writes: dict f (n, sy, sx), y (rows, wpr), settled_y (rows,) and, in 3-D, z and
  settled_z."""
  vol, depth = slices(lab, ndim)
  f = x_pass(oracle, vol, w[0], w[1], border)
  out = {"f": f, "y": pack_bits(y_starts(vol)), "settled_y": segments_settled(f, square(w[1]))}
  if ndim == 3:
    out["z"] = pack_bits(z_starts(vol, depth))
    out["settled_z"] = segments_settled(f, square(w[2]))
  return out


def y_tiles_run(settled_y, n, sy, sx):
  """(n, wpr) bool: the Y tile of segment s of slice z runs (some row has bit s of settled_y clear)."""
  words = settled_y.reshape(n, sy)
  return np.stack([np.any((words >> np.uint32(s)) & 1 == 0, axis=1) for s in range(wpr(sx))], axis=1)


def refresh(settled_z, settled_y, f_after, tz):
  """settled_z after the Y pass's refresh (refresh_settled), from the X pass's planes and f after Y."""
  n, sy, sx = f_after.shape
  z = settled_z.reshape(n, sy).copy()
  ran = y_tiles_run(settled_y, n, sy, sx)
  for s in range(wpr(sx)):
    bit = np.uint32(1 << s)
    ok = np.all(f_after[:, :, s * SEG:(s + 1) * SEG] <= tz, axis=2)    # (n, sy)
    for c in np.nonzero(ran[:, s])[0]:
      clear = (z[c] & bit) == 0
      if 1 <= clear.sum() <= REFRESH_ROWS:
        z[c, clear & ok[c]] |= bit
  return z.reshape(-1)


def restate_after_y(oracle, lab, ndim, w, border, x, sqrt=False, refreshes=False):
  """What the Y pass leaves after the X pass x (restate): f, and the planes with settled_z refreshed
  where `refreshes`; sqrt: the Y pass is the last one and takes the root."""
  vol, _ = slices(lab, ndim)
  f = oracle.pass_later(vol, x["f"].copy(), 1, w[1], border, border)
  out = dict(x)
  out["f"] = np.sqrt(f) if sqrt else f
  if ndim == 3 and refreshes:
    out["settled_z"] = refresh(x["settled_z"], x["settled_y"], f, square(w[2]))
  return out


def layout(sx, sy, rows_total, ndim):
  """[(name, start, words)] of the planes buffer: [y plane | settled_y | z plane | settled_z]."""
  words = rows_total * wpr(sx)
  parts = [("y", 0, words), ("settled_y", words, rows_total)]
  if ndim == 3:
    at = words + rows_total
    parts += [("z", at, words), ("settled_z", at + words, rows_total)]
  return parts


def split(buf, sx, sy, rows_total, ndim):
  """The planes buffer (flat uint32) as the dict restate returns (without f)."""
  out = {}
  for name, start, n in layout(sx, sy, rows_total, ndim):
    part = buf[start:start + n]
    out[name] = part.reshape(rows_total, wpr(sx)) if name in ("y", "z") else part
  return out


def buffer_words(sx, sy, rows_total, ndim):
  return sum(n for _, _, n in layout(sx, sy, rows_total, ndim))


def runs_from_plane(words, n, sy, sx):
  """Labels rebuilt from a run-start plane along y: a new run id at every set bit, so that a later
  pass over them sees the same runs as over the labels."""
  bits = np.unpackbits(words.view(np.uint8), axis=1, bitorder="little")[:, :sx].astype(bool)
  bits = bits.reshape(n, sy, sx)
  return np.cumsum(bits, axis=1).astype(np.uint32) + 1


# ---- volumes ----

def noise(shape, dtype, rng, background=0.02):
  lab = rng.integers(1, 1 << 20, shape).astype(dtype)
  lab[rng.random(shape) < background] = 0
  return lab


def settled_pattern(shape, dtype, rng, kind):
  """Label noise along x with whole segments settled or not: kind "all" (every voxel has x- and y-runs
  of one: every segment settles for the Y pass), "none" (slices of a single label: f = +inf without a
  border and y-runs of sy rows, no segment settles), "some" (every other segment is one x-run over
  pairs of rows)."""
  lab = noise(shape, dtype, rng, background=0.0)
  sx = shape[-1]
  if kind == "none":
    lab[...] = lab[..., :1, :1]
  elif kind == "some":
    pairs = np.arange(shape[-2]) // 2 * 2
    for s in range(0, wpr(sx), 2):
      lab[..., s * SEG:(s + 1) * SEG] = lab[..., pairs, s * SEG:s * SEG + 1]
  return lab
