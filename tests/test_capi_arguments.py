"""CPU tests: the argument checks of every C-ABI entry point that takes arguments.

Every entry point rejects a bad argument with a return code and a message before it touches a
device, so these checks run on any machine.  For each entry point the table below gives its
argument checks, the order of those checks where one call can fail two of them, and a fully
valid call, which must get past every check and stop at the device probe (abi_checks.expect_probe).
Nothing here launches a kernel or copies a byte.
"""
import ctypes

import numpy as np
import pytest

from abi_checks import BIG, EINVAL, ELIMIT, LABELS_FLOAT, LABELS_ON_DEVICE, OUT_ON_DEVICE, PROBE, SIGNED, check_case

_HOST = np.zeros(64, np.uint64)    # stands in for every data pointer: the checks only test for NULL
P = _HOST.ctypes.data


def ptrs(*values):
  return (ctypes.c_void_p * len(values))(*values)


def _transform(labels=P, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, w=(1.0, 1.0, 1.0), border=0, flags=0, out=P,
               device=63, stream=None):
  return (labels, label_bytes, ndim, sx, sy, sz, *w, border, flags, out, device, stream)


def _feature(labels=P, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, w=(1.0, 1.0, 1.0), border=0, flags=0, dist=None,
             idx=None, device=63, stream=None):
  idx = ptrs(P, P, P) if idx is None else idx
  return (labels, label_bytes, ndim, sx, sy, sz, *w, border, flags, dist, idx, device, stream)


def _voxel_graph(labels=P, label_bytes=4, graph=P, ndim=3, sx=4, sy=4, sz=4, w=(1.0, 1.0, 1.0), border=0, flags=0,
                 out=P, device=63, stream=None):
  return (labels, label_bytes, graph, ndim, sx, sy, sz, *w, border, flags, out, device, stream)


def _batch(labels=None, outs=None, count=2, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, w=(1.0, 1.0, 1.0), border=0,
           flags=0, device=63):
  labels = ptrs(P, P) if labels is None else labels
  outs = ptrs(P, P) if outs is None else outs
  return (labels, outs, count, label_bytes, ndim, sx, sy, sz, *w, border, flags, device)


def _multi(labels=P, label_bytes=4, ndim=3, sx=4, sy=4, sz=4, w=(1.0, 1.0, 1.0), border=0, flags=0, out=P,
           devices=(63,), ndevices=None, device=63):
  """`device` takes the place of device 63 in the list."""
  if devices is not None:
    devices = tuple(device if d == 63 else d for d in devices)
  arr = (ctypes.c_int * len(devices))(*devices) if devices is not None else None
  n = len(devices) if ndevices is None else ndevices
  return (labels, label_bytes, ndim, sx, sy, sz, *w, border, flags, out, arr, n)


def _pass_first(labels=P, label_bytes=4, sx=4, sy=4, sz=4, wx=1.0, border=0, flags=0, f=P, device=63, stream=None):
  return (labels, label_bytes, sx, sy, sz, wx, border, flags, f, device, stream)


def _pass_later(labels=P, label_bytes=4, axis=1, sx=4, sy=4, sz=4, w=1.0, lo=0, hi=0, flags=0, f=P, device=63,
                stream=None):
  return (labels, label_bytes, axis, sx, sy, sz, w, lo, hi, flags, f, device, stream)


_FIN, _FOUT, _CODES = (np.zeros(64, np.float32) for _ in range(3))   # three disjoint buffers
FIN, FOUT, CODES = _FIN.ctypes.data, _FOUT.ctypes.data, _CODES.ctypes.data


def _pass_window(labels=P, label_bytes=4, axis=1, sx=4, sy=4, sz=4, w=1.0, lo=0, hi=0, flags=0, d=3.0, fin=FIN,
                 fout=FOUT, codes=None, device=63, stream=None):
  return (labels, label_bytes, axis, sx, sy, sz, w, lo, hi, flags, d, fin, fout, codes, device, stream)


_ALIGNED = np.zeros(32, np.uint64)
PA = (_ALIGNED.ctypes.data + 63) // 64 * 64          # aligned for vector access by every label width


def _noise_planes(labels=PA, label_bytes=4, ndim=3, sx=64, sy=8, sz=8, count=1, w=(1.0, 1.0, 1.0), border=0,
                  flags=0, passes=1, nchunks=0, ctas=0, f=PA, planes=PA, info=P, device=63, stream=None):
  return (labels, label_bytes, ndim, sx, sy, sz, count, *w, border, flags, passes, nchunks, ctas, f, planes, info,
          device, stream)


def _face_runs(labels=P, label_bytes=4, sx=4, sy=4, sz=4, high_face=0, halo=2, flags=0, m=P, overflow=P, device=63,
               stream=None):
  return (labels, label_bytes, sx, sy, sz, high_face, halo, flags, m, overflow, device, stream)


def _face_fixup(labels=P, label_bytes=4, sx=4, sy=4, sz=4, high_face=0, halo=2, wz=1.0, flags=0, nb_label=P,
                nb_m=P, nb_f=P, f=P, inexact=None, device=63, stream=None):
  return (labels, label_bytes, sx, sy, sz, high_face, halo, wz, flags, nb_label, nb_m, nb_f, f, inexact, device,
          stream)


def _slab_pack(src=P, dst=P, zc=2, sy=4, row_bytes=16, parts=2, y_start=(0, 2, 4), unpack=0, device=63, stream=None):
  starts = (ctypes.c_int64 * len(y_start))(*y_start) if y_start is not None else None
  return (src, dst, zc, sy, row_bytes, parts, starts, unpack, device, stream)


def _slab_step(labels=P, label_bytes=4, sx=4, sy=4, sz=8, w=(1.0, 1.0, 1.0), border=0, has_lo=1, has_hi=1, flags=0,
               f=P, halo=2, sym_self=P, sym_lo=P, sym_hi=P, step=1, status=P, device=63, stream=None):
  return (labels, label_bytes, sx, sy, sz, *w, border, has_lo, has_hi, flags, f, halo, sym_self, sym_lo, sym_hi,
          step, status, device, stream)


def _label_stats(labels=P, label_bytes=4, dt=P, sx=4, sy=4, sz=4, capacity=64, keys=P, count=P, mx=P, argmax=P,
                 box=P, overflow=P, device=63, stream=None):
  return (labels, label_bytes, dt, sx, sy, sz, capacity, keys, count, mx, argmax, box, overflow, device, stream)


def _label_extract(labels=P, label_bytes=4, dt=P, sx=4, sy=4, sz=4, key=1, box=None, erase=0, out=P, device=63,
                   stream=None):
  cbox = (ctypes.c_int * 6)(*box) if box is not None else None
  return (labels, label_bytes, dt, sx, sy, sz, key, cbox, erase, out, device, stream)


# entry point -> (argument builder, [(case name, overrides, expected rc or PROBE, message substring)])
CASES = {
  "edtb200_transform": (_transform, [
    ("label_bytes", dict(label_bytes=3), EINVAL, "label_bytes"),
    ("ndim", dict(ndim=4), EINVAL, "ndim"),
    ("ndim_zero", dict(ndim=0), EINVAL, "ndim"),
    ("negative_size", dict(sy=-1), EINVAL, "negative size"),
    ("axis_too_long", dict(sz=BIG), ELIMIT, "axis longer than 2^30"),
    ("null_labels", dict(labels=None), EINVAL, "null pointer"),
    ("null_out", dict(out=None), EINVAL, "null pointer"),
    # order: the label width is checked before the pointers, emptiness before the pointers
    ("label_bytes_before_null", dict(label_bytes=3, labels=None, out=None), EINVAL, "label_bytes"),
    ("empty_before_null", dict(sx=0, labels=None, out=None), 0, ""),
    ("negative_before_empty", dict(sx=0, sy=-1), EINVAL, "negative size"),
    # the extents of missing axes are not read
    ("ndim1_ignores_sy_sz", dict(ndim=1, sy=-1, sz=BIG), PROBE, ""),
    ("ndim2_ignores_sz", dict(ndim=2, sz=-1), PROBE, ""),
    ("valid", dict(), PROBE, ""),
    ("valid_on_device", dict(flags=LABELS_ON_DEVICE | OUT_ON_DEVICE), PROBE, ""),
    ("valid_mixed", dict(flags=LABELS_ON_DEVICE), PROBE, ""),
  ]),
  "edtb200_feature_transform": (_feature, [
    ("label_bytes", dict(label_bytes=3), EINVAL, "label_bytes"),
    ("ndim", dict(ndim=4), EINVAL, "ndim"),
    ("negative_size", dict(sx=-4), EINVAL, "negative size"),
    ("axis_too_long", dict(ndim=1, sx=BIG), ELIMIT, "axis longer than 2^30"),
    ("null_labels", dict(labels=None), EINVAL, "null pointer"),
    ("null_planes", dict(idx=0), EINVAL, "null pointer"),
    ("null_plane_0", dict(idx=ptrs(None, P, P)), EINVAL, "null index plane 0"),
    ("null_plane_2", dict(idx=ptrs(P, P, None)), EINVAL, "null index plane 2"),
    ("empty_before_null", dict(sz=0, labels=None), 0, ""),
    ("label_bytes_before_null", dict(label_bytes=5, labels=None), EINVAL, "label_bytes"),
    # planes beyond ndim are not read; the distances are optional
    ("ndim2_ignores_plane_2", dict(ndim=2, idx=ptrs(P, P, None)), PROBE, ""),
    ("ndim1_ignores_planes_1_2", dict(ndim=1, idx=ptrs(P, None, None)), PROBE, ""),
    ("valid", dict(), PROBE, ""),
    ("valid_with_distances", dict(dist=P), PROBE, ""),
    ("valid_on_device", dict(flags=LABELS_ON_DEVICE | OUT_ON_DEVICE, dist=P), PROBE, ""),
  ]),
  "edtb200_transform_voxel_graph": (_voxel_graph, [
    ("ndim_1", dict(ndim=1), EINVAL, "2-D or 3-D"),
    ("ndim_4", dict(ndim=4), EINVAL, "2-D or 3-D"),
    ("signed", dict(flags=SIGNED), EINVAL, "EDTB200_SIGNED"),
    ("float_labels_width", dict(flags=LABELS_FLOAT, label_bytes=2), EINVAL, "EDTB200_LABELS_FLOAT"),
    ("label_bytes", dict(label_bytes=3), EINVAL, "label_bytes"),
    ("negative_size", dict(sz=-1), EINVAL, "negative size"),
    ("axis_too_long", dict(sx=BIG), ELIMIT, "axis longer than 2^30"),
    ("null_labels", dict(labels=None), EINVAL, "null pointer"),
    ("null_graph", dict(graph=None), EINVAL, "null pointer"),
    ("null_out", dict(out=None), EINVAL, "null pointer"),
    ("doubled_axis_too_long", dict(sx=(1 << 29) + 1, sy=1, sz=1), ELIMIT, "axis longer than 2^30"),
    # order: dimensionality, then sign, then float labels, then the label width
    ("ndim_before_signed", dict(ndim=1, flags=SIGNED), EINVAL, "2-D or 3-D"),
    ("signed_before_float", dict(flags=SIGNED | LABELS_FLOAT, label_bytes=1), EINVAL, "EDTB200_SIGNED"),
    ("float_before_label_bytes", dict(flags=LABELS_FLOAT, label_bytes=3), EINVAL, "EDTB200_LABELS_FLOAT"),
    ("empty_before_null", dict(sy=0, labels=None, graph=None, out=None), 0, ""),
    ("null_before_doubled", dict(sx=(1 << 29) + 1, sy=1, sz=1, graph=None), EINVAL, "null pointer"),
    ("valid", dict(), PROBE, ""),
    ("valid_2d_float", dict(ndim=2, sz=-1, flags=LABELS_FLOAT, label_bytes=8), PROBE, ""),
    ("valid_on_device", dict(flags=LABELS_ON_DEVICE | OUT_ON_DEVICE), PROBE, ""),
  ]),
  "edtb200_transform_batch": (_batch, [
    ("negative_count", dict(count=-1), EINVAL, "negative count"),
    ("labels_on_device", dict(flags=LABELS_ON_DEVICE), EINVAL, "HOST buffers"),
    ("out_on_device", dict(flags=OUT_ON_DEVICE), EINVAL, "HOST buffers"),
    ("label_bytes", dict(label_bytes=3), EINVAL, "label_bytes"),
    ("axis_too_long", dict(sy=BIG), ELIMIT, "axis longer than 2^30"),
    ("null_labels", dict(labels=0), EINVAL, "null pointer"),
    ("null_outs", dict(outs=0), EINVAL, "null pointer"),
    ("null_in_volume_1", dict(outs=ptrs(P, None)), EINVAL, "null pointer in volume 1"),
    ("negative_count_first", dict(count=-1, flags=OUT_ON_DEVICE, label_bytes=3), EINVAL, "negative count"),
    ("flags_before_label_bytes", dict(flags=OUT_ON_DEVICE, label_bytes=3), EINVAL, "HOST buffers"),
    ("no_volumes", dict(count=0, labels=0, outs=0), 0, ""),
    ("empty_before_null", dict(sx=0, labels=0), 0, ""),
    ("valid", dict(), PROBE, ""),
  ]),
  "edtb200_transform_multi": (_multi, [
    ("no_devices", dict(devices=None, ndevices=1), EINVAL, "no devices given"),
    ("zero_devices", dict(ndevices=0), EINVAL, "no devices given"),
    ("on_device", dict(flags=LABELS_ON_DEVICE), EINVAL, "HOST volume"),
    ("label_bytes", dict(label_bytes=3), EINVAL, "label_bytes"),
    ("negative_size", dict(sz=-2), EINVAL, "negative size"),
    ("null_out", dict(out=None), EINVAL, "null pointer"),
    ("listed_twice", dict(devices=(63, 62, 63)), EINVAL, "device 63 listed twice"),
    ("devices_first", dict(devices=None, ndevices=1, flags=LABELS_ON_DEVICE), EINVAL, "no devices given"),
    ("empty_before_null", dict(sx=0, labels=None), 0, ""),
    ("null_before_twice", dict(out=None, devices=(63, 63)), EINVAL, "null pointer"),
    ("valid", dict(), PROBE, ""),
    ("valid_two_devices", dict(devices=(63, 62)), PROBE, ""),
  ]),
  "edtb200_pass_first": (_pass_first, [
    ("label_bytes", dict(label_bytes=0), EINVAL, "label_bytes"),
    ("negative_size", dict(sz=-1), EINVAL, "negative size"),
    ("axis_too_long", dict(sz=BIG), ELIMIT, "axis longer than 2^30"),
    ("null_labels", dict(labels=None), EINVAL, "null pointer"),
    ("null_f", dict(f=None), EINVAL, "null pointer"),
    ("empty_before_null", dict(sz=0, labels=None, f=None), 0, ""),
    ("valid", dict(), PROBE, ""),
  ]),
  "edtb200_pass_later": (_pass_later, [
    ("label_bytes", dict(label_bytes=16), EINVAL, "label_bytes"),
    ("negative_size", dict(sx=-1), EINVAL, "negative size"),
    ("axis_0", dict(axis=0), EINVAL, "axis must be 1 (Y) or 2 (Z)"),
    ("axis_3", dict(axis=3), EINVAL, "axis must be 1 (Y) or 2 (Z)"),
    ("null_labels", dict(labels=None), EINVAL, "null pointer"),
    ("null_f", dict(f=None), EINVAL, "null pointer"),
    ("label_bytes_before_axis", dict(label_bytes=3, axis=0), EINVAL, "label_bytes"),
    ("axis_before_empty", dict(axis=0, sy=0), EINVAL, "axis must be"),
    ("empty_before_null", dict(sy=0, f=None), 0, ""),
    ("valid_y", dict(), PROBE, ""),
    ("valid_z", dict(axis=2), PROBE, ""),
  ]),
  "edtb200_pass_window": (_pass_window, [
    ("label_bytes", dict(label_bytes=3), EINVAL, "label_bytes"),
    ("negative_size", dict(sz=-1), EINVAL, "negative size"),
    ("axis_too_long", dict(sy=BIG), ELIMIT, "axis longer than 2^30"),
    ("axis_0", dict(axis=0), EINVAL, "axis must be 1 (Y) or 2 (Z)"),
    ("weight_0", dict(w=0.0), EINVAL, "weight"),
    ("weight_nan", dict(w=float("nan")), EINVAL, "weight"),
    ("weight_inf", dict(w=float("inf")), EINVAL, "weight"),
    ("negative_distance", dict(d=-1.0), EINVAL, "max_distance"),
    ("nan_distance", dict(d=float("nan")), EINVAL, "max_distance"),
    ("no_bound", dict(d=float("inf")), EINVAL, "window radius 4611686018427387904 out of range"),
    ("radius_129", dict(d=129.0), EINVAL, "window radius 129 out of range"),
    ("radius_129_weight", dict(w=0.5, d=64.5), EINVAL, "window radius 129 out of range"),
    ("null_labels", dict(labels=None), EINVAL, "null pointer"),
    ("null_fin", dict(fin=None), EINVAL, "null pointer"),
    ("null_fout", dict(fout=None), EINVAL, "null pointer"),
    ("in_place", dict(fout=FIN), EINVAL, "must not overlap"),
    ("fout_inside_fin", dict(fout=FIN + 16), EINVAL, "must not overlap"),
    ("codes_on_fin", dict(codes=FIN + 60), EINVAL, "must not overlap"),
    ("codes_on_fout", dict(codes=FOUT), EINVAL, "must not overlap"),
    # order: label width, sizes, axis, weight, distance, radius, emptiness, pointers, overlap
    ("label_bytes_before_axis", dict(label_bytes=5, axis=3), EINVAL, "label_bytes"),
    ("size_before_axis", dict(sx=-1, axis=0), EINVAL, "negative size"),
    ("axis_before_weight", dict(axis=0, w=0.0), EINVAL, "axis must be"),
    ("weight_before_distance", dict(w=-1.0, d=-1.0), EINVAL, "weight"),
    ("distance_before_empty", dict(d=-1.0, sx=0), EINVAL, "max_distance"),
    ("radius_before_empty", dict(d=200.0, sx=0), EINVAL, "window radius 200 out of range"),
    ("empty_before_null", dict(sy=0, labels=None, fin=None), 0, ""),
    ("null_before_overlap", dict(labels=None, fout=FIN), EINVAL, "null pointer"),
    ("valid", dict(), PROBE, ""),
    ("valid_radius_0", dict(d=0.0), PROBE, ""),
    ("valid_radius_128", dict(d=128.0, axis=2, flags=3), PROBE, ""),
    ("valid_radius_128_weight", dict(w=0.5, d=64.0), PROBE, ""),
    ("valid_with_codes", dict(codes=CODES, lo=1, hi=1), PROBE, ""),
  ]),
  "edtb200_noise_planes": (_noise_planes, [
    ("label_bytes", dict(label_bytes=3), EINVAL, "label_bytes"),
    ("label_bytes_1", dict(label_bytes=1), EINVAL, "labels of 4 or 8 bytes"),
    ("label_bytes_2", dict(label_bytes=2), EINVAL, "labels of 4 or 8 bytes"),
    ("ndim_1", dict(ndim=1), EINVAL, "2-D or 3-D"),
    ("axis_too_long", dict(sz=BIG), ELIMIT, "axis longer than 2^30"),
    ("count_0", dict(count=0), EINVAL, "count must be 1 or more"),
    ("weight_0", dict(w=(1.0, 0.0, 1.0)), EINVAL, "weight"),
    ("weight_nan", dict(w=(1.0, 1.0, float("nan"))), EINVAL, "weight"),
    ("signed", dict(flags=SIGNED), EINVAL, "EDTB200_SIGNED"),
    ("signed_sqrt", dict(flags=SIGNED | 1), EINVAL, "EDTB200_SIGNED"),
    ("other_flag", dict(flags=LABELS_ON_DEVICE), EINVAL, "flags may only hold EDTB200_SQRT"),
    ("passes_0", dict(passes=0), EINVAL, "passes must be 1 or 2"),
    ("passes_3", dict(passes=3), EINVAL, "passes must be 1 or 2"),
    ("sx_516", dict(sx=516), EINVAL, "rows of at most 512 voxels"),
    ("sx_6", dict(sx=6), EINVAL, "a multiple of 4"),
    ("slices_beyond_32_bits", dict(sz=1 << 30, count=2), EINVAL, "counts in 32 bits"),
    ("rows_beyond_32_bits", dict(sy=1 << 30), EINVAL, "counts in 32 bits"),
    ("nchunks_negative", dict(nchunks=-1), EINVAL, "nchunks must be 0 or 1..sy = 8"),
    ("nchunks_above_sy", dict(nchunks=9), EINVAL, "nchunks must be 0 or 1..sy = 8"),
    ("ctas_negative", dict(nchunks=2, ctas=-1), EINVAL, "ctas must be 0"),
    ("ctas_without_nchunks", dict(ctas=1), EINVAL, "with nchunks given"),
    ("ctas_above_items", dict(nchunks=2, ctas=3), EINVAL, "ctas must be 0 or 1..items = 2"),
    ("ctas_above_items_3d_stack", dict(sz=3, count=3, nchunks=2, ctas=5), EINVAL, "1..items = 4"),
    ("ctas_above_items_2d", dict(ndim=2, count=20, nchunks=1, ctas=4), EINVAL, "1..items = 3"),
    ("null_labels", dict(labels=None), EINVAL, "null pointer"),
    ("null_f", dict(f=None), EINVAL, "null pointer"),
    ("null_planes", dict(planes=None), EINVAL, "null pointer"),
    ("null_info", dict(info=None), EINVAL, "null pointer"),
    ("labels_misaligned", dict(labels=PA + 4), EINVAL, "aligned for vector access"),
    ("labels_misaligned_8", dict(labels=PA + 16, label_bytes=8), EINVAL, "aligned for vector access"),
    ("f_misaligned", dict(f=PA + 4), EINVAL, "aligned for vector access"),
    ("planes_misaligned", dict(planes=PA + 2), EINVAL, "aligned for vector access"),
    # order: label width and sizes, label width >= 4, ndim, count, weights, flags, passes, sx, counters,
    # nchunks, ctas, emptiness, pointers, alignment
    ("label_bytes_before_ndim", dict(label_bytes=2, ndim=1), EINVAL, "labels of 4 or 8 bytes"),
    ("ndim_before_count", dict(ndim=1, count=0), EINVAL, "2-D or 3-D"),
    ("count_before_weight", dict(count=0, w=(0.0, 1.0, 1.0)), EINVAL, "count"),
    ("weight_before_flags", dict(w=(0.0, 1.0, 1.0), flags=SIGNED), EINVAL, "weight"),
    ("flags_before_passes", dict(flags=SIGNED, passes=0), EINVAL, "EDTB200_SIGNED"),
    ("passes_before_sx", dict(passes=0, sx=6), EINVAL, "passes"),
    ("sx_before_nchunks", dict(sx=516, nchunks=-1), EINVAL, "rows of at most 512 voxels"),
    ("nchunks_before_ctas", dict(nchunks=9, ctas=1), EINVAL, "nchunks"),
    ("ctas_before_empty", dict(nchunks=1, ctas=2, sx=0), EINVAL, "ctas"),
    ("empty_before_null", dict(sx=0, labels=None, info=None), 0, ""),
    ("null_before_alignment", dict(labels=None, f=PA + 4), EINVAL, "null pointer"),
    # the weight of a missing axis is not read
    ("valid", dict(), PROBE, ""),
    ("valid_2d", dict(ndim=2, sz=-1, w=(1.0, 1.0, 0.0), count=20, nchunks=1, ctas=3), PROBE, ""),
    ("valid_overrides", dict(nchunks=8, ctas=8, passes=2, flags=1, border=1), PROBE, ""),
    ("valid_8_bytes", dict(label_bytes=8, sx=512, count=5), PROBE, ""),
  ]),
  "edtb200_slab_face_runs": (_face_runs, [
    ("label_bytes", dict(label_bytes=3), EINVAL, "label_bytes"),
    ("axis_too_long", dict(sy=BIG), ELIMIT, "axis longer than 2^30"),
    ("halo_0", dict(halo=0), EINVAL, "halo must be in 1..254"),
    ("halo_255", dict(halo=255), EINVAL, "halo must be in 1..254"),
    ("null_labels", dict(labels=None), EINVAL, "null pointer"),
    ("null_m", dict(m=None), EINVAL, "null pointer"),
    ("null_overflow", dict(overflow=None), EINVAL, "null pointer"),
    ("halo_before_empty", dict(halo=0, sz=0), EINVAL, "halo"),
    ("empty_before_null", dict(sz=0, m=None), 0, ""),
    ("valid", dict(), PROBE, ""),
  ]),
  "edtb200_slab_face_fixup": (_face_fixup, [
    ("label_bytes", dict(label_bytes=3), EINVAL, "label_bytes"),
    ("negative_size", dict(sz=-1), EINVAL, "negative size"),
    ("halo_0", dict(halo=0), EINVAL, "halo must be in 1..254"),
    ("null_labels", dict(labels=None), EINVAL, "null pointer"),
    ("null_nb_label", dict(nb_label=None), EINVAL, "null pointer"),
    ("null_nb_m", dict(nb_m=None), EINVAL, "null pointer"),
    ("null_nb_f", dict(nb_f=None), EINVAL, "null pointer"),
    ("null_f", dict(f=None), EINVAL, "null pointer"),
    ("halo_before_empty", dict(halo=300, sx=0), EINVAL, "halo"),
    ("empty_before_null", dict(sx=0, f=None), 0, ""),
    ("valid", dict(), PROBE, ""),
    ("valid_with_inexact", dict(inexact=P), PROBE, ""),
  ]),
  "edtb200_slab_pack": (_slab_pack, [
    ("negative_zc", dict(zc=-1), EINVAL, "negative extent"),
    ("negative_row", dict(row_bytes=-16), EINVAL, "negative extent"),
    ("parts_0", dict(parts=0), EINVAL, "parts must be in 1..64"),
    ("parts_65", dict(parts=65), EINVAL, "parts must be in 1..64"),
    ("null_y_start", dict(y_start=None), EINVAL, "null pointer"),
    ("y_start_from_1", dict(y_start=(1, 2, 4)), EINVAL, "y_start must rise from 0 to sy"),
    ("y_start_falls", dict(y_start=(0, 3, 2)), EINVAL, "y_start must rise from 0 to sy"),
    ("y_start_short_of_sy", dict(y_start=(0, 2, 3)), EINVAL, "y_start must rise from 0 to sy"),
    ("null_src", dict(src=None), EINVAL, "null pointer"),
    ("null_dst", dict(dst=None), EINVAL, "null pointer"),
    ("y_start_before_empty", dict(zc=0, y_start=(0, 3, 2)), EINVAL, "y_start"),
    ("empty_before_null", dict(zc=0, src=None, dst=None), 0, ""),
    ("valid", dict(), PROBE, ""),
    ("valid_unpack", dict(unpack=1, parts=1, y_start=(0, 4)), PROBE, ""),
  ]),
  "edtb200_slab_step": (_slab_step, [
    ("label_bytes", dict(label_bytes=3), EINVAL, "label_bytes"),
    ("axis_too_long", dict(sx=BIG), ELIMIT, "axis longer than 2^30"),
    ("halo_0", dict(halo=0), EINVAL, "halo must be in 1..254"),
    ("slab_not_deeper_than_halo", dict(sz=2), EINVAL, "deeper than the halo"),
    ("null_labels", dict(labels=None), EINVAL, "null pointer"),
    ("null_f", dict(f=None), EINVAL, "null pointer"),
    ("null_sym_self", dict(sym_self=None), EINVAL, "null pointer"),
    ("null_status", dict(status=None), EINVAL, "null pointer"),
    ("missing_lo", dict(sym_lo=None), EINVAL, "missing neighbour buffer"),
    ("missing_hi", dict(sym_hi=None), EINVAL, "missing neighbour buffer"),
    ("step_0", dict(step=0), EINVAL, "steps are counted from 1"),
    ("depth_before_null", dict(sz=2, labels=None), EINVAL, "deeper than the halo"),
    ("null_before_neighbour", dict(f=None, sym_lo=None), EINVAL, "null pointer"),
    ("neighbour_before_step", dict(sym_hi=None, step=0), EINVAL, "missing neighbour buffer"),
    # a slab without neighbours may be as thin as it likes and needs no neighbour buffers
    ("valid_alone", dict(sz=1, has_lo=0, has_hi=0, sym_lo=None, sym_hi=None), PROBE, ""),
    ("valid", dict(), PROBE, ""),
  ]),
  "edtb200_label_stats": (_label_stats, [
    ("label_bytes", dict(label_bytes=3), EINVAL, "label_bytes"),
    ("negative_size", dict(sy=-1), EINVAL, "negative size"),
    ("capacity_1", dict(capacity=1), EINVAL, "capacity must be a power of two"),
    ("capacity_48", dict(capacity=48), EINVAL, "capacity must be a power of two"),
    ("null_keys", dict(keys=None), EINVAL, "null pointer"),
    ("null_overflow", dict(overflow=None), EINVAL, "null pointer"),
    ("capacity_before_null", dict(capacity=3, dt=None), EINVAL, "capacity"),
    # an empty volume still initialises the table, so it reaches the device
    ("valid_empty", dict(sz=0), PROBE, ""),
    ("valid", dict(), PROBE, ""),
  ]),
  "edtb200_label_extract": (_label_extract, [
    ("label_bytes", dict(label_bytes=3), EINVAL, "label_bytes"),
    ("axis_too_long", dict(sx=BIG), ELIMIT, "axis longer than 2^30"),
    ("null_labels", dict(labels=None), EINVAL, "null pointer"),
    ("null_dt", dict(dt=None), EINVAL, "null pointer"),
    ("null_out", dict(out=None), EINVAL, "null pointer"),
    ("box_below", dict(box=(-1, 0, 0, 3, 3, 3)), EINVAL, "box outside the volume"),
    ("box_above", dict(box=(0, 0, 0, 3, 3, 4)), EINVAL, "box outside the volume"),
    ("null_before_box", dict(out=None, box=(0, 0, 0, 9, 9, 9)), EINVAL, "null pointer"),
    ("empty_box", dict(box=(2, 0, 0, 1, 3, 3)), 0, ""),
    ("valid", dict(), PROBE, ""),
    ("valid_box", dict(box=(1, 1, 1, 2, 3, 3), erase=1), PROBE, ""),
  ]),
}

TABLE = [(name, case, overrides, rc, msg)
         for name, (_, cases) in CASES.items() for case, overrides, rc, msg in cases]


@pytest.mark.parametrize("name,case,overrides,rc,msg", TABLE, ids=["%s-%s" % (t[0][8:], t[1]) for t in TABLE])
def test_argument_check(edt, name, case, overrides, rc, msg):
  check_case(edt, getattr(edt._lib(), name), CASES[name][0], overrides, rc, msg)


@pytest.mark.parametrize("name", sorted(CASES))
def test_every_entry_point_reaches_the_probe_last(edt, name):
  """The table of each entry point has a fully valid call and every one of its rejections."""
  cases = CASES[name][1]
  assert any(rc == PROBE for _, _, rc, _ in cases)
  assert any(rc not in (PROBE, 0) for _, _, rc, _ in cases)


def test_slab_stage_bytes_checks(edt):
  """edtb200_slab_stage_bytes touches no device and reports a bad argument as -1."""
  lib = edt._lib()
  ok = lib.edtb200_slab_stage_bytes(64, 32, 4, 8)
  assert ok > 0
  assert lib.edtb200_slab_stage_bytes(64, 32, 4, 16) > ok
  for args in [(0, 32, 4, 8), (64, 0, 4, 8), (-1, 32, 4, 8), (64, 32, 3, 8), (64, 32, 4, 0), (64, 32, 4, 255)]:
    assert lib.edtb200_slab_stage_bytes(*args) == -1, args
