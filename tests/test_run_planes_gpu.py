"""GPU tests (-m gpu) of the run-start bit planes: on predicted label noise with labels of 4 or 8
bytes, the X pass writes one run-start bit per voxel and later axis, and the later passes read those
instead of the labels.  The prediction comes from the previous transform on the device, so every
volume here is transformed twice in a row and the second result is compared with the oracle bit for
bit: ragged extents (sx, sy, sz not multiples of 32 or 128), 2-D and 3-D, black_border, sqrt, both
label widths, the device-resident and batch entry points, shapes in turn, and a structured volume
right after noise (planes written for a prediction that turns out wrong).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

WIDE = (np.uint32, np.uint64)


def noise(shape, dtype, seed, background=0.02):
  """Label noise: almost every voxel differs from its neighbours, a few are background."""
  rng = np.random.default_rng(seed)
  lab = rng.integers(1, 1 << 20, shape).astype(dtype)
  lab[rng.random(shape) < background] = 0
  return lab


def blocky(shape, dtype, seed, cell=3):
  rng = np.random.default_rng(seed)
  out = rng.integers(0, 5, [-(-s // cell) for s in shape]).astype(dtype)
  for ax in range(len(shape)):
    out = np.repeat(out, cell, axis=ax)
  return np.ascontiguousarray(out[tuple(slice(0, s) for s in shape)])


def twice(fn, labels, **kw):
  fn(labels, **kw)                      # leaves the run statistic of this volume behind
  return fn(labels, **kw)


# C order: the last extent is x
SHAPES_3D = [(33, 37, 44), (17, 70, 132), (40, 33, 256), (9, 65, 100), (20, 31, 512), (5, 6, 4)]


@pytest.mark.parametrize("shape", SHAPES_3D, ids=["x".join(map(str, s)) for s in SHAPES_3D])
@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_3d_noise_bit_exact(edt, oracle, shape, dtype):
  lab = noise(shape, dtype, sum(shape))
  for border in (False, True):
    for fn in ("edtsq", "edt"):
      got = twice(getattr(edt, fn), lab, anisotropy=(1.0, 2.0, 3.0), black_border=border)
      want = getattr(oracle, fn)(lab, anisotropy=(1.0, 2.0, 3.0), black_border=border)
      assert np.array_equal(got, want), (fn, border, int((got != want).sum()))


def test_noise_takes_the_label_noise_plan(edt):
  lab = noise((16, 40, 256), np.uint32, 1)
  twice(edt.edtsq, lab)
  info = edt.last_later_launch()
  assert info["kernel"] == "tile" and info["ctas"] == 2, info


SHAPES_2D = [(37, 44), (70, 132), (65, 512), (3, 4)]


@pytest.mark.parametrize("shape", SHAPES_2D, ids=["x".join(map(str, s)) for s in SHAPES_2D])
@pytest.mark.parametrize("dtype", WIDE, ids=[d.__name__ for d in WIDE])
def test_2d_noise_bit_exact(edt, oracle, shape, dtype):
  lab = noise(shape, dtype, sum(shape) + 7)
  for border in (False, True):
    got = twice(edt.edtsq, lab, anisotropy=(1.5, 1.0), black_border=border)
    assert np.array_equal(got, oracle.edtsq(lab, anisotropy=(1.5, 1.0), black_border=border)), border


def test_signed_and_narrow_labels_after_noise(edt, oracle):
  # planes are not taken for these; the prediction is still "noise"
  lab = noise((20, 33, 132), np.uint32, 3)
  edt.edtsq(lab)
  assert np.array_equal(edt.sdf(lab, black_border=True), oracle.sdf(lab, black_border=True))
  for dtype in (np.uint8, np.uint16):
    small = noise((20, 33, 132), dtype, 4) if dtype == np.uint16 else \
        np.random.default_rng(4).integers(0, 256, (20, 33, 132)).astype(np.uint8)
    assert np.array_equal(twice(edt.edtsq, small), oracle.edtsq(small)), dtype


def test_structured_right_after_noise(edt, oracle):
  edt.edtsq(noise((24, 40, 128), np.uint32, 5))
  lab = blocky((24, 40, 128), np.uint32, 6)
  assert np.array_equal(edt.edtsq(lab, black_border=True), oracle.edtsq(lab, black_border=True))


def test_shapes_in_turn(edt, oracle):
  for shape in [(20, 30, 40), (64, 64, 512), (7, 9, 12), (33, 40, 256), (20, 30, 40)]:
    lab = noise(shape, np.uint32, sum(shape))
    assert np.array_equal(twice(edt.edtsq, lab, black_border=True), oracle.edtsq(lab, black_border=True)), shape


def test_device_resident_and_batch(edt, oracle):
  torch = pytest.importorskip("torch")
  lab = noise((24, 40, 68), np.int32, 8)
  t = torch.from_numpy(lab).cuda()
  got = twice(edt.edt_cuda, t, sqrt=True).cpu().numpy()
  assert np.array_equal(got, oracle.edt(lab.astype(np.uint32)))
  batch = [noise((24, 40, 68), np.uint32, s) for s in range(4)]
  outs = twice(edt.transform_batch, batch, black_border=True)
  for v, o in zip(batch, outs):
    assert np.array_equal(o, oracle.edtsq(v, black_border=True))
