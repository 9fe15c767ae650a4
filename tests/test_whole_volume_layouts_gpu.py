"""GPU tests: the input layouts every whole-volume operation and transform accepts -- the spherical
morphology, parabolic erosion and dilation with and without return_indices, medial_axis, skeletonize,
nearest_labels, edt and sdf (max_distance= applies to single volumes only, so their stacked rows run
unbounded), feature_transform with distances and expand_labels.  A device
tensor that is neither C- nor F-contiguous, a __cuda_array_interface__ object that is not a torch tensor, an
F-ordered device stack and a strided host array each give, bit for bit, what the host call gives on a numpy
array of the same values in the same memory order (a strided one: its C-contiguous copy; a wrapper: the
tensor it wraps), with the strides that call returns."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CALLS = {
  "spherical_erode": lambda edt, x, w, s: (edt.spherical_erode(x, 2.0, w, True, stacked=s),),
  "spherical_dilate": lambda edt, x, w, s: (edt.spherical_dilate(x, 2.0, w, stacked=s),),
  "spherical_open": lambda edt, x, w, s: (edt.spherical_open(x, 2.0, w, True, stacked=s),),
  "spherical_close": lambda edt, x, w, s: (edt.spherical_close(x, 2.0, w, True, stacked=s),),
  "parabolic_erode": lambda edt, x, w, s: (edt.parabolic_erode(x, w, stacked=s),),
  "parabolic_dilate": lambda edt, x, w, s: (edt.parabolic_dilate(x, w, stacked=s),),
  "parabolic_erode_indices": lambda edt, x, w, s: edt.parabolic_erode(x, w, stacked=s, return_indices=True),
  "parabolic_dilate_indices": lambda edt, x, w, s: edt.parabolic_dilate(x, w, stacked=s, return_indices=True),
  "medial_axis": lambda edt, x, w, s: edt.medial_axis(x, w, True, return_distance=True, stacked=s),
  "skeletonize": lambda edt, x, w, s: edt.skeletonize(x, w, return_distance=True, stacked=s),
  "nearest_labels": lambda edt, x, w, s: edt.nearest_labels(x, 2.0, w, k=2, stacked=s),
  "edt": lambda edt, x, w, s: (edt.edt(x, w, True, stacked=s),),
  "sdf": lambda edt, x, w, s: (edt.sdf(x, w, stacked=s),),
  "edt_max_distance": lambda edt, x, w, s: (edt.edt(x, w, True, stacked=s, max_distance=None if s else 2.5),),
  "sdf_max_distance": lambda edt, x, w, s: (edt.sdf(x, w, stacked=s, max_distance=None if s else 2.5),),
  "feature_transform": lambda edt, x, w, s: edt.feature_transform(x, w, True, return_distances=True, stacked=s),
  "expand_labels": lambda edt, x, w, s: (edt.expand_labels(x, 2.0, w, stacked=s),),
}
WEIGHTS = (1.0, 2.0, 3.0)


def _labels(seed):
  """int32 blocks of three labels and background, 3 voxels wide, with single-voxel specks."""
  rng = np.random.default_rng(seed)
  lab = rng.integers(0, 4, (3, 4, 4)).astype(np.int32)
  for axis in range(3):
    lab = np.repeat(lab, 3, axis)
  specks = rng.random(lab.shape) < 0.05
  lab[specks] = rng.integers(0, 4, int(specks.sum()))
  return lab                                      # (9, 12, 12)


def _host(x):
  return x if isinstance(x, np.ndarray) else x.cpu().numpy()


def _strides(x):
  """Strides in elements, of a numpy array or a torch tensor."""
  return tuple(s // x.itemsize for s in x.strides) if isinstance(x, np.ndarray) else tuple(x.stride())


def _same(got, want):
  """Bit for bit, with the same strides."""
  assert len(got) == len(want)
  for g, w in zip(got, want):
    assert _strides(g) == _strides(w), (_strides(g), _strides(w))
    g, w = _host(g), _host(w)
    assert g.shape == w.shape and g.dtype == w.dtype
    assert g.tobytes() == w.tobytes()


class _Interface:
  """A device array that is not a torch tensor: it only exports __cuda_array_interface__."""

  def __init__(self, t):
    self._t = t

  @property
  def __cuda_array_interface__(self):
    return self._t.__cuda_array_interface__


@pytest.mark.parametrize("name", list(CALLS))
def test_a_strided_device_tensor(edt, name):
  import torch
  lab = _labels(1)
  t = torch.from_numpy(lab).cuda()[:, ::2]
  assert not t.is_contiguous() and not t.permute(2, 1, 0).is_contiguous()
  got = CALLS[name](edt, t, WEIGHTS, False)
  for g in got:
    assert isinstance(g, torch.Tensor) and g.is_cuda and g.is_contiguous()
  _same(got, CALLS[name](edt, t.contiguous(), WEIGHTS, False))
  want = CALLS[name](edt, np.ascontiguousarray(lab[:, ::2]), WEIGHTS, False)
  assert len(got) == len(want)
  for g, w in zip(got, want):
    assert _host(g).tobytes() == w.tobytes()


@pytest.mark.parametrize("name", list(CALLS))
@pytest.mark.parametrize("order", ["C", "F"])
def test_a_cuda_array_interface_object(edt, name, order):
  import torch
  lab = _labels(2)
  t = torch.from_numpy(lab).cuda()
  if order == "F":
    t = t.permute(2, 1, 0).contiguous().permute(2, 1, 0)
  got = CALLS[name](edt, _Interface(t), WEIGHTS, False)
  for g in got:
    assert isinstance(g, torch.Tensor) and g.is_cuda
  _same(got, CALLS[name](edt, t, WEIGHTS, False))


@pytest.mark.parametrize("name", list(CALLS))
def test_an_f_ordered_device_stack(edt, name):
  import torch
  lab = np.asfortranarray(_labels(3))             # 12 volumes of 9 x 12 along the last axis
  t = torch.from_numpy(np.ascontiguousarray(lab.T)).cuda().permute(2, 1, 0)
  got = CALLS[name](edt, t, WEIGHTS[:2], True)
  for g in got:
    assert isinstance(g, torch.Tensor) and g.is_cuda
  _same(got, CALLS[name](edt, lab, WEIGHTS[:2], True))


@pytest.mark.parametrize("name", list(CALLS))
def test_a_strided_host_array(edt, name):
  lab = _labels(4)
  view = lab[:, ::2]
  assert not view.flags.c_contiguous and not view.flags.f_contiguous
  got = CALLS[name](edt, view, WEIGHTS, False)
  for g in got:
    assert isinstance(g, np.ndarray)
  _same(got, CALLS[name](edt, np.ascontiguousarray(view), WEIGHTS, False))
