"""What the C-ABI argument tests share: the return codes and flags of include/edt_b200.h, the ABI
version the entry points are additions at, its prototypes and doc comments, and the runner of a table
of argument cases.

Every entry point rejects a bad argument with a return code and a message before it touches a device,
so these checks run on any machine.  A fully valid call stops at the device probe: device 63 is "no
usable CUDA device" on a machine without a GPU and "out of range" on one with a GPU, device 64 is a
"bad device" everywhere.
"""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "include", "edt_b200.h")) as _f:
  HEADER = _f.read()

ABI_VERSION = 202                 # the entry points added since are additions at this version

_CODES = {name: int(value) for name, value in re.findall(r"#define EDTB200_(E[A-Z]+)\s+\((-\d+)\)", HEADER)}
EINVAL, ECUDA, ELIMIT = (_CODES[name] for name in ("EINVAL", "ECUDA", "ELIMIT"))
_FLAGS = {name: int(value) for name, value in re.findall(r"#define EDTB200_([A-Z_]+)\s+(\d+)", HEADER)}
SQRT, SIGNED, LABELS_ON_DEVICE, OUT_ON_DEVICE, LABELS_FLOAT = (
  _FLAGS[name] for name in ("SQRT", "SIGNED", "LABELS_ON_DEVICE", "OUT_ON_DEVICE", "LABELS_FLOAT"))
BOTH = LABELS_ON_DEVICE | OUT_ON_DEVICE

PROBE = "probe"                   # expected outcome of a call that passes every argument check
BIG = (1 << 30) + 1               # one more than the longest axis
INF, NAN = float("inf"), float("nan")

_PROTOTYPE = re.compile(r"^(\w[\w ]*?\**)\s*\b(edtb200_\w+)\(([^)]*)\);", re.M)


def prototypes():
  """{name: (return type, [parameter, ...])} of every function the header declares, with the whitespace
  of each normalised; a (void) prototype has no parameters."""
  out = {}
  for m in _PROTOTYPE.finditer(HEADER):
    params = [" ".join(p.split()) for p in m.group(3).split(",")]
    out[m.group(2)] = (" ".join(m.group(1).split()), [] if params == ["void"] else params)
  return out


def header_doc(name):
  """The doc comment above the prototype of `name`, on one line."""
  at = HEADER.index("int %s(" % name)
  return " ".join(HEADER[HEADER.rindex("/*", 0, at):at].replace("\n *", " ").split())


def expect_probe(edt, device):
  """The return code and message of a fully valid call on `device`."""
  if device >= 64:
    return EINVAL, b"bad device %d" % device
  if edt.device_count() == 0:
    return ECUDA, b"no usable CUDA device"
  return EINVAL, b"device %d out of range" % device


def check_case(edt, fn, build, overrides, rc, msg):
  """Calls fn(*build(**overrides)) and checks its return code and that the last error holds msg.  A
  PROBE case is called on devices 63 and 64 instead and must stop at the probe of each."""
  last_error = edt._lib().edtb200_last_error
  if rc != PROBE:
    got = fn(*build(**overrides))
    err = last_error() or b""
    assert got == rc, (got, err)
    assert msg.encode() in err, err
    return
  for device in (63, 64):
    got = fn(*build(**dict(overrides, device=device)))
    err = last_error() or b""
    want_rc, want_msg = expect_probe(edt, device)
    assert got == want_rc and want_msg in err, (device, got, err)


@pytest.fixture
def no_device_use(edt, monkeypatch):
  """Fails the test if a call reaches the C library."""
  class Tripwire:
    def __getattr__(self, name):
      raise AssertionError("the library was used (%s) before the arguments were checked" % name)
  monkeypatch.setattr(edt, "_lib", lambda: Tripwire())
  return edt
