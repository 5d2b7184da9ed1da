"""The C-ABI shared library loads on a CPU-only box and exports exactly what include/ovn_b200.h
declares; the product path fails loudly (no CPU fallback) when no GPU is present."""
import ctypes as C
import os
import re

import pytest

from conftest import ROOT


@pytest.fixture(scope='module')
def built():
  from overlapnet_b200 import build
  return build.build()


def header_functions():
  src = open(os.path.join(ROOT, 'include', 'ovn_b200.h')).read()
  src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
  return sorted(set(re.findall(r'\b(ovn_[a-z0-9_A-Z]+)\s*\(', src)))


def test_header_and_binding_agree(built):
  from overlapnet_b200 import _cabi
  assert sorted(_cabi.SYMBOLS) == header_functions()


def test_library_exports_every_declared_symbol(built):
  lib = C.CDLL(built)
  for name in header_functions():
    assert hasattr(lib, name), name
  from overlapnet_b200 import _cabi
  assert _cabi.lib().ovn_abi_version() == _cabi.OVN_ABI_VERSION


def test_config_struct_layout_matches_header(built):
  from overlapnet_b200 import _cabi
  cfg = _cabi.OvnConfig()
  _cabi.lib().ovn_default_config(C.byref(cfg))
  assert (cfg.abi_version, cfg.proj_H, cfg.proj_W) == (1, 64, 900)
  assert (cfg.fov_up_deg, cfg.fov_down_deg, cfg.max_range) == (3.0, -25.0, 50.0)
  assert (cfg.use_depth, cfg.use_normals, cfg.n_prob_channels, cfg.use_intensity) == (1, 1, 0, 0)
  assert list(cfg.strides_layer1) == [2, 2] and cfg.additional_unsymmetric_layer3a == 1
  assert (cfg.leg_output_width, cfg.conv1size, cfg.precision) == (360, 15, 1)
  assert (cfg.max_batch_scans, cfg.max_batch_pairs) == (16, 1101)
  assert C.sizeof(_cabi.OvnConfig) == 18 * 4


def test_no_cpu_fallback(built):
  """Without a CUDA device ovn_create must fail with OVN_ERR_NO_DEVICE, never compute on the CPU."""
  import torch
  if torch.cuda.is_available():
    pytest.skip('a GPU is present')
  from overlapnet_b200 import _cabi
  L = _cabi.lib()
  cfg = _cabi.OvnConfig()
  L.ovn_default_config(C.byref(cfg))
  h = C.c_void_p(0)
  st = L.ovn_create(C.byref(cfg), C.byref(h))
  assert st == -5 and L.ovn_status_string(st) == b'OVN_ERR_NO_DEVICE'
  assert b'no CPU fallback' in L.ovn_last_error(None)
  from overlapnet_b200.engine import Engine
  with pytest.raises(_cabi.OvnError):
    Engine()


def test_product_never_imports_oracle():
  """Only tests/, __graft_entry__.smoke() and bench.py may touch oracle/."""
  pkg = os.path.join(ROOT, 'overlapnet_b200')
  for dp, _, files in os.walk(pkg):
    for f in files:
      if f.endswith(('.py', '.cu', '.cuh', '.h')):
        txt = open(os.path.join(dp, f)).read()
        assert 'import oracle' not in txt and 'from oracle' not in txt, os.path.join(dp, f)


def test_only_buffer_allocates_and_frees():
  """Every device and pinned block is owned by ovn::Buffer (common.cuh): its class body and Buffer::ensure are
  the only code that allocates or frees one."""
  csrc = os.path.join(ROOT, 'overlapnet_b200', 'csrc')
  alloc = re.compile(r'\bcuda(Malloc\w*|Free\w*|HostAlloc)\s*\(')
  owner = re.compile(r'^class Buffer \{$.*?^\};$|^int Buffer<T, Pinned>::ensure\(.*?^\}$', re.S | re.M)
  seen_owner = 0
  for f in sorted(os.listdir(csrc)):
    src = open(os.path.join(csrc, f)).read()
    if f == 'common.cuh':
      seen_owner = len(owner.findall(src))
      src = owner.sub('', src)
    code = re.sub(r'//.*', '', src)
    assert not alloc.search(code), (f, alloc.findall(code))
  assert seen_owner == 2


def csrc_code():
  """{file name: source of csrc/ without // comments}"""
  csrc = os.path.join(ROOT, 'overlapnet_b200', 'csrc')
  return {f: re.sub(r'//.*', '', open(os.path.join(csrc, f)).read()) for f in sorted(os.listdir(csrc))}


def device_error_names():
  enum = re.search(r'enum DeviceError : int \{(.*?)\};', csrc_code()['common.cuh'], re.S)
  assert enum, 'enum DeviceError in common.cuh'
  return dict((n, int(v)) for n, v in re.findall(r'\b(kErr\w+) = (\d+)', enum.group(1)))


def test_only_mbar_ring_touches_mbarriers():
  """Every mbarrier pipeline goes through MbarRing (hopper.cuh): no kernel inits, arrives on or waits on an
  mbarrier itself."""
  direct = re.compile(r'\bmbar_(init|arrive|arrive_expect_tx|wait|try_wait)\s*\(')
  for f, code in csrc_code().items():
    if f != 'hopper.cuh':
      assert not direct.search(code), (f, direct.findall(code))
  assert 'struct MbarRing' in csrc_code()['hopper.cuh']


def test_device_error_codes_are_named():
  """Kernels write only DeviceError names to the error flag, directly or through the ring-wait macros and
  sanitize_indices; the numbers live in the enum alone."""
  names = device_error_names()
  assert len(set(names.values())) == len(names) and {900, 901, 950, 501} <= set(names.values())
  writes = re.compile(r'\batomicExch\(\s*err\s*,\s*([^;]*?)\);|\batomicCAS\(\s*err\s*,\s*0\s*,\s*([^;]*?)\);')
  waits = re.compile(r'\b(?:PIPE_WAIT|INFLIGHT_WAIT)\((.*?),\s*(\w+)\);')
  n_writes = n_waits = 0
  for f, code in csrc_code().items():
    code = re.sub(r'#define (PIPE_WAIT|INFLIGHT_WAIT)\(ok, code\)(.*\\\n)*.*\n', '', code)
    for m in writes.finditer(code):
      value = (m.group(1) or m.group(2)).strip('() ')
      n_writes += 1
      # k_sanitize_idx writes the code its caller passes, checked below
      assert value in names or (f == 'api.cu' and value == 'code'), (f, m.group(0))
    for m in waits.finditer(code):
      n_waits += 1
      assert m.group(2) in names, (f, m.group(0))
    for m in re.finditer(r'\bsanitize_indices\(([^;]*)\);', code):
      args = [a.strip() for a in m.group(1).split(',')]
      assert args[4] in names or args[4] == 'int code', (f, m.group(0))
  assert n_writes >= 3 and n_waits == 16


def test_every_device_error_has_a_message():
  body = re.search(r'^int check_device_error\(.*?^\}$', csrc_code()['api.cu'], re.S | re.M)
  assert body, 'check_device_error in api.cu'
  cases = set(re.findall(r'\bcase (kErr\w+):', body.group(0)))
  assert cases == set(device_error_names())
