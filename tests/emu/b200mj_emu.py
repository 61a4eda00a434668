"""CPU emulation build of the CUDA engine, for tests only (see cuda_emu.h).

`build()` compiles dm_control_b200/csrc/b200mj.cu with g++ -DB200MJ_CPU_EMU into tests/emu/_build/; `EmuPhysics` drives
the resulting library through the very same C ABI (include/b200mj.h) with numpy arrays standing in for device memory.
Nothing here is reachable from the product package.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

from dm_control_b200 import lib as blib
from dm_control_b200.physics import APPLIED_FIELDS, STATE_FIELDS, BatchedPhysics

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SRC = os.path.join(_ROOT, 'dm_control_b200', 'csrc', 'b200mj.cu')
# the kernel source and every header it includes: an edit to any of them rebuilds the emulation library
_DEPS = [_SRC, os.path.join(_HERE, 'cuda_emu.h')] + [os.path.join(_ROOT, 'include', h) for h in
                                                    ('b200mj.h', 'b200mj_model_fields.h', 'b200mj_convex.h')]
_SO = os.path.join(_HERE, '_build', 'libb200mj_emu.so')
_lib = None


def build(force=False):
  if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(d) for d in _DEPS):
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    subprocess.check_call(['g++', '-std=c++20', '-O1', '-fPIC', '-shared', '-pthread', '-x', 'c++', '-DB200MJ_CPU_EMU',
                           '-Wno-unknown-pragmas', '-I' + _HERE, '-o', _SO, _SRC])
  return _SO


def load():
  global _lib
  if _lib is None:
    L = ctypes.CDLL(build())
    vp = ctypes.c_void_p
    L.b200mj_model_create.argtypes = [ctypes.POINTER(ctypes.c_int32), ctypes.c_int, ctypes.POINTER(ctypes.c_double),
                                      ctypes.c_int, ctypes.POINTER(vp)]
    L.b200mj_model_destroy.argtypes = [vp]; L.b200mj_model_destroy.restype = None
    L.b200mj_step.argtypes = [vp, ctypes.POINTER(blib.IO), ctypes.c_int, ctypes.c_int, ctypes.c_int, vp]
    L.b200mj_forward.argtypes = [vp, ctypes.POINTER(blib.IO), ctypes.c_int, ctypes.c_int, ctypes.c_int, vp]
    L.b200mj_model_set_disableflags.argtypes = [vp, ctypes.c_int]
    L.b200mj_describe.argtypes = [vp, ctypes.c_char_p, ctypes.c_int]
    _lib = L
  return _lib


class EmuPhysics:
  """B environments stepped by the emulated kernels; `data.<field>` are numpy arrays with a leading batch axis."""

  def __init__(self, model, batch, sensors=True, full_final=True, legacy_step=True, applied_forces=False, outputs='all',
               reuse_pos=False):
    self._reuse_pos, self._pos_current = reuse_pos, False
    self._L = load()
    self.model, self.batch = model, int(batch)
    self._sensors, self._full_final, self.legacy_step = sensors, full_final, legacy_step
    idata, rdata = model.pack()
    self._blob = (idata, rdata)
    self._h = ctypes.c_void_p()
    rc = self._L.b200mj_model_create(idata.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), idata.size,
                                     rdata.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), rdata.size, ctypes.byref(self._h))
    if rc:
      raise RuntimeError(f'b200mj_model_create (emulation) failed: {rc}')
    self.data = type('Data', (), {})()
    self._io = blib.IO()
    for name, shp in BatchedPhysics._FIELDS:
      setattr(self.data, name, np.zeros((batch,) + tuple(shp(model)), np.float64))
    for name, shp in BatchedPhysics._INT_FIELDS:
      setattr(self.data, name, np.zeros((batch,) + tuple(shp(model)), np.int32))
    for name, ctype in blib.IO_FIELDS:
      a = getattr(self.data, name, None)
      if outputs != 'all' and name not in STATE_FIELDS + APPLIED_FIELDS + ('warning',) and name not in outputs:
        a = None                                   # this output pointer crosses the ABI as NULL
      if a is None or a.size == 0 or (name in APPLIED_FIELDS and not applied_forces):
        setattr(self._io, name, ctypes.cast(None, ctype))
      else:
        setattr(self._io, name, ctypes.cast(a.ctypes.data, ctype))
    self.data.qpos[:] = np.asarray(model.qpos0)

  def _flags(self):
    return ((blib.STEP_LEGACY if self.legacy_step else 0) | (blib.STEP_FULL_FINAL if self._full_final else 0) |
            (blib.STEP_SENSORS if self._sensors else 0))

  def step(self, nstep=1):
    flags = self._flags() | (8 if (self._reuse_pos and self._pos_current) else 0)
    rc = self._L.b200mj_step(self._h, ctypes.byref(self._io), self.batch, int(nstep), flags, None)
    self._pos_current = True
    if rc:
      raise RuntimeError(f'b200mj_step (emulation) failed: {rc}')

  def forward(self, extra_disableflags=0):
    self._pos_current = False
    rc = self._L.b200mj_forward(self._h, ctypes.byref(self._io), self.batch, int(extra_disableflags),
                                blib.STEP_SENSORS if self._sensors else 0, None)
    if rc:
      raise RuntimeError(f'b200mj_forward (emulation) failed: {rc}')

  def step_host(self, ctrl_host, obs_dev, obs_host, nstep=1):
    """b200mj_step_host: host action block in, packed observation block out."""
    vp = ctypes.c_void_p
    self._L.b200mj_step_host.argtypes = [vp, ctypes.POINTER(blib.IO), ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, vp, vp, vp,
                                         ctypes.c_int, vp]
    rc = self._L.b200mj_step_host(self._h, ctypes.byref(self._io), self.batch, int(nstep), self._flags(),
                                  ctrl_host.ctypes.data, self.data.ctrl.ctypes.data, obs_dev.ctypes.data, obs_host.ctypes.data,
                                  obs_dev.shape[1], None)
    if rc:
      raise RuntimeError(f'b200mj_step_host (emulation) failed: {rc}')

  def set_disableflags(self, flags):
    self._L.b200mj_model_set_disableflags(self._h, int(flags))

  def describe(self):
    import json
    buf = ctypes.create_string_buffer(4096)
    self._L.b200mj_describe(self._h, buf, 4096)
    return json.loads(buf.value.decode())

  def __del__(self):
    try:
      if self._h:
        self._L.b200mj_model_destroy(self._h)
    except Exception:
      pass
