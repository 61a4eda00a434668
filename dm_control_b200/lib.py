"""ctypes binding of libb200mj.so (C ABI: include/b200mj.h). No fallback: a missing library raises."""
from __future__ import annotations

import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
# B200MJ_SO: developer override (A/B runs of two builds of the library side by side); the default is the
# in-tree library __graft_entry__.build() produces
SO_PATH = os.environ.get('B200MJ_SO') or os.path.join(_HERE, 'csrc', 'libb200mj.so')
HEADER = os.path.join(_ROOT, 'include', 'b200mj.h')

_c_double_p = ctypes.POINTER(ctypes.c_double)
_c_int_p = ctypes.POINTER(ctypes.c_int32)


def _io_fields_from_header():
  """Parse `struct b200mj_io` out of include/b200mj.h so the ctypes mirror cannot drift."""
  text = open(HEADER).read()
  body = re.search(r'typedef struct b200mj_io \{(.*?)\} b200mj_io;', text, flags=re.S).group(1)
  body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
  fields = []
  for m in re.finditer(r'(const\s+)?(double|int32_t)\s*\*\s*(\w+)\s*;', body):
    fields.append((m.group(3), _c_double_p if m.group(2) == 'double' else _c_int_p))
  return fields


IO_FIELDS = _io_fields_from_header()


class IO(ctypes.Structure):
  _fields_ = IO_FIELDS


STEP_LEGACY, STEP_FULL_FINAL, STEP_SENSORS, STEP_REUSE_POS = 1, 2, 4, 8

# every symbol include/b200mj.h declares
SYMBOLS = ('b200mj_model_create', 'b200mj_model_destroy', 'b200mj_model_set_disableflags', 'b200mj_model_set_capacity',
           'b200mj_step', 'b200mj_forward', 'b200mj_step_host', 'b200mj_workspace_bytes', 'b200mj_envs_per_block', 'b200mj_describe',
           'b200mj_launch_count', 'b200mj_error_string', 'b200mj_version', 'b200mj_reset', 'b200mj_forward_masked',
           'b200mj_contact_force', 'b200mj_subtree_vel', 'b200mj_model_set_variable_geoms', 'b200mj_render',
           'b200mj_model_set_env_fields')

_lib = None


class EngineError(RuntimeError):
  pass


def load():
  """Load the engine. Raises (never falls back) when the CUDA library has not been built."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(SO_PATH):
    raise EngineError(f'{SO_PATH} is missing: run `python -c "import __graft_entry__ as g; g.build()"` '
                      '(nvcc, sm_90a). There is no CPU fallback.')
  L = ctypes.CDLL(SO_PATH)
  vp = ctypes.c_void_p
  L.b200mj_model_create.argtypes = [_c_int_p, ctypes.c_int, _c_double_p, ctypes.c_int, ctypes.POINTER(vp)]
  L.b200mj_model_create.restype = ctypes.c_int
  L.b200mj_model_destroy.argtypes = [vp]
  L.b200mj_model_destroy.restype = None
  L.b200mj_model_set_disableflags.argtypes = [vp, ctypes.c_int]
  L.b200mj_model_set_capacity.argtypes = [vp, ctypes.c_int, ctypes.c_int]
  L.b200mj_step.argtypes = [vp, ctypes.POINTER(IO), ctypes.c_int, ctypes.c_int, ctypes.c_int, vp]
  L.b200mj_forward.argtypes = [vp, ctypes.POINTER(IO), ctypes.c_int, ctypes.c_int, ctypes.c_int, vp]
  L.b200mj_step_host.argtypes = [vp, ctypes.POINTER(IO), ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, vp, vp, vp,
                                 ctypes.c_int, vp]
  L.b200mj_reset.argtypes = [vp, ctypes.POINTER(IO), ctypes.c_int, vp, ctypes.c_int, vp]
  L.b200mj_forward_masked.argtypes = [vp, ctypes.POINTER(IO), ctypes.c_int, vp, ctypes.c_int, ctypes.c_int, vp]
  L.b200mj_contact_force.argtypes = [vp, ctypes.POINTER(IO), ctypes.c_int, ctypes.c_int, vp, vp]
  L.b200mj_subtree_vel.argtypes = [vp, ctypes.POINTER(IO), ctypes.c_int, ctypes.c_int, vp]
  L.b200mj_model_set_variable_geoms.argtypes = [vp, _c_int_p, ctypes.c_int]
  L.b200mj_model_set_env_fields.argtypes = [vp, _c_int_p, ctypes.c_int, vp, ctypes.c_int]
  for f in ('b200mj_step', 'b200mj_forward', 'b200mj_step_host', 'b200mj_model_set_disableflags',
            'b200mj_model_set_capacity', 'b200mj_envs_per_block', 'b200mj_reset', 'b200mj_forward_masked', 'b200mj_contact_force',
            'b200mj_subtree_vel', 'b200mj_model_set_variable_geoms', 'b200mj_model_set_env_fields'):
    getattr(L, f).restype = ctypes.c_int
  if hasattr(L, 'b200mj_render'):      # (absent from the CPU emulation build of the physics kernels, tests/emu: no renderer there)
    L.b200mj_render.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, vp, vp, vp]
    L.b200mj_render.restype = ctypes.c_int
  L.b200mj_workspace_bytes.argtypes = [vp]
  L.b200mj_workspace_bytes.restype = ctypes.c_int64
  L.b200mj_envs_per_block.argtypes = [vp]
  L.b200mj_describe.argtypes = [vp, ctypes.c_char_p, ctypes.c_int]
  L.b200mj_describe.restype = ctypes.c_int
  L.b200mj_launch_count.restype = ctypes.c_int64
  L.b200mj_error_string.argtypes = [ctypes.c_int]
  L.b200mj_error_string.restype = ctypes.c_char_p
  L.b200mj_version.restype = ctypes.c_char_p
  _lib = L
  return L


def check(code):
  if code != 0:
    raise EngineError(f'b200mj error {code}: {load().b200mj_error_string(code).decode()}')
