"""`SingleEnvPhysics`: the reference's numpy `mujoco.Physics` surface (dm_control/mujoco/engine.py) on a B = 1 view of
`BatchedPhysics`, so that UNMODIFIED reference tasks (`suite/humanoid.py`, ...) and the unmodified
`rl/control.py:Environment` can drive this engine: `physics.data.qpos[7:]`, `physics.named.data.xmat['torso', 'zz']`,
`physics.named.data.qpos[joint_name] = x`, `physics.data.ncon`, `physics.data.contact[i].geom1`, `reset_context()`, ...

The host arrays under `.data` are the state between engine calls: every call uploads the state fields and applied forces
of `physics.DATA_FIELDS` from them, runs on the device, and downloads state and outputs back IN PLACE (views
handed out earlier stay valid, as with MuJoCo's own arrays). It exists for API conformance and debugging — one
environment per process is the reference's execution model, not this engine's.
"""
from __future__ import annotations

import contextlib
import types

import numpy as np
import torch

from . import index as _index
from . import mjcf_compile
from . import lib as _lib
from .physics import APPLIED_FIELDS, STATE_FIELDS, BatchedPhysics, PhysicsError


class _Contact:
  __slots__ = ('geom1', 'geom2', 'dist', 'pos', 'frame', 'efc_address')


class _HostData:
  """numpy mirror of one environment's mjData fields (attribute access, like `physics.data`)."""

  def __init__(self, batched):
    object.__setattr__(self, '_arrays', {})
    for name, t in vars(batched.data).items():
      if isinstance(t, torch.Tensor):
        self._arrays[name] = np.zeros(tuple(t.shape[1:]), dtype=np.float64 if t.dtype == torch.float64 else np.int32)

  def __getattr__(self, name):
    arrays = object.__getattribute__(self, '_arrays')
    if name == 'time':
      return float(arrays['time'].reshape(-1)[0])
    if name in ('ncon', 'nefc', 'solver_niter'):
      return int(arrays[name].reshape(-1)[0])
    if name == 'contact':
      n = int(arrays['ncon'].reshape(-1)[0])
      out = []
      for k in range(n):
        c = _Contact()
        c.geom1, c.geom2 = (int(x) for x in arrays['contact_geom'].reshape(-1, 2)[k])
        c.dist = float(arrays['contact_dist'].reshape(-1)[k]); c.pos = arrays['contact_pos'].reshape(-1, 3)[k].copy()
        c.frame = arrays['contact_frame'].reshape(-1, 9)[k].copy(); c.efc_address = int(arrays['contact_efc_address'].reshape(-1)[k])
        out.append(c)
      return out
    if name in arrays:
      return arrays[name]
    raise AttributeError(name)

  def __setattr__(self, name, value):
    arrays = object.__getattribute__(self, '_arrays')
    if name not in arrays:
      raise AttributeError(name)
    arrays[name][...] = value          # `physics.data.time = t`, `physics.data.qpos = q`: in place, views stay valid


class _WritableModel:
  """`physics.model` as the reference hands it out: arrays a task may write in place (`physics.model.wrap_prm[i] = w`,
  suite/point_mass.py:101-112; `named.model.geom_rgba[...] = ...`). The batched facade refuses raw array writes because it
  could not see them; this B = 1 conformance view takes the other route: every array handed out marks the model as
  modified, so the next engine call re-uploads it (cheap for one small model, and never on the throughput path)."""

  def __init__(self, model):
    object.__setattr__(self, '_m', model)

  def __getattr__(self, name):
    m = object.__getattribute__(self, '_m')
    if name in m.fields:
      m.touch()
      return m.fields[name]
    return getattr(m, name)

  def id2name(self, object_id, object_type):
    """MuJoCo's answer: the empty string for an element the MJCF left unnamed (the compiler's internal `_geom12`-style
    placeholders are not names)."""
    n = object.__getattribute__(self, '_m').id2name(object_id, object_type)
    return '' if n.startswith('_') else n

  def __setattr__(self, name, value):
    setattr(object.__getattribute__(self, '_m'), name, value)


class SingleEnvPhysics:
  legacy_step = True

  def __init__(self, model, device=None):
    self._b = BatchedPhysics(model, batch=1, device=device, outputs='all')
    self._b.enable_applied_forces(True)
    self.model = _WritableModel(model)
    self.data = _HostData(self._b)
    named_model = _index.NamedIndexStructs(types.SimpleNamespace(model=model, data=types.SimpleNamespace())).model
    self.named = types.SimpleNamespace(data=_index._Struct(self.data._arrays.get, model, False), model=named_model)
    self._pull()
    self._reload_from_data(self.data)

  def _reload_from_data(self, data):
    """The hook `mujoco.Physics.__init__` / `reload_from_*` / `__setstate__` run when a Physics is bound to its data
    (engine.py:116-123, 370-392). Domain subclasses override it to reset caches (suite/quadruped.py:148-152) and call up."""

  # ---- construction (engine.py:451-503) ----
  @classmethod
  def _with_full_capacity(cls, model):
    """MuJoCo sizes its constraint arena dynamically; the compiler's default `njmax` is capped for the throughput path's
    shared-memory budget (160 rows). This single-environment view asks for every row the model can produce (equality +
    friction + limits + 4 per contact slot) when the workspace still fits, so that e.g. the CMU humanoid lying on the floor
    (56 limited joints, dozens of contacts) does not hit mjWARN_CNSTRFULL where the reference would not."""
    need = int(6 * model.neq + np.count_nonzero(np.asarray(model.dof_frictionloss) > 0) + np.count_nonzero(model.jnt_limited) + 4 * model.nconmax)
    for rows in (need, (3 * need + model.njmax) // 4, (need + model.njmax) // 2, (need + 3 * model.njmax) // 4):
      if rows <= model.njmax:
        break
      big = model.copy()
      big.set_capacity(njmax=rows)
      try:
        return cls(big)
      except _lib.EngineError:
        continue        # does not fit 227 KB of shared memory: try fewer rows, in the end the default capacity
    return cls(model)

  @classmethod
  def from_xml_string(cls, xml_string, assets=None):
    return cls._with_full_capacity(mjcf_compile.compile_xml(xml_string, assets=assets))

  @classmethod
  def from_xml_path(cls, path):
    return cls._with_full_capacity(mjcf_compile.compile_file(path))

  # ---- host <-> device ----
  def _push(self):
    a, d = self.data._arrays, self._b.data
    for name in STATE_FIELDS + APPLIED_FIELDS:
      t = getattr(d, name, None)
      if t is not None and name in a and t.numel():
        t[0].copy_(torch.as_tensor(np.ascontiguousarray(a[name]).reshape(tuple(t.shape[1:]))))

  def _pull(self):
    a, d = self.data._arrays, self._b.data
    for name, arr in a.items():
      t = getattr(d, name, None)
      if t is not None and t.numel():
        arr[...] = t[0].cpu().numpy().reshape(arr.shape)

  # ---- reference Physics API (engine.py:139-176, 306-343, 505-640) ----
  def set_control(self, control):
    np.copyto(self.data._arrays['ctrl'], np.asarray(control, dtype=np.float64).reshape(-1))

  def step(self, nstep=1):
    self._b.legacy_step = self.legacy_step
    self._push()
    self._b.mark_as_dirty()             # the host arrays may have been edited: never start from a stale position stage
    try:
      self._b.step(nstep)
    finally:
      self._pull()

  def forward(self):
    self._push()
    try:
      self._b.forward()
    finally:
      self._pull()

  def reset(self, keyframe_id=None):
    try:
      self._b.reset(keyframe_id)
    finally:
      self._pull()

  def after_reset(self):
    self._push()
    try:
      self._b.after_reset()
    finally:
      self._pull()

  @contextlib.contextmanager
  def reset_context(self):
    try:
      self.reset()
    except PhysicsError:
      pass
    yield self
    self.after_reset()

  def check_divergence(self):
    a = self.data._arrays
    if not (np.isfinite(a['qpos']).all() and np.isfinite(a['qvel']).all()):
      raise PhysicsError('Physics state has diverged (non-finite qpos/qvel).')

  @contextlib.contextmanager
  def suppress_physics_errors(self):
    with self._b.suppress_physics_errors():
      yield

  def time(self):
    return self.data.time

  def timestep(self):
    return self._b.timestep()

  # engine.py:589-614: each returns a COPY (the reference's own suite_test.py checks that consecutive observations do not
  # share memory)
  def control(self):
    return self.data._arrays['ctrl'].copy()

  def activation(self):
    return self.data._arrays['act'].copy()

  def position(self):
    return self.data._arrays['qpos'].copy()

  def velocity(self):
    return self.data._arrays['qvel'].copy()

  def state(self):
    a = self.data._arrays
    return np.concatenate([a['qpos'], a['qvel'], a['act']])

  def get_state(self):
    return self.state()

  def set_state(self, state):
    a = self.data._arrays
    nq, nv = a['qpos'].size, a['qvel'].size
    a['qpos'][:] = state[:nq]; a['qvel'][:] = state[nq:nq + nv]; a['act'][:] = state[nq + nv:]

  def free(self):
    self._b.free()
