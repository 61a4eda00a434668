"""`BatchedPhysics`: the drop-in for `dm_control.mujoco.Physics` on the forward-dynamics hot path.

Mirrors the reference surface the `rl.control.Environment` loop and the suite tasks touch
(dm_control/mujoco/engine.py:83-622 and the `control.Physics` ABC at dm_control/rl/control.py:206-267):
`step`, `forward`, `reset`, `after_reset`, `reset_context`, `set_control`, `time`, `timestep`, `get_state`,
`set_state`, `check_invalid_state`, `suppress_physics_errors`, `.model`, `.data`. The difference is the leading
batch axis: every `data.<field>` is a `[B, ...]` float64 torch tensor resident in HBM, and one `step()` advances
all B environments with a single launch of the hand-written sm_90a kernel through the C ABI (include/b200mj.h).

There is no CPU path here. If libb200mj.so is missing, construction raises `lib.EngineError`.
"""
from __future__ import annotations

import contextlib
import ctypes
import types
from typing import NamedTuple

import numpy as np
import torch

from . import lib as _lib
from . import mjcf_compile
from . import model as _model

_WARNING_NAMES = ('mjWARN_INERTIA', 'mjWARN_CONTACTFULL', 'mjWARN_CNSTRFULL', 'mjWARN_VGEOMFULL', 'mjWARN_BADQPOS',
                  'mjWARN_BADQVEL', 'mjWARN_BADQACC', 'mjWARN_BADCTRL')
DSBL_ACTUATION = 1 << 10

_INVALID_PHYSICS_STATE = ('Physics state is invalid. Warning(s) raised: {warning_names}')


class PhysicsError(RuntimeError):
  """Raised if the state of the physics simulation becomes divergent (reference: rl/control.py:270)."""


def action_spec(physics):
  """(minimum, maximum) float64 arrays of shape [nu]; unlimited controls get -/+ mjMAXVAL (engine.py:1093-1103)."""
  m = physics.model
  limited = m.actuator_ctrllimited.astype(bool)
  lo = np.where(limited, m.actuator_ctrlrange[:, 0], -1e10)
  hi = np.where(limited, m.actuator_ctrlrange[:, 1], 1e10)
  return lo.astype(np.float64), hi.astype(np.float64)


STATE, APPLIED, OUTPUT = 'state', 'applied', 'output'


class DataField(NamedTuple):
  """One batched `data.<name>` field, a `b200mj_io` pointer (include/b200mj.h)."""
  name: str
  dims: tuple        # per-environment shape: model sizes by name ('nbody') and constants
  dtype: torch.dtype
  rows: str | None   # row axis: element kind ('body', 'geom', 'site', 'actuator') or ragged axis ('nq', 'nv', 'na', 'nsensordata')
  cols: str | None   # column names of index.py: 'xyz', 'quat' or 'mat'
  role: str          # STATE: uploaded and downloaded by every call; APPLIED: state once enable_applied_forces(); OUTPUT

  def shape(self, m):
    return tuple(getattr(m, d) if isinstance(d, str) else d for d in self.dims)


_F8, _I4 = torch.float64, torch.int32
# every b200mj_io pointer in the header's order, except var_geom_pos / var_geom_size (set_variable_geoms)
DATA_FIELDS = {f.name: f for f in (DataField(*row) for row in (
    ('qpos', ('nq',), _F8, 'nq', None, STATE),
    ('qvel', ('nv',), _F8, 'nv', None, STATE),
    ('act', ('na',), _F8, 'na', None, STATE),
    ('qacc_warmstart', ('nv',), _F8, 'nv', None, STATE),
    ('time', (), _F8, None, None, STATE),
    ('ctrl', ('nu',), _F8, 'actuator', None, STATE),
    ('qfrc_applied', ('nv',), _F8, 'nv', None, APPLIED),
    ('xfrc_applied', ('nbody', 6), _F8, 'body', None, APPLIED),
    ('xpos', ('nbody', 3), _F8, 'body', 'xyz', OUTPUT),
    ('xquat', ('nbody', 4), _F8, 'body', 'quat', OUTPUT),
    ('xmat', ('nbody', 9), _F8, 'body', 'mat', OUTPUT),
    ('xipos', ('nbody', 3), _F8, 'body', 'xyz', OUTPUT),
    ('geom_xpos', ('ngeom', 3), _F8, 'geom', 'xyz', OUTPUT),
    ('geom_xmat', ('ngeom', 9), _F8, 'geom', 'mat', OUTPUT),
    ('site_xpos', ('nsite', 3), _F8, 'site', 'xyz', OUTPUT),
    ('site_xmat', ('nsite', 9), _F8, 'site', 'mat', OUTPUT),
    ('subtree_com', ('nbody', 3), _F8, 'body', 'xyz', OUTPUT),
    ('subtree_linvel', ('nbody', 3), _F8, 'body', 'xyz', OUTPUT),
    ('cvel', ('nbody', 6), _F8, 'body', None, OUTPUT),
    ('sensordata', ('nsensordata',), _F8, 'nsensordata', None, OUTPUT),
    ('qM', ('nv', 'nv'), _F8, None, None, OUTPUT),
    ('qfrc_bias', ('nv',), _F8, 'nv', None, OUTPUT),
    ('qfrc_passive', ('nv',), _F8, 'nv', None, OUTPUT),
    ('qacc', ('nv',), _F8, 'nv', None, OUTPUT),
    ('qfrc_actuator', ('nv',), _F8, 'nv', None, OUTPUT),
    ('actuator_force', ('nu',), _F8, 'actuator', None, OUTPUT),
    ('qfrc_constraint', ('nv',), _F8, 'nv', None, OUTPUT),
    ('efc_force', ('njmax',), _F8, None, None, OUTPUT),
    ('ncon', (), _I4, None, None, OUTPUT),
    ('contact_geom', ('nconmax', 2), _I4, None, None, OUTPUT),
    ('contact_efc_address', ('nconmax',), _I4, None, None, OUTPUT),
    ('contact_dist', ('nconmax',), _F8, None, None, OUTPUT),
    ('contact_pos', ('nconmax', 3), _F8, None, None, OUTPUT),
    ('contact_frame', ('nconmax', 9), _F8, None, None, OUTPUT),
    ('nefc', (), _I4, None, None, OUTPUT),
    ('solver_niter', (), _I4, None, None, OUTPUT),
    ('warning', (8,), _I4, None, None, OUTPUT)))}    # always allocated: check_invalid_state reads it
STATE_FIELDS = tuple(n for n, f in DATA_FIELDS.items() if f.role == STATE)
APPLIED_FIELDS = tuple(n for n, f in DATA_FIELDS.items() if f.role == APPLIED)

# model fields an environment may hold values of its own (b200mj_model_set_env_fields, include/b200mj.h): the tables a
# domain-randomising task varies per episode and from which the engine derives nothing at model creation
ENV_MODEL_FIELDS = tuple(f.name for f in sorted((f for f in _model.MODEL_FIELDS.values() if f.env is not None),
                                                 key=lambda f: f.env))
_FIELD_ID = {name: k for k, (name, _) in enumerate(_model.FIELDS)}


def check_env_model_fields(names):
  """Raises ValueError naming the first field of `names` that cannot vary per environment, or that is listed twice."""
  seen = set()
  for n in names:
    if n not in ENV_MODEL_FIELDS:
      raise ValueError(f'model field {n!r} cannot vary per environment; the per-environment fields are '
                       f'{", ".join(ENV_MODEL_FIELDS)}')
    if n in seen:
      raise ValueError(f'model field {n!r} is listed twice')
    seen.add(n)


class _Data:
  """Batched mjData slice: `[B, ...]` torch tensors, MuJoCo field names."""


class BatchedPhysics:
  """B copies of one compiled model stepped in lock-step on one GPU."""

  legacy_step = True   # reference default: rl/control.py:209

  # (name, per-environment shape as a function of the model) of the float64 and of the int32 fields
  _FIELDS = tuple((n, f.shape) for n, f in DATA_FIELDS.items() if f.dtype == _F8)
  _INT_FIELDS = tuple((n, f.shape) for n, f in DATA_FIELDS.items() if f.dtype == _I4)

  def __init__(self, model, batch=1, device=None, outputs='all', sensors=True, full_final=True, nconmax=None,
               njmax=None):
    """Args:
      model: `dm_control_b200.model.Model`.
      batch: number of environments B.
      device: torch CUDA device (default: current).
      outputs: 'all' or an iterable of output field names to materialise in HBM each step (the rest stay in
        shared memory only — the observation-contract idea of SURVEY.md Appendix B).
      sensors: evaluate sensors (mj_sensorPos/Vel/Acc) inside the step.
      full_final: the trailing step1 also runs collision + constraint assembly (needed for `data.ncon`/contacts).
      nconmax, njmax: per-environment contact / constraint-row capacities (MJCF <size nconmax njmax>); they size
        the shared-memory workspace, hence occupancy. Overflow raises mjWARN_CONTACTFULL / mjWARN_CNSTRFULL.
    """
    if not torch.cuda.is_available():
      raise _lib.EngineError('BatchedPhysics needs a CUDA device (H100); there is no CPU fallback.')
    self._L = _lib.load()
    if nconmax is not None or njmax is not None:
      model = model.copy()
      model.set_capacity(nconmax, njmax)
    self.model = model
    self.batch = int(batch)
    self.device = torch.device(device if device is not None else f'cuda:{torch.cuda.current_device()}')
    self._sensors = bool(sensors)
    self._full_final = bool(full_final)
    self._suppress = False
    # True while the position stage of the current state is the one the last step() left behind (its trailing
    # mj_step1): the next step() then starts from it, as the reference's legacy ordering does. Every method that
    # changes the state clears it; code that writes `data.qpos/qvel/act` directly must call forward() (the
    # reference's contract) or mark_as_dirty().
    self._pos_current = False
    self._handle = ctypes.c_void_p()
    # bumped whenever what a launch captures by value changes (model handle, disable flags, io pointers, per-environment
    # geoms / model fields): a CUDA graph of a step recorded before that must not be replayed (control.py)
    self._launch_epoch = 0
    self._env_model_names, self._env_rows, self.env_model = (), None, None
    self._upload_model()
    self.data = _Data()
    self._io = _lib.IO()
    self._applied_dirty = False
    self._applied_on = False
    want = None if outputs == 'all' else set(outputs) | {'warning'}
    for f in DATA_FIELDS.values():
      # the applied forces are allocated by enable_applied_forces(): writing to them before that must fail loudly, not be ignored
      if f.role == STATE or (f.role == OUTPUT and (want is None or f.name in want)):
        self._alloc(f)
    self._bind_io()
    self._warn_seen = torch.zeros((self.batch, 8), dtype=torch.int32, device=self.device)
    self.reset()

  @property
  def named(self):
    """Named indexing (`physics.named.data.xpos['torso', 'z']`), batched: see dm_control_b200/index.py."""
    if getattr(self, '_named', None) is None:
      from . import index
      self._named = index.NamedIndexStructs(self)
    return self._named

  # ---- construction helpers (reference: engine.py:451-503) -------------------------------------------
  @classmethod
  def from_xml_string(cls, xml_string, assets=None, **kw):
    return cls(mjcf_compile.compile_xml(xml_string, assets=assets), **kw)

  @classmethod
  def from_xml_path(cls, path, **kw):
    return cls(mjcf_compile.compile_file(path), **kw)

  def _upload_model(self):
    self._pos_current = False
    self._launch_epoch += 1
    if self._handle:
      self._L.b200mj_model_destroy(self._handle)
      self._handle = ctypes.c_void_p()
    with torch.cuda.device(self.device):
      idata, rdata = self.model.pack()
      self._blob = (idata, rdata)
      _lib.check(self._L.b200mj_model_create(
          idata.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), idata.size,
          rdata.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), rdata.size, ctypes.byref(self._handle)))
    self._model_version = self.model._version
    self._model_flags_version = self.model._flags_version
    self._apply_variable_geoms()       # a re-uploaded model forgets its per-environment geom list
    self._apply_env_model()            # and its per-environment model fields

  def _alloc(self, f):
    setattr(self.data, f.name, torch.zeros((self.batch,) + f.shape(self.model), dtype=f.dtype, device=self.device))

  def _bind_io(self):
    self._launch_epoch += 1
    for name, ctype in _lib.IO_FIELDS:
      t = getattr(self.data, name, None)
      if t is None or t.numel() == 0 or (name in APPLIED_FIELDS and not self._applied_on):
        setattr(self._io, name, ctypes.cast(None, ctype))
      else:
        setattr(self._io, name, ctypes.cast(t.data_ptr(), ctype))

  def _state_fields(self):
    """The fields that carry an environment's state: pickled, copied, and uploaded by every call."""
    return STATE_FIELDS + (APPLIED_FIELDS if self._applied_on else ())

  def enable_applied_forces(self, on=True):
    """Allocate `data.qfrc_applied` [B, nv] / `data.xfrc_applied` [B, nbody, 6] and route them into every step (the
    reference's arrays always act; here they are opt-in — two HBM reads per physics step and the fused kernel instead
    of the split path — and do not exist until enabled, so a write without this call raises AttributeError)."""
    self._pos_current = False
    self._applied_on = bool(on)
    for name in APPLIED_FIELDS:
      if on and getattr(self.data, name, None) is None:
        self._alloc(DATA_FIELDS[name])
    self._bind_io()

  def free(self):
    if getattr(self, '_handle', None):
      self._L.b200mj_model_destroy(self._handle)
      self._handle = ctypes.c_void_p()

  def __del__(self):
    try:
      self.free()
    except Exception:
      pass

  # ---- engine calls -----------------------------------------------------------------------------------
  def _stream(self):
    return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

  def _flags(self):
    f = 0
    if self.legacy_step:
      f |= _lib.STEP_LEGACY
    if self._full_final:
      f |= _lib.STEP_FULL_FINAL
    if self._sensors:
      f |= _lib.STEP_SENSORS
    if self._pos_current:
      f |= _lib.STEP_REUSE_POS
    return f

  # ---- pickling (reference: engine.py:287-304 copy / 370-378 __getstate__: model + data travel, the handle is rebuilt) ----
  def __getstate__(self):
    state = {n: getattr(self.data, n).cpu() for n in self._state_fields()}
    var = getattr(self, '_var_geom_ids', None)
    if var is not None:
      state['var_geom_pos'] = self.data.var_geom_pos.cpu(); state['var_geom_size'] = self.data.var_geom_size.cpu()
    st = dict(model=self.model, batch=self.batch, device=str(self.device), sensors=self._sensors, full_final=self._full_final,
              legacy_step=self.legacy_step, check_errors=self.check_errors, applied=self._applied_on, var_geom_ids=var, state=state,
              outputs=[n for n in DATA_FIELDS if hasattr(self.data, n)])
    if self._env_model_names:
      st['env_model'] = (self._env_model_names, self._env_rows.cpu())
    return st

  def __setstate__(self, st):
    self.__init__(st['model'], batch=st['batch'], device=st['device'], outputs=st['outputs'], sensors=st['sensors'],
                  full_final=st['full_final'])
    self.legacy_step, self.check_errors = st['legacy_step'], st['check_errors']
    if st['applied']:
      self.enable_applied_forces(True)
    if st['var_geom_ids'] is not None:
      self.set_variable_geoms(st['var_geom_ids'])
    if 'env_model' in st:
      names, rows = st['env_model']
      self.set_env_model_fields(names)
      self._env_rows.copy_(rows.to(self.device))
    for n, t in st['state'].items():
      getattr(self.data, n).copy_(t.to(self.device))
    self.forward()

  def _sync_model(self):
    if self.model._version != self._model_version:
      self._upload_model()
    elif self.model._flags_version != self._model_flags_version:
      _lib.check(self._L.b200mj_model_set_disableflags(self._handle, int(self.model.opt.disableflags)))
      self._launch_epoch += 1
      self._model_flags_version = self.model._flags_version

  def copy(self, share_model=False):
    """A new BatchedPhysics with the same model and a copy of the batched state (reference: engine.py:287-304)."""
    other = type(self)(self.model if share_model else self.model.copy(), batch=self.batch, device=self.device,
                       sensors=self._sensors, full_final=self._full_final)
    other.legacy_step = self.legacy_step
    other.check_errors = self.check_errors
    if self._applied_on:
      other.enable_applied_forces(True)
    if self._env_model_names:
      other.set_env_model_fields(self._env_model_names)
      other._env_rows.copy_(self._env_rows)
    for name in self._state_fields():
      getattr(other.data, name).copy_(getattr(self.data, name))
    other.forward()
    return other

  def step(self, nstep=1):
    """Advance all environments by `nstep` physics steps (reference: engine.py:164-176).

    With `legacy_step` (default) the state is advanced `nstep` times and position/velocity dependent fields are
    then refreshed for the new state (step2, (step1+step2)*(nstep-1), step1 — engine.py:147-162); acceleration
    stage outputs are those of the last step2.
    """
    self._sync_model()
    with self.check_invalid_state():
      with torch.cuda.device(self.device):
        _lib.check(self._L.b200mj_step(self._handle, ctypes.byref(self._io), self.batch, int(nstep), self._flags(),
                                       self._stream()))
    self._pos_current = bool(self.legacy_step and self._full_final and nstep >= 1)

  def bind(self, kind, names):
    """Batched counterpart of `mjcf.Physics.bind` (dm_control/mjcf/physics.py:516-652): attribute access to the model
    and data rows of the named elements, prefix-free; state writes mark the physics dirty and the next derived read
    runs `forward()` lazily. See dm_control_b200/binding.py."""
    from . import binding
    return binding.Binding(self, kind, names)

  def render(self, height=240, width=320, camera_id=-1, depth=False, segmentation=False, **unsupported):
    """`Physics.render` (engine.py:178-233), batched: [B,H,W,3] uint8 rgb, [B,H,W] float32 depth or [B,H,W,2] int32
    segmentation of every environment, on the device (dm_control_b200/render.py; a ray caster, not MuJoCo's GL renderer:
    overlays, scene options / callbacks and render flags are refused)."""
    from . import render as _render
    bad = [k for k, v in unsupported.items() if v]
    if bad:
      raise NotImplementedError(f'{bad} need MuJoCo\'s OpenGL renderer and are outside the rendering hand-off')
    return _render.Camera(self, height=height, width=width, camera_id=camera_id).render(depth=depth, segmentation=segmentation)

  @property
  def is_dirty(self):
    return bool(getattr(self, '_bind_dirty', False))

  def mark_as_dirty(self):
    """The state tensors were written directly: the next step() recomputes the position stage first."""
    self._pos_current = False

  def forward(self, extra_disableflags=0):
    """mj_forward on every environment (reference: engine.py:335-343)."""
    self._pos_current = False
    self._bind_dirty = False
    self._sync_model()
    with self.check_invalid_state():
      with torch.cuda.device(self.device):
        _lib.check(self._L.b200mj_forward(self._handle, ctypes.byref(self._io), self.batch, int(extra_disableflags),
                                          _lib.STEP_SENSORS if self._sensors else 0, self._stream()))

  def step_host(self, ctrl_host, obs_dev, obs_host, nstep=1):
    """End-to-end step with HOST buffers: pinned numpy/torch ctrl in, packed observation tensor out."""
    self._sync_model()
    nobs = obs_dev.shape[1]
    with torch.cuda.device(self.device):
      _lib.check(self._L.b200mj_step_host(
          self._handle, ctypes.byref(self._io), self.batch, int(nstep), self._flags(),
          ctypes.c_void_p(ctrl_host.data_ptr()), ctypes.c_void_p(self.data.ctrl.data_ptr()),
          ctypes.c_void_p(obs_dev.data_ptr()), ctypes.c_void_p(obs_host.data_ptr()), nobs, self._stream()))
    self._pos_current = bool(self.legacy_step and self._full_final and nstep >= 1)

  # ---- reference Physics API ----------------------------------------------------------------------------
  def set_control(self, control):
    """Reference: engine.py:139-145 (`np.copyto(self.data.ctrl, control)`)."""
    c = torch.as_tensor(control, dtype=torch.float64, device=self.device)
    self.data.ctrl.copy_(c.expand_as(self.data.ctrl))

  def _mask_ptr(self, env_mask):
    """Device pointer of a [B] uint8 mask (None -> NULL = every environment); keeps the tensor alive on `self`."""
    if env_mask is None:
      self._mask_keep = None
      return ctypes.c_void_p(None)
    self._mask_keep = torch.as_tensor(env_mask, device=self.device).to(torch.uint8).contiguous()
    return ctypes.c_void_p(self._mask_keep.data_ptr())

  def reset(self, keyframe_id=None, env_mask=None):
    """mj_resetData[Keyframe] + mj_forward with actuation disabled (reference: engine.py:306-327), for every
    environment or for those of `env_mask`; one b200mj_reset call (a state-reset launch + a masked forward launch):
    the environments outside the mask keep their state AND their outputs."""
    m, d = self.model, self.data
    if keyframe_id is not None and not 0 <= keyframe_id < m.nkey:
      raise ValueError(f'`keyframe_id` must be between 0 and {m.nkey}, got: {keyframe_id}')
    self._pos_current = False
    self._sync_model()
    if env_mask is None:
      for name in APPLIED_FIELDS + ('sensordata', 'actuator_force', 'qacc'):
        t = getattr(d, name, None)
        if t is not None:
          t.zero_()
      if hasattr(d, 'warning'):
        d.warning.zero_()
        self._warn_seen.zero_()
    else:
      mask = torch.as_tensor(env_mask, dtype=torch.bool, device=self.device)
      for name in APPLIED_FIELDS:      # mj_resetData clears the applied forces of the reset environments too
        t = getattr(d, name, None)
        if t is not None:
          t[mask] = 0
    with self.suppress_physics_errors():   # reference swallows errors here too (control.py:248-251)
      with self.check_invalid_state():
        with torch.cuda.device(self.device):
          _lib.check(self._L.b200mj_reset(self._handle, ctypes.byref(self._io), self.batch, self._mask_ptr(env_mask),
                                          -1 if keyframe_id is None else int(keyframe_id), self._stream()))

  def after_reset(self, env_mask=None):
    """Reference: engine.py:329-333 (mj_forward with actuation disabled); `env_mask` restricts it to the environments
    being reset, leaving the others' outputs untouched."""
    if env_mask is None:
      return self.forward(extra_disableflags=DSBL_ACTUATION)
    self._pos_current = False
    self._sync_model()
    with self.check_invalid_state():
      with torch.cuda.device(self.device):
        _lib.check(self._L.b200mj_forward_masked(self._handle, ctypes.byref(self._io), self.batch, self._mask_ptr(env_mask),
                                                 DSBL_ACTUATION, _lib.STEP_SENSORS if self._sensors else 0, self._stream()))

  def contact_force(self, contact_id):
    """`mj_contactForce` (reference: mujoco/wrapper/core.py:546-551) for contact `contact_id` of every environment:
    [B, 6] force and torque in the contact frame (zeros where an environment has fewer contacts)."""
    out = torch.zeros(self.batch, 6, dtype=torch.float64, device=self.device)
    with torch.cuda.device(self.device):
      _lib.check(self._L.b200mj_contact_force(self._handle, ctypes.byref(self._io), self.batch, int(contact_id),
                                              ctypes.c_void_p(out.data_ptr()), self._stream()))
    return out

  def subtree_vel(self):
    """`mj_subtreeVel` on the current state (reference: locomotion/walkers/legacy_base.py:179-186): refreshes
    `data.subtree_linvel` (and the other position / velocity-stage outputs) without integrating. After `step()` in the
    legacy ordering they are current already — this is for states written by hand."""
    self._sync_model()
    with torch.cuda.device(self.device):
      _lib.check(self._L.b200mj_subtree_vel(self._handle, ctypes.byref(self._io), self.batch, self._flags() & ~_lib.STEP_REUSE_POS,
                                            self._stream()))
    self._pos_current = False

  def set_variable_geoms(self, geom_ids):
    """Per-environment geoms: `data.var_geom_pos / var_geom_size` [B, n, 3] replace `model.geom_pos / geom_size` of the
    listed geoms (initialised from the model). The composer corridor arenas re-draw their wall / platform boxes every
    episode and the reference recompiles (composer/environment.py:378-383); here the environments share one topology."""
    ids = np.ascontiguousarray(geom_ids, dtype=np.int32)
    m, B = self.model, self.batch
    self._var_geom_ids = ids
    gp = torch.as_tensor(m.geom_pos[ids], device=self.device)
    gs = torch.as_tensor(m.geom_size[ids], device=self.device)
    self.data.var_geom_pos = gp[None].repeat(B, 1, 1).contiguous()
    self.data.var_geom_size = gs[None].repeat(B, 1, 1).contiguous()
    self._apply_variable_geoms()
    self._bind_io()
    self._pos_current = False

  def _apply_variable_geoms(self):
    self._launch_epoch += 1
    ids = getattr(self, '_var_geom_ids', None)
    if ids is not None:
      _lib.check(self._L.b200mj_model_set_variable_geoms(self._handle, ids.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), int(ids.size)))

  def set_env_model_fields(self, names):
    """Per-environment model fields: each environment reads the listed model fields (of ENV_MODEL_FIELDS) from its
    own row of one `[B, row]` float64 device buffer instead of the shared model. `physics.env_model.<field>` is the
    `[B, *model.<field>.shape]` view of that buffer; `bind(kind, names).<attr>` and `named.model.<field>` read and write
    it for these fields. Fields already per-environment keep their rows; the others start from the model's current
    values. `set_env_model_fields(())` turns the feature off.

    The reference sets these per `Physics`, e.g. `PhysicsVariator.apply_variations` (composer/variation/__init__.py:90-136);
    here each environment is one `Physics`. An environment then steps exactly as a BatchedPhysics on a copy of the model
    with its values written through `model.set`: nothing derived is recomputed (body_subtreemass, the invweight0 tables,
    stat.meaninertia, the actuator moments keep the shared model's values), and an environment whose `dof_damping` row
    has a positive entry takes mj_Euler's implicit damping update. While a field is per-environment, its rows are what
    the engine uses: a write to the shared model's field still re-uploads the model but does not reach the rows. A
    direct in-place write to `env_model.*` is like one to `data.qpos`: call `forward()` or `mark_as_dirty()` before
    the next step (writes through `bind` and `named.model` do this)."""
    names = tuple(names)
    check_env_model_fields(names)
    m, B = self.model, self.batch
    parts = []
    for n in names:
      if n in self._env_model_names:
        parts.append(getattr(self.env_model, n).reshape(B, -1))
      else:
        parts.append(torch.as_tensor(np.asarray(m.fields[n], dtype=np.float64).reshape(1, -1), device=self.device).expand(B, -1))
    if names:
      self._env_rows = torch.cat(parts, dim=1).contiguous()
      self.env_model, o = types.SimpleNamespace(), 0
      for n in names:
        k = m.fields[n].size
        setattr(self.env_model, n, self._env_rows[:, o:o + k].view((B,) + m.fields[n].shape))
        o += k
    else:
      self._env_rows, self.env_model = None, None
    self._env_model_names = names
    self._apply_env_model()
    self._pos_current = False

  @property
  def env_model_fields(self):
    """The model fields that are per-environment (set_env_model_fields), in row order."""
    return self._env_model_names

  def _apply_env_model(self):
    self._launch_epoch += 1
    names = self._env_model_names
    ids = np.array([_FIELD_ID[n] for n in names], dtype=np.int32)
    rows = ctypes.c_void_p(self._env_rows.data_ptr() if names else None)
    _lib.check(self._L.b200mj_model_set_env_fields(self._handle, ids.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), len(names),
                                                    rows, self.batch if names else 0))

  @contextlib.contextmanager
  def reset_context(self):
    """Reference: rl/control.py:232-253."""
    try:
      self.reset()
    except PhysicsError:
      pass
    yield self
    self.after_reset()

  def time(self):
    return self.data.time

  def timestep(self):
    return self.model.opt.timestep

  def control(self):
    return self.data.ctrl

  def position(self):
    return self.data.qpos

  def velocity(self):
    return self.data.qvel

  def activation(self):
    return self.data.act

  def get_state(self):
    """[B, nq+nv+na] (reference: engine.py:235-250 / :567-585)."""
    d = self.data
    return torch.cat([d.qpos, d.qvel, d.act], dim=1)

  def set_state(self, physics_state):
    m, d = self.model, self.data
    s = torch.as_tensor(physics_state, dtype=torch.float64, device=self.device)
    if s.shape[-1] != m.nq + m.nv + m.na:
      raise ValueError(f'Input physics state has shape {tuple(s.shape)}. Expected (..., {m.nq + m.nv + m.na}).')
    s = s.expand(self.batch, -1)
    d.qpos.copy_(s[:, :m.nq])
    d.qvel.copy_(s[:, m.nq:m.nq + m.nv])
    d.act.copy_(s[:, m.nq + m.nv:])
    self._pos_current = False

  # ---- warnings -> PhysicsError (reference: engine.py:345-368) -----------------------------------------
  @contextlib.contextmanager
  def suppress_physics_errors(self):
    prev = self._suppress
    self._suppress = True
    try:
      yield
    finally:
      self._suppress = prev

  check_errors = True   # set False on the throughput path: skips the device->host sync of the warning counters

  @contextlib.contextmanager
  def check_invalid_state(self):
    yield
    if not self.check_errors or not hasattr(self.data, 'warning'):
      return
    new = self.data.warning - self._warn_seen
    if bool((new > 0).any()):
      self._warn_seen.copy_(self.data.warning)
      which = (new > 0).any(dim=0).cpu().numpy()
      names = [n for n, w in zip(_WARNING_NAMES, which) if w]
      message = _INVALID_PHYSICS_STATE.format(warning_names=', '.join(names))
      if self._suppress:
        return
      raise PhysicsError(message)

  def check_divergence(self):
    """Reference: rl/control.py:255-267 (abstract) — raise if any state value is not finite."""
    d = self.data
    ok = torch.isfinite(d.qpos).all() & torch.isfinite(d.qvel).all() & torch.isfinite(d.qacc_warmstart).all()
    if not bool(ok):
      raise PhysicsError('Physics state has diverged (non-finite qpos/qvel).')

  # ---- instrumentation ------------------------------------------------------------------------------------
  def workspace_bytes(self):
    return int(self._L.b200mj_workspace_bytes(self._handle))

  def describe(self):
    """Kernel workspaces of this model (fused / position / acceleration row-buckets), as a dict."""
    import json
    buf = ctypes.create_string_buffer(2048)
    _lib.check(self._L.b200mj_describe(self._handle, buf, 2048))
    return json.loads(buf.value.decode())

  def envs_per_block(self):
    return int(self._L.b200mj_envs_per_block(self._handle))
