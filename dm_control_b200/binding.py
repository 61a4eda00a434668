"""`physics.bind(kind, names)`: the batched counterpart of `mjcf.Physics.bind` (dm_control/mjcf/physics.py:209-237,516-652).

The reference binds `mjcf.Element`s; the PyMJCF object model is out of scope here, so elements are named by
`(kind, names)` — `physics.bind('body', ['rradius', 'lradius']).xpos`, `physics.bind('joint', 'rfemurrx').qpos = 0.3`,
`physics.bind('geom', 'wall_3').pos`. What carries over is the contract:

  * one attribute namespace per element kind with the type prefix removed (`geom_pos` -> `.pos`, `body_mass` -> `.mass`,
    `jnt_range` -> `.range`, `actuator_gear` -> `.gear`; a joint's `.damping` / `.armature` are the dof_damping /
    dof_armature columns of its dofs, ragged like its `qvel`), data fields by their own name (`xpos`, `qpos`, `qvel`, `ctrl`,
    `sensordata`, `subtree_linvel`, ...), `element_id`;
  * ragged fields resolve through the address tables (`qpos`/`qvel` of a joint, `sensordata` of a sensor);
  * writes to the STATE through a binding (the fields `physics.DATA_FIELDS` marks STATE) mark the physics dirty, and the
    next read of a DERIVED field through any binding runs `forward()` first — lazily, once
    (mjcf/physics.py:211-237 `_triggers_dirty` / `is_dirty`). Model writes re-upload the model before the next call.

Every value has the leading batch axis: `bind('body', names).xpos` is `[B, len(names), 3]` (or `[B, 3]` for one name).
"""
from __future__ import annotations

import numpy as np
import torch

from . import index
from .physics import DATA_FIELDS, STATE

_PREFIX = dict(body='body_', geom='geom_', site='site_', joint='jnt_', actuator='actuator_', sensor='sensor_', tendon='tendon_',
               dof='dof_')
# model fields a joint reaches through its dofs (mjcf/physics.py binds a joint's `damping` / `armature` to dof_damping /
# dof_armature the same way): ragged, one column per dof of the bound joints
_MODEL_ALIAS = {'joint': {'damping': 'dof_damping', 'armature': 'dof_armature'}}
_DATA_ALIAS = {'geom': {'xpos': 'geom_xpos', 'xmat': 'geom_xmat'}, 'site': {'xpos': 'site_xpos', 'xmat': 'site_xmat'},
               'actuator': {'force': 'actuator_force'}}


def model_field(kind, attr):
  """The model field behind attribute `attr` of a bound `kind` element."""
  return _MODEL_ALIAS.get(kind, {}).get(attr, _PREFIX[kind] + attr)


def model_rows(model, kind, field, ids):
  """(ragged, rows of `field` that belong to the elements `ids` of `kind`): a joint's dofs for the dof fields."""
  if field.startswith('dof_') and kind == 'joint':
    slices = index._ragged(model, 'nv')
    return True, [c for i in ids for c in range(slices[i].start, slices[i].stop)]
  return False, [int(i) for i in ids]


class Binding:

  def __init__(self, physics, kind, names):
    object.__setattr__(self, '_p', physics)
    object.__setattr__(self, '_kind', kind)
    single = isinstance(names, str)
    names = [names] if single else list(names)
    m = physics.model
    ids = np.array([m.name2id(n, kind) for n in names], dtype=np.int64)
    object.__setattr__(self, '_single', single)
    object.__setattr__(self, 'element_id', int(ids[0]) if single else ids)
    object.__setattr__(self, '_ids', ids)
    object.__setattr__(self, '_tids', torch.as_tensor(ids, device=physics.device))

  # ---- helpers ----
  def _index(self, name, field):
    """(ragged, indices along axis 1 of `data.<field>`) of the bound elements: the columns of their slices of a ragged
    field (the slices `physics.named` uses), or their rows of a per-element field."""
    rows = DATA_FIELDS[field].rows if field in DATA_FIELDS else None
    if rows in index._RAGGED_AXES and index._RAGGED_AXES[rows][0] == self._kind:
      slices = index._ragged(self._p.model, rows)
      cols = [c for i in self._ids if slices[i] is not None for c in range(slices[i].start, slices[i].stop)]
      return True, torch.tensor(cols, dtype=torch.int64, device=self._p.device)
    if rows == self._kind:
      return False, self._tids
    raise AttributeError(f'{name!r} is not a per-{self._kind} data field')

  def _data_field(self, name):
    d = self._p.data
    name = _DATA_ALIAS.get(self._kind, {}).get(name, name)
    t = getattr(d, name, None)
    return (name, t) if isinstance(t, torch.Tensor) else (name, None)

  def _env_rows(self, mname):
    """[B, n, w] view of a per-environment model field (physics.set_env_model_fields)."""
    t = getattr(self._p.env_model, mname)
    return t.reshape(t.shape[0], t.shape[1], -1)

  def _squeeze(self, t):
    return t[:, 0] if self._single and t.dim() >= 2 else t

  # ---- attribute access ----
  def __getattr__(self, name):
    p = self._p
    field, t = self._data_field(name)
    if t is not None:
      ragged, idx = self._index(name, field)
      if DATA_FIELDS[field].role != STATE and getattr(p, '_bind_dirty', False):
        p.forward()                              # lazily, once: derived quantities after a state write through a binding
      out = t.index_select(1, idx)
      return out if ragged else self._squeeze(out)
    mname = model_field(self._kind, name)
    if mname in getattr(p, 'env_model_fields', ()):          # per-environment model field: [B, k(, w)]
      ragged, rows = model_rows(p.model, self._kind, mname, self._ids)
      out = self._env_rows(mname)[:, torch.as_tensor(rows, dtype=torch.int64, device=p.device)]
      out = out[..., 0] if out.shape[2] == 1 else out
      return out if ragged else self._squeeze(out)
    arr = p.model.fields.get(mname)
    if arr is None:
      raise AttributeError(f'bound {self._kind} has no attribute {name!r}')
    ragged, idx = model_rows(p.model, self._kind, mname, self._ids)
    if ragged:
      return np.asarray(arr)[idx]
    n = len(p.model.ordered_names[self._kind]) if self._kind in p.model.ordered_names else arr.shape[0]
    rows = np.asarray(arr).reshape(n, -1)[idx]
    rows = rows[:, 0] if rows.shape[1] == 1 else rows
    return rows[0] if self._single else rows

  def __setattr__(self, name, value):
    p = self._p
    field, t = self._data_field(name)
    if t is not None:
      v = torch.as_tensor(value, dtype=t.dtype, device=p.device)
      ragged, idx = self._index(name, field)
      if ragged:
        t[:, idx] = v
      else:
        view = t.reshape(p.batch, t.shape[1], -1)
        view[:, idx] = v.reshape((-1, len(self._ids), view.shape[2])) if v.numel() > view.shape[2] * len(self._ids) or v.dim() >= 2 \
            else v.reshape(1, -1, view.shape[2]).expand(p.batch, len(self._ids), view.shape[2])
      if DATA_FIELDS[field].role == STATE:
        p.mark_as_dirty()
        if field != 'ctrl':                      # ctrl does not invalidate position / velocity-stage quantities
          object.__setattr__(p, '_bind_dirty', True)
      return
    mname = model_field(self._kind, name)
    if mname in getattr(p, 'env_model_fields', ()):          # per-environment model field: [B, k, w], [k, w] or a scalar
      rows = self._env_rows(mname)
      _, idx = model_rows(p.model, self._kind, mname, self._ids)
      tidx = torch.as_tensor(idx, dtype=torch.int64, device=p.device)
      k, w = len(idx), rows.shape[2]
      v = torch.as_tensor(value, dtype=rows.dtype, device=p.device)
      n = v.numel()
      shape = (p.batch, k, w) if n == p.batch * k * w and n != k * w else (1, k, w) if n == k * w else (1, 1, w) if n == w else (1, 1, 1)
      if n != shape[0] * shape[1] * shape[2]:
        raise ValueError(f'{name!r}: cannot write a value of shape {tuple(v.shape)} to [{p.batch}, {k}, {w}]')
      rows[:, tidx] = v.reshape(shape).expand(p.batch, k, w)
      p.mark_as_dirty()
      object.__setattr__(p, '_bind_dirty', True)
      return
    if mname not in p.model.fields:
      raise AttributeError(f'bound {self._kind} has no attribute {name!r}')
    arr = p.model.fields[mname]
    ragged, idx = model_rows(p.model, self._kind, mname, self._ids)
    if ragged:
      arr[idx] = np.asarray(value, dtype=arr.dtype)
      p.model.touch()
      object.__setattr__(p, '_bind_dirty', True)
      return
    n = len(p.model.ordered_names[self._kind])
    arr.reshape(n, -1)[self._ids] = np.asarray(value, dtype=arr.dtype).reshape(len(self._ids), -1) if np.ndim(value) else value
    p.model.touch()
    object.__setattr__(p, '_bind_dirty', True)
