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
from .model import MODEL_FIELDS
from .physics import DATA_FIELDS, STATE

# model fields a joint reaches through its dofs (mjcf/physics.py binds a joint's `damping` / `armature` to dof_damping /
# dof_armature the same way): ragged, one column per dof of the bound joints
_MODEL_ALIAS = {'joint': {'damping': 'dof_damping', 'armature': 'dof_armature'}}
# (row axis, attribute) -> model field: `geom_pos` is a geom's `pos`, `jnt_range` a joint's `range`
_MODEL_ATTR = {(f.rows, n.split('_', 1)[1]): n for n, f in MODEL_FIELDS.items() if '_' in n}
_DATA_ALIAS = {'geom': {'xpos': 'geom_xpos', 'xmat': 'geom_xmat'}, 'site': {'xpos': 'site_xpos', 'xmat': 'site_xmat'},
               'actuator': {'force': 'actuator_force'}}


def model_field(kind, attr):
  """The model field behind attribute `attr` of a bound `kind` element (`<kind>_<attr>` where there is none)."""
  return _MODEL_ALIAS.get(kind, {}).get(attr) or _MODEL_ATTR.get((kind, attr), f'{kind}_{attr}')


def element_rows(model, axis, kind, ids):
  """(ragged, indices along row axis `axis` that belong to the elements `ids` of `kind`): the columns of their slices
  of a ragged axis (the slices `physics.named` uses), or their rows; None where `axis` is not `kind`'s."""
  if axis in index._RAGGED_AXES and index._RAGGED_AXES[axis][0] == kind:
    slices = index._ragged(model, axis)
    return True, [c for i in ids if slices[i] is not None for c in range(slices[i].start, slices[i].stop)]
  return (False, [int(i) for i in ids]) if axis == kind else None


def model_rows(model, kind, attr, ids):
  """(field, ragged, rows) of the model field behind attribute `attr` of the elements `ids` of `kind` (element_rows)."""
  field = model_field(kind, attr)
  found = field in MODEL_FIELDS and element_rows(model, MODEL_FIELDS[field].rows, kind, ids)
  if not found:
    raise AttributeError(f'bound {kind} has no attribute {attr!r}')
  return (field,) + found


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
  def _data(self, name):
    """(field, tensor, ragged, indices along axis 1) of the data field behind `name` for the bound elements
    (element_rows); None where `name` is no data field of this kind."""
    field = _DATA_ALIAS.get(self._kind, {}).get(name, name)
    t = getattr(self._p.data, field, None)
    found = (isinstance(t, torch.Tensor) and field in DATA_FIELDS and
             element_rows(self._p.model, DATA_FIELDS[field].rows, self._kind, self._ids))
    if not found:
      return None
    ragged, idx = found
    return field, t, ragged, torch.tensor(idx, dtype=torch.int64, device=self._p.device) if ragged else self._tids

  def _squeeze(self, t):
    return t[:, 0] if self._single and t.dim() >= 2 else t

  # ---- attribute access ----
  def __getattr__(self, name):
    p = self._p
    data = self._data(name)
    if data is not None:
      field, t, ragged, idx = data
      if DATA_FIELDS[field].role != STATE and getattr(p, '_bind_dirty', False):
        p.forward()                              # lazily, once: derived quantities after a state write through a binding
      out = t.index_select(1, idx)
      return out if ragged else self._squeeze(out)
    field, ragged, idx = model_rows(p.model, self._kind, name, self._ids)
    if field in getattr(p, 'env_model_fields', ()):          # per-environment model field: [B, k(, w)]
      out = getattr(p.env_model, field)[:, torch.as_tensor(idx, dtype=torch.int64, device=p.device)]
      return out if ragged else self._squeeze(out)
    out = p.model.fields[field][idx]
    return out[0] if self._single and not ragged else out

  def __setattr__(self, name, value):
    p = self._p
    data = self._data(name)
    if data is not None:
      field, t, ragged, idx = data
      v = torch.as_tensor(value, dtype=t.dtype, device=p.device)
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
    field, ragged, idx = model_rows(p.model, self._kind, name, self._ids)
    if field in getattr(p, 'env_model_fields', ()):          # per-environment model field: [B, k, w], [k, w] or a scalar
      rows = getattr(p.env_model, field)
      rows = rows.reshape(rows.shape[0], rows.shape[1], -1)    # [B, n, w]
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
    arr = p.model.fields[field]
    if ragged:
      arr[idx] = np.asarray(value, dtype=arr.dtype)
    else:                                        # [n, w]: k rows, or one row for all
      arr.reshape(arr.shape[0], -1)[idx] = np.asarray(value, dtype=arr.dtype).reshape(len(idx), -1) if np.ndim(value) else value
    p.model.touch()
    object.__setattr__(p, '_bind_dirty', True)
