"""`physics.bind(kind, names)`: the batched counterpart of `mjcf.Physics.bind` (dm_control/mjcf/physics.py:209-237,516-652).

The reference binds `mjcf.Element`s; the PyMJCF object model is out of scope here, so elements are named by
`(kind, names)` — `physics.bind('body', ['rradius', 'lradius']).xpos`, `physics.bind('joint', 'rfemurrx').qpos = 0.3`,
`physics.bind('geom', 'wall_3').pos`. What carries over is the contract:

  * one attribute namespace per element kind with the type prefix removed (`geom_pos` -> `.pos`, `body_mass` -> `.mass`,
    `jnt_range` -> `.range`, `actuator_gear` -> `.gear`), data fields by their own name (`xpos`, `qpos`, `qvel`, `ctrl`,
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
_DATA_ALIAS = {'geom': {'xpos': 'geom_xpos', 'xmat': 'geom_xmat'}, 'site': {'xpos': 'site_xpos', 'xmat': 'site_xmat'},
               'actuator': {'force': 'actuator_force'}}


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
    mname = _PREFIX[self._kind] + name
    arr = p.model.fields.get(mname)
    if arr is None:
      raise AttributeError(f'bound {self._kind} has no attribute {name!r}')
    n = len(p.model.ordered_names[self._kind]) if self._kind in p.model.ordered_names else arr.shape[0]
    rows = np.asarray(arr).reshape(n, -1)[self._ids]
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
    mname = _PREFIX[self._kind] + name
    if mname not in p.model.fields:
      raise AttributeError(f'bound {self._kind} has no attribute {name!r}')
    arr = p.model.fields[mname]
    n = len(p.model.ordered_names[self._kind])
    arr.reshape(n, -1)[self._ids] = np.asarray(value, dtype=arr.dtype).reshape(len(self._ids), -1) if np.ndim(value) else value
    p.model.touch()
    object.__setattr__(p, '_bind_dirty', True)
