"""Named indexing on batched tensors: `physics.named.data.xpos['torso', 'z']`, `named.data.qpos['root']`, ...

Batched twin of `dm_control/mujoco/index.py` (row names from the model's name tables, ragged `nq/nv/na/
nsensordata` axes via `jnt_qposadr/jnt_dofadr/actuator_actadr/sensor_adr` — index.py:94-100 — and the column names
`x y z`, `qw qx qy qz`, `xx … zz` — index.py:103-175). Every field keeps its leading batch axis: an indexing
expression that yields shape `S` in the reference yields `[B, *S]` here. Model-side fields (`named.model.*`) are
unbatched numpy arrays and index exactly as in the reference, except the per-environment model fields
(`physics.set_env_model_fields`), which index the batched `physics.env_model.<field>` tensor with its leading batch axis.
"""
from __future__ import annotations

import numpy as np
import torch

from .model import MODEL_FIELDS
from .physics import DATA_FIELDS

_COLS = {'xyz': ['x', 'y', 'z'], 'quat': ['qw', 'qx', 'qy', 'qz'], 'mat': ['xx', 'xy', 'xz', 'yx', 'yy', 'yz', 'zx', 'zy', 'zz'],
         'rgba': ['r', 'g', 'b', 'a']}
_FIELDS = {**MODEL_FIELDS, **DATA_FIELDS}
# field -> kind of its column names; the visual tables (Model.vis) are not blob fields
_COL_KIND = {**dict.fromkeys(('geom_rgba', 'site_rgba', 'mat_rgba'), 'rgba'),      # index.py:103-175 `rgba`
             **{n: f.cols for n, f in _FIELDS.items() if f.cols}}
# field -> kind of its row axis
_ROW_KIND = {
    **{f: 'geom' for f in ('geom_rgba', 'geom_group')}, **{f: 'site' for f in ('site_rgba', 'site_group')},
    **{f: 'camera' for f in ('cam_pos', 'cam_quat', 'cam_fovy', 'cam_bodyid', 'cam_mode', 'cam_targetbodyid')},
    'mat_rgba': 'material',
    **{n: f.rows for n, f in _FIELDS.items() if f.rows},
}

# ragged axis -> (element kind that owns its slices, address table)
_RAGGED_AXES = {'nq': ('joint', 'jnt_qposadr'), 'nv': ('joint', 'jnt_dofadr'), 'na': ('actuator', 'actuator_actadr'),
               'nsensordata': ('sensor', 'sensor_adr')}


def _ragged(model, axis):
  """Slice of every element along a ragged axis, in element order (index.py:245-267); None for an actuator without an
  activation (an `na` slice is one column)."""
  adr = [int(a) for a in getattr(model, _RAGGED_AXES[axis][1])]
  if axis == 'na':
    return [slice(a, a + 1) if a >= 0 else None for a in adr]
  return [slice(a, b) for a, b in zip(adr, adr[1:] + [getattr(model, axis)])]


class FieldIndexer:
  """One field with name-aware `__getitem__` / `__setitem__` (index.py:455-600)."""

  def __init__(self, name, array, model, batched, on_write=None):
    self._name, self._a, self._batched, self._on_write = name, array, batched, on_write
    kind = _ROW_KIND.get(name)
    if kind in _RAGGED_AXES:
      names = model.ordered_names[_RAGGED_AXES[kind][0]]
      self._rows = {n: s for n, s in zip(names, _ragged(model, kind)) if s is not None}
    else:
      self._rows = dict(model.names.get(kind, {}))       # name -> id
    self._cols = {c: i for i, c in enumerate(_COLS.get(_COL_KIND.get(name), []))}

  def _row_key(self, k):
    if isinstance(k, str):
      if k not in self._rows:
        raise IndexError(f'{k!r} is not a valid row name for field {self._name!r}; valid: {sorted(self._rows)[:8]}...')
      return self._rows[k]
    if isinstance(k, (list, tuple)) and k and all(isinstance(x, str) for x in k):
      idx = []
      for x in k:
        r = self._row_key(x)
        idx.extend(range(r.start, r.stop) if isinstance(r, slice) else [r])
      return idx
    return k

  def _col_key(self, k):
    if isinstance(k, str):
      if k not in self._cols:
        raise IndexError(f'{k!r} is not a valid column name for field {self._name!r}')
      return self._cols[k]
    if isinstance(k, (list, tuple)) and k and all(isinstance(x, str) for x in k):
      return [self._col_key(x) for x in k]
    return k

  def _translate(self, key):
    if not isinstance(key, tuple):
      key = (key,)
    out = [self._row_key(key[0])] + ([self._col_key(key[1])] if len(key) > 1 else []) + list(key[2:])
    if len(out) == 2 and isinstance(out[0], list) and isinstance(out[1], list):
      out = [np.asarray(out[0])[:, None], np.asarray(out[1])[None, :]]     # outer indexing, as np.ix_ in the reference
    return tuple([slice(None)] + out) if self._batched else tuple(out)

  def __getitem__(self, key):
    return self._a[self._translate(key)]

  def __setitem__(self, key, value):
    k = self._translate(key)
    if isinstance(self._a, torch.Tensor):
      self._a[k] = torch.as_tensor(value, dtype=self._a.dtype, device=self._a.device)
      if self._on_write is not None:
        self._on_write()          # per-environment model field: the next step recomputes the position stage
    else:
      self._a[k] = value
      if self._on_write is not None:
        self._on_write()          # model field: the device copy must be refreshed before the next step

  @property
  def row_names(self):
    return list(self._rows)

  def __repr__(self):
    return f'FieldIndexer({self._name}, rows={len(self._rows)}, shape={tuple(self._a.shape)})'


class _Struct:
  def __init__(self, getter, model, batched, dirty=None):
    object.__setattr__(self, '_dirty', dirty)
    object.__setattr__(self, '_g', getter)
    object.__setattr__(self, '_m', model)
    object.__setattr__(self, '_b', batched)
    object.__setattr__(self, '_cache', {})

  def __getattr__(self, name):
    arr = self._g(name)
    if arr is None:
      raise AttributeError(name)
    c = self._cache.get(name)
    if c is None or c._a is not arr:
      env = not self._b and isinstance(arr, torch.Tensor)      # a per-environment model field
      c = FieldIndexer(name, arr, self._m, self._b or env, on_write=self._dirty if env else None if self._b else self._m.touch)
      self._cache[name] = c
    return c


class NamedIndexStructs:
  """`physics.named` (engine.py:427-430): `.data.<field>[names]` on `[B, ...]` tensors, `.model.<field>[names]` on numpy."""

  def __init__(self, physics):
    m = physics.model

    def model_get(name):
      if name in getattr(physics, 'env_model_fields', ()):
        return getattr(physics.env_model, name)
      a = m.fields.get(name)
      # colours, groups, cameras: visual tables outside the physics blob
      return a if a is not None else getattr(m, 'vis', {}).get(name)
    self.data = _Struct(lambda name: getattr(physics.data, name, None), m, True)
    self.model = _Struct(model_get, m, False, dirty=getattr(physics, 'mark_as_dirty', None))
