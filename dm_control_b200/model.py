"""Compiled model container + blob packer.

`Model` stands where `dm_control.mujoco.wrapper.core.MjModel` stands in the reference
(dm_control/mujoco/wrapper/core.py:253-432): attribute access to MuJoCo-named model arrays
(`model.nq`, `model.jnt_range`, `model.opt.timestep`, `model.name2id(...)`), plus `pack()` which
produces the (idata, rdata) blob that crosses the C ABI (layout: include/b200mj_model_fields.h).
"""
from __future__ import annotations

import os
import re
import types
from typing import NamedTuple

import numpy as np

_HDR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'b200mj_model_fields.h')


def _parse_header():
  text = open(_HDR).read()
  body = text.split('#define B200MJ_MODEL_FIELDS(BMJ_I, BMJ_R)')[1].split('/* indices into `sizes` */')[0]
  body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
  fields = [(m.group(2), 'i' if m.group(1) == 'I' else 'r') for m in re.finditer(r'BMJ_([IR])\((\w+)\)', body)]

  def enum_names(tag):
    blk = re.search(r'enum %s \{(.*?)\};' % tag, text, flags=re.S).group(1)
    blk = re.sub(r'/\*.*?\*/', '', blk, flags=re.S)
    return [n.split('=')[0].strip() for n in blk.split(',') if n.strip()]
  sizes = enum_names('b200mj_size')
  optr = enum_names('b200mj_optr')
  opti = enum_names('b200mj_opti')
  return fields, sizes, optr, opti


FIELDS, _SIZES, _OPTR, _OPTI = _parse_header()
SIZE = {n[len('BMJ_'):]: i for i, n in enumerate(_SIZES[:-1])}
NSIZES = len(_SIZES) - 1
OPTR = {n[len('BMJ_OPT_'):]: i for i, n in enumerate(_OPTR[:-1])}
NOPTR = len(_OPTR) - 1
OPTI = {n[len('BMJ_OPT_'):]: i for i, n in enumerate(_OPTI[:-1])}
NOPTI = len(_OPTI) - 1


class ModelField(NamedTuple):
  """One blob field of the compiled model, in the header's order."""
  name: str
  dtype: type        # np.int32 or np.float64
  rows: str | None   # row axis: element kind ('body', ..., 'key'), ragged axis ('nq', 'nv'), unnamed count or None
  width: tuple = ()  # per-row shape: constants and model sizes by name
  cols: str | None = None   # column names of index.py: 'xyz' or 'quat'
  env: int | None = None    # position among the per-environment fields (ENV_FIELDS, csrc/b200mj.cu)

  def shape(self, m):
    count = () if self.rows is None else (getattr(m, _COUNT[self.rows]) if self.rows in _COUNT else -1,)
    return count + tuple(getattr(m, d) if isinstance(d, str) else d for d in self.width)


# row axis by name prefix where it is not the prefix itself (`body_pos` has one row per body, `pair_geom1` per pair)
_AXIS = dict(jnt='joint', dof='nv', eq='equality', qpos0='nq', qpos='nq', sizes=None, opt=None)
# the size that counts a row axis; the levels have none (`level_adr` has nlevel + 1 entries, `level_body` nbody)
_COUNT = dict(body='nbody', joint='njnt', geom='ngeom', site='nsite', actuator='nu', tendon='ntendon', equality='neq',
              sensor='nsensor', key='nkey', nq='nq', nv='nv', pair='npair', wrap='nwrap')
_XYZ, _QUAT, _W2, _W5 = dict(width=(3,), cols='xyz'), dict(width=(4,), cols='quat'), dict(width=(2,)), dict(width=(5,))
# how each field differs from one value per row
_DECLARED = {
    'sizes': dict(width=(NSIZES,)), 'opt_real': dict(width=(NOPTR,)), 'opt_int': dict(width=(NOPTI,)),
    'body_pos': _XYZ, 'body_quat': _QUAT, 'body_ipos': dict(_XYZ, env=2), 'body_iquat': _QUAT, 'body_mass': dict(env=0),
    'body_inertia': dict(_XYZ, env=1), 'body_invweight0': _W2, 'body_dofmask': _W2,
    'jnt_pos': _XYZ, 'jnt_axis': _XYZ, 'jnt_stiffness': dict(env=8), 'jnt_range': _W2, 'jnt_solref': _W2, 'jnt_solimp': _W5,
    'dof_armature': dict(env=7), 'dof_damping': dict(env=6), 'dof_solref': _W2, 'dof_solimp': _W5,
    'geom_size': _XYZ, 'geom_pos': _XYZ, 'geom_quat': _QUAT, 'geom_friction': dict(width=(3,), env=3),
    'geom_solref': dict(_W2, env=4), 'geom_solimp': dict(_W5, env=5),
    'site_pos': _XYZ, 'site_quat': _QUAT, 'site_size': _XYZ,
    'actuator_gainprm': dict(width=(3,), env=9), 'actuator_biasprm': dict(width=(3,), env=10), 'actuator_ctrlrange': _W2,
    'actuator_forcerange': _W2, 'actuator_actrange': _W2,
    'eq_data': dict(width=(11,)), 'eq_solref': _W2, 'eq_solimp': _W5,
    'key_qpos': dict(width=('nq',)),
}
MODEL_FIELDS = {name: ModelField(name, np.int32 if kind == 'i' else np.float64, _AXIS.get(prefix, prefix), **_DECLARED.get(name, {}))
                for name, kind in FIELDS for prefix in [name.split('_')[0]]}

# MuJoCo mjtObj names accepted by name2id/id2name (reference: wrapper/core.py:334-387)
_OBJ_ALIASES = dict(body='body', xbody='body', joint='joint', geom='geom', site='site', actuator='actuator',
                    tendon='tendon', sensor='sensor', equality='equality', key='key', camera='camera', light='light',
                    material='material', texture='texture', mesh='mesh', hfield='hfield', numeric='numeric', text='text',
                    tuple='tuple')
# sizes that are not part of the physics blob: counted from the name tables the compiler keeps for visual / custom elements
_NAME_SIZES = dict(ncam='camera', nlight='light', nmat='material', ntex='texture', nmesh='mesh', nhfield='hfield', nnumeric='numeric',
                   ntext='text', ntuple='tuple', nsensor='sensor', neq='equality', ntendon='tendon')


class _Opt:
  """`model.opt` view (timestep, gravity, integrator, disableflags, ...) backed by the packed arrays."""

  def __init__(self, model):
    object.__setattr__(self, '_m', model)

  def __getattr__(self, name):
    if name.startswith('_'):
      raise AttributeError(name)      # (unpickling probes dunder names before `_m` exists)
    m = self._m
    if name == 'gravity':
      return m.fields['opt_real'][OPTR['GRAVITY_X']:OPTR['GRAVITY_X'] + 3]
    key = name.upper()
    if key in OPTR:
      return float(m.fields['opt_real'][OPTR[key]])
    if key in OPTI:
      return int(m.fields['opt_int'][OPTI[key]])
    raise AttributeError(name)

  def __setattr__(self, name, value):
    m = self._m
    key = name.upper()
    if name == 'gravity':
      m.fields['opt_real'][OPTR['GRAVITY_X']:OPTR['GRAVITY_X'] + 3] = value
    elif key in OPTR:
      m.fields['opt_real'][OPTR[key]] = value
    elif key in OPTI:
      m.fields['opt_int'][OPTI[key]] = value
    else:
      raise AttributeError(name)
    if key == 'DISABLEFLAGS':
      m._flags_version += 1      # cheap path: the uploaded model only needs its flag word refreshed
    else:
      m._version += 1


class Model:
  """Compiled model: numpy tables keyed by MuJoCo field names."""

  def __init__(self, fields, names, ordered_names, vis=None):
    # visual-only tables (colours, groups, cameras, extent): rendering hand-off, never part of the physics blob
    self.vis = {k: np.asarray(v) for k, v in (vis or {}).items()}
    self.fields = {}
    for f in MODEL_FIELDS.values():     # `sizes` comes first: the other shapes read it
      arr = np.ascontiguousarray(fields[f.name], dtype=f.dtype)
      try:
        self.fields[f.name] = arr.reshape(f.shape(self))
      except ValueError:
        raise ValueError(f'model field {f.name!r}: {arr.size} values do not make its shape {f.shape(self)}') from None
    self.names = names
    self.ordered_names = ordered_names
    self.opt = _Opt(self)
    self._version = 0
    self._flags_version = 0

  # --- sizes ---------------------------------------------------------------------------------
  def __getattr__(self, name):
    if name.startswith('__'):
      raise AttributeError(name)
    fields = self.__dict__.get('fields')
    if fields is None:
      raise AttributeError(name)
    if name in fields:
      # read-only view: the device copy of the model is refreshed when `_version` changes, which a write through a raw
      # array could not signal. Write with `model.set(field, value)` or `physics.named.model.<field>[...] = v`.
      v = fields[name].view()
      v.flags.writeable = False
      return v
    key = name.upper()
    if key in SIZE:
      return int(fields['sizes'][SIZE[key]])
    if name in _NAME_SIZES and 'ordered_names' in self.__dict__:
      return len(self.ordered_names.get(_NAME_SIZES[name], []))
    if name == 'name':
      return next(iter(self.names.get('model', {})), 'MuJoCo Model')      # <mujoco model="...">
    vis = self.__dict__.get('vis') or {}
    if name in vis and name not in ('stat_center', 'stat_extent', 'global_fovy'):
      return vis[name]                                  # geom_rgba, site_rgba, geom_group, cam_*: writable (host-side only)
    if name == 'stat':
      return types.SimpleNamespace(meaninertia=float(fields['opt_real'][OPTR['MEANINERTIA']]),
                                   extent=float(vis['stat_extent'][0]) if 'stat_extent' in vis else None,
                                   center=vis.get('stat_center'))
    raise AttributeError(name)

  def set(self, field, value, index=slice(None)):
    """`model.<field>[index] = value` with the bookkeeping the device copy needs (the next step / forward re-uploads
    the model). The reference edits `physics.model.<field>` in place (e.g. domain randomisation); here the arrays
    handed out by attribute access are read-only so that such an edit cannot be silently ignored."""
    self.fields[field][index] = value
    self._version += 1

  def touch(self):
    """Mark the model as modified (after writing `model.fields[...]` directly)."""
    self._version += 1

  def name2id(self, name, object_type):
    """Mirror of `MjModel.name2id` (dm_control/mujoco/wrapper/core.py:334-362): -> id or raises."""
    kind = _OBJ_ALIASES.get(str(object_type).replace('mjOBJ_', '').lower())
    if kind is None or name not in self.names.get(kind, {}):
      raise ValueError(f'No {object_type} with name {name!r} exists.')
    return self.names[kind][name]

  def id2name(self, object_id, object_type):
    kind = _OBJ_ALIASES[str(object_type).replace('mjOBJ_', '').lower()]
    return self.ordered_names.get(kind, [])[object_id]

  _DISABLE_NAMES = dict(constraint=1 << 0, equality=1 << 1, frictionloss=1 << 2, limit=1 << 3, contact=1 << 4,
                        passive=1 << 5, gravity=1 << 6, clampctrl=1 << 7, warmstart=1 << 8, filterparent=1 << 9,
                        actuation=1 << 10, refsafe=1 << 11, sensor=1 << 12, midphase=1 << 13, eulerdamp=1 << 14)

  def disable(self, *flags):
    """Context manager that sets `opt.disableflags` bits for its body (reference: wrapper/core.py:389-426).

    `flags` are names ('contact', 'gravity', ...) or `mjtDisableBit` integers; anything else raises ValueError.
    """
    import contextlib
    bits = 0
    for f in flags:
      if isinstance(f, str):
        if f not in self._DISABLE_NAMES:
          raise ValueError(f'{f!r} is not a valid flag name. Valid names: {", ".join(sorted(self._DISABLE_NAMES))}')
        bits |= self._DISABLE_NAMES[f]
      else:
        f = int(f)
        if f <= 0 or f not in self._DISABLE_NAMES.values():
          raise ValueError(f'{f!r} is not a value in `mjtDisableBit`.')
        bits |= f

    @contextlib.contextmanager
    def ctx():
      old = self.opt.disableflags
      self.opt.disableflags = old | bits
      try:
        yield
      finally:
        self.opt.disableflags = old
    return ctx()

  def set_capacity(self, nconmax=None, njmax=None):
    if nconmax is not None:
      self.fields['sizes'][SIZE['NCONMAX']] = nconmax
    if njmax is not None:
      self.fields['sizes'][SIZE['NJMAX']] = njmax
    self._version += 1

  # --- blob ----------------------------------------------------------------------------------
  def pack(self):
    """-> (idata int32[ni], rdata float64[nr]) with the directory at idata[0 : 2*len(FIELDS)]."""
    nf = len(FIELDS)
    ichunks, rchunks = [], []
    ioff, roff = 2 * nf, 0
    directory = np.zeros(2 * nf, np.int32)
    for k, (name, kind) in enumerate(FIELDS):
      flat = self.fields[name].reshape(-1)
      if kind == 'i':
        directory[2 * k], directory[2 * k + 1] = ioff, flat.size
        ichunks.append(flat.astype(np.int32))
        ioff += flat.size
      else:
        directory[2 * k], directory[2 * k + 1] = roff, flat.size
        rchunks.append(flat.astype(np.float64))
        roff += flat.size
    idata = np.concatenate([directory] + ichunks).astype(np.int32)
    rdata = np.concatenate(rchunks + [np.zeros(1)]).astype(np.float64)
    return np.ascontiguousarray(idata), np.ascontiguousarray(rdata)

  def copy(self):
    return Model({k: v.copy() for k, v in self.fields.items()}, self.names, self.ordered_names,
                 vis={k: v.copy() for k, v in self.vis.items()})

  # --- binary model I/O (stands where MJB save/load stands: wrapper/core.py:208-234,323-332) ---
  def save(self, path):
    import json
    meta = json.dumps(dict(names=self.names, ordered_names=self.ordered_names, layout=[f for f, _ in FIELDS]))
    np.savez_compressed(path, __meta__=np.frombuffer(meta.encode(), dtype=np.uint8), **self.fields,
                        **{'vis__' + k: v for k, v in self.vis.items()})

  @classmethod
  def load(cls, path):
    import json
    with np.load(path) as z:
      meta = json.loads(bytes(z['__meta__']).decode())
      fields = {name: z[name] for name, _ in FIELDS if name in z}
      vis = {k[len('vis__'):]: z[k] for k in z.files if k.startswith('vis__')}
    missing = [name for name, _ in FIELDS if name not in fields]
    if missing:
      raise ValueError(f'{path}: model file predates the current blob layout (missing {missing}); regenerate it')
    return cls(fields, meta['names'], meta['ordered_names'], vis=vis)
