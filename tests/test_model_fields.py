"""The compiled model's field table (`model.MODEL_FIELDS`) against the blob header and the kernels' per-environment
list, and the named indexing and `physics.bind` it drives on the model side -- no GPU needed."""
import os
import re
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import dof_models                                        # noqa: E402
import tree_models                                       # noqa: E402
from dm_control_b200 import binding, index, mjcf_compile  # noqa: E402
from dm_control_b200 import model as bmodel               # noqa: E402
from dm_control_b200 import testing_models as tm          # noqa: E402
from dm_control_b200.physics import ENV_MODEL_FIELDS      # noqa: E402

# keyframes, a joint equality and a fixed tendon: the row axes the fixtures leave empty
KEYS_AND_EQUALITIES = """
<mujoco><worldbody>
  <body name="a" pos="0 0 1"><joint name="hinge" axis="0 1 0"/><geom size=".1"/>
    <body name="b" pos=".2 0 0"><joint name="slide" type="slide" axis="1 0 0"/><geom size=".05"/></body></body>
  <body name="free" pos="1 0 1"><freejoint name="free"/><geom size=".1"/></body>
</worldbody>
<tendon><fixed name="couple"><joint joint="hinge" coef="1"/><joint joint="slide" coef="-.5"/></fixed></tendon>
<equality><joint name="lock" joint1="hinge" joint2="slide"/></equality>
<keyframe><key name="home" qpos="0.1 0.2 1 0 1 1 0 0 0"/><key name="away" qpos="-.3 .1 2 1 1 0 0 0 1"/></keyframe>
</mujoco>"""

ASSETS = sorted(f[:-len('.npz')] for f in os.listdir(tm._ASSETS) if f.endswith('.npz'))
MODELS = (sorted(tm.XML) + ASSETS + [f'dof{nv}' for nv in dof_models.NV_TARGETS] + [f'tree_{n}' for n in tree_models.MODELS]
          + ['keys_and_equalities'])

# the model entries of index.py's row and column kinds before they were derived from MODEL_FIELDS
OLD_COL_KIND = {
    **dict.fromkeys(('body_pos', 'body_ipos', 'body_inertia', 'jnt_pos', 'jnt_axis', 'geom_size', 'geom_pos', 'site_size',
                     'site_pos'), 'xyz'),
    **dict.fromkeys(('body_quat', 'body_iquat', 'geom_quat', 'site_quat'), 'quat'),
    **dict.fromkeys(('geom_rgba', 'site_rgba', 'mat_rgba'), 'rgba'),
}
OLD_ROW_KIND = {
    **{f: 'body' for f in ('body_pos', 'body_quat', 'body_ipos', 'body_iquat', 'body_mass', 'body_inertia', 'body_parentid',
                           'body_rootid', 'body_subtreemass')},
    **{f: 'geom' for f in ('geom_size', 'geom_pos', 'geom_quat', 'geom_type', 'geom_bodyid', 'geom_friction', 'geom_rbound',
                           'geom_condim', 'geom_rgba', 'geom_group', 'geom_solref', 'geom_solimp')},
    **{f: 'site' for f in ('site_pos', 'site_quat', 'site_size', 'site_bodyid', 'site_rgba', 'site_group')},
    **{f: 'camera' for f in ('cam_pos', 'cam_quat', 'cam_fovy', 'cam_bodyid', 'cam_mode', 'cam_targetbodyid')},
    'mat_rgba': 'material',
    **{f: 'joint' for f in ('jnt_type', 'jnt_range', 'jnt_limited', 'jnt_pos', 'jnt_axis', 'jnt_stiffness', 'jnt_qposadr',
                            'jnt_dofadr', 'jnt_bodyid')},
    **{f: 'actuator' for f in ('actuator_ctrlrange', 'actuator_gear', 'actuator_ctrllimited', 'actuator_gainprm',
                               'actuator_biasprm')},
    'qpos0': 'nq', 'dof_damping': 'nv', 'dof_armature': 'nv',
}
_LOADED = {}


def load(name):
  if name not in _LOADED:
    if name.startswith('dof'):
      _LOADED[name] = dof_models.model(int(name[3:]))
    elif name.startswith('tree_'):
      _LOADED[name] = tree_models.model(name[len('tree_'):])
    elif name == 'keys_and_equalities':
      _LOADED[name] = mjcf_compile.compile_xml(KEYS_AND_EQUALITIES)
    else:
      _LOADED[name] = tm.load(name)
  return _LOADED[name]


def _element_rows(m, field, name):
  """Rows of `field` that belong to element `name`, from the model's own tables."""
  rows = bmodel.MODEL_FIELDS[field].rows
  if rows in ('nq', 'nv'):
    j = m.name2id(name, 'joint')
    adr = m.jnt_qposadr if rows == 'nq' else m.jnt_dofadr
    end = list(adr[1:]) + [getattr(m, rows)]
    return slice(int(adr[j]), int(end[j]))
  return m.name2id(name, rows)


def _named_fields():
  """(field, kind of the elements that name its rows) of every model field with named rows."""
  owner = {'nq': 'joint', 'nv': 'joint', 'pair': None, 'wrap': None, 'level': None, None: None}
  return [(n, owner.get(f.rows, f.rows)) for n, f in bmodel.MODEL_FIELDS.items() if owner.get(f.rows, f.rows)]


def test_table_is_the_header():
  assert [(n, f.dtype) for n, f in bmodel.MODEL_FIELDS.items()] == \
      [(n, np.int32 if k == 'i' else np.float64) for n, k in bmodel.FIELDS]
  assert set(bmodel._DECLARED) <= set(bmodel.MODEL_FIELDS)        # no declaration of a field the header lacks
  assert len(_named_fields()) + 3 + 6 == len(bmodel.FIELDS)          # sizes, opt_*; pair_*, wrap_*, level_*


def test_per_environment_fields_are_the_kernels():
  src = open(os.path.join(os.path.dirname(HERE), 'dm_control_b200', 'csrc', 'b200mj.cu')).read()
  macro = re.search(r'#define ENV_FIELDS\(X\)((?:.*\\\n)*.*)', src).group(1)
  kernel = tuple(re.findall(r'X\((\w+)\)', macro))
  assert len(kernel) == 11
  assert ENV_MODEL_FIELDS == kernel
  assert sorted(f.env for f in bmodel.MODEL_FIELDS.values() if f.env is not None) == list(range(len(kernel)))
  assert all(bmodel.MODEL_FIELDS[n].dtype == np.float64 for n in kernel)
  import test_smooth_dynamics                # randomises every per-environment field, in this order
  assert test_smooth_dynamics.ENV_FIELDS == ENV_MODEL_FIELDS


def test_row_and_column_kinds_are_unchanged():
  for f, kind in OLD_ROW_KIND.items():
    assert index._ROW_KIND[f] == kind, f
  for f, kind in OLD_COL_KIND.items():
    assert index._COL_KIND[f] == kind, f
  model_side = set(bmodel.MODEL_FIELDS) | {'geom_rgba', 'site_rgba', 'mat_rgba', 'geom_group', 'site_group', 'cam_pos', 'cam_quat'}
  assert {f for f in index._COL_KIND if f in model_side} == set(OLD_COL_KIND)       # no new column names


@pytest.mark.parametrize('name', MODELS)
def test_every_field_has_its_declared_shape(name):
  m = load(name)
  count = dict(body=m.nbody, joint=m.njnt, geom=m.ngeom, site=m.nsite, actuator=m.nu, tendon=m.ntendon, equality=m.neq,
               sensor=m.nsensor, key=m.nkey, nq=m.nq, nv=m.nv, pair=m.npair, wrap=m.nwrap)    # no one size counts the levels
  for f in bmodel.MODEL_FIELDS.values():
    a = m.fields[f.name]
    want = (() if f.rows is None else (count.get(f.rows, a.shape[0]),)) + \
        tuple(getattr(m, w) if isinstance(w, str) else w for w in f.width)
    assert a.dtype == f.dtype and a.shape == want and a.flags.c_contiguous, (f.name, a.shape, want)
  for n, a in m.copy().fields.items():
    assert a.shape == m.fields[n].shape and np.array_equal(a, m.fields[n]), n


@pytest.mark.parametrize('name', MODELS)
def test_named_model_fields_and_bind_read_the_elements_rows(name):
  m = load(name)
  phys = types.SimpleNamespace(model=m, data=types.SimpleNamespace(), device=torch.device('cpu'), batch=1)
  named = index.NamedIndexStructs(phys).model
  checked = 0
  for field, kind in _named_fields():
    rows = bmodel.MODEL_FIELDS[field].rows
    # the attribute `bind` gives the field: its name without the prefix, or a joint's damping / armature
    attr = field.split('_', 1)[1] if rows == kind else {'dof_damping': 'damping', 'dof_armature': 'armature'}.get(field)
    for el in m.names.get(kind, {}):
      want = m.fields[field][_element_rows(m, field, el)]
      np.testing.assert_array_equal(getattr(named, field)[el], want, err_msg=f'named.model.{field}[{el!r}]')
      if attr is not None:
        np.testing.assert_array_equal(getattr(binding.Binding(phys, kind, el), attr), want, err_msg=f'bind({kind!r}, {el!r}).{attr}')
      checked += 1
  assert checked > 0


def test_keyframes_equalities_and_ragged_fields_are_named():
  m = load('keys_and_equalities')
  phys = types.SimpleNamespace(model=m, data=types.SimpleNamespace(), device=torch.device('cpu'), batch=1)
  named = index.NamedIndexStructs(phys).model
  np.testing.assert_array_equal(named.key_qpos['away'], [-.3, .1, 2, 1, 1, 0, 0, 0, 1])
  np.testing.assert_array_equal(binding.Binding(phys, 'key', 'home').qpos, [.1, .2, 1, 0, 1, 1, 0, 0, 0])
  assert named.eq_solref['lock'].shape == (2,) and named.eq_data['lock'].shape == (11,)
  assert named.qpos0['free'].shape == (7,) and named.dof_solimp['free'].shape == (6, 5)
  assert named.tendon_length0.row_names == ['couple']
  np.testing.assert_array_equal(binding.Binding(phys, 'joint', ['free', 'hinge']).damping, np.zeros(7))


@pytest.mark.parametrize('field', ['body_pos', 'jnt_range', 'key_qpos', 'sizes', 'dof_solimp'])
def test_a_wrong_size_is_refused_by_name(field):
  m = load('keys_and_equalities')
  fields = dict(m.fields)
  fields[field] = np.concatenate([m.fields[field].reshape(-1), [0]])
  with pytest.raises(ValueError, match=field):
    bmodel.Model(fields, m.names, m.ordered_names)
  bmodel.Model({**fields, field: m.fields[field].reshape(-1)}, m.names, m.ordered_names)       # flat but whole: shaped
