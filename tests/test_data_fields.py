"""The batched data-field table (`physics.DATA_FIELDS`) against the C ABI, and the ragged columns `physics.bind` takes
from it — no GPU needed."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch

from dm_control_b200 import binding, mjcf_compile
from dm_control_b200 import lib as blib
from dm_control_b200 import testing_models as tm
from dm_control_b200.physics import APPLIED_FIELDS, DATA_FIELDS, STATE_FIELDS

# free, ball, hinge and slide joints; actuators with and without an activation; sensors of width 1 and 3
BALL_FREE = """
<mujoco><worldbody>
  <geom name="floor" type="plane" size="1 1 .1"/>
  <body name="root" pos="0 0 1"><freejoint name="root"/><geom size=".1"/>
    <body name="arm" pos=".2 0 0"><joint name="shoulder" type="ball"/><geom size=".05"/>
      <body name="fore" pos=".2 0 0"><joint name="elbow" type="hinge" axis="0 1 0"/><geom size=".05"/>
        <body name="hand" pos=".2 0 0"><joint name="wrist" type="ball"/><joint name="slide" type="slide" axis="1 0 0"/>
          <geom size=".04"/><site name="tip"/></body></body></body></body>
  <body name="ball" pos="1 0 1"><freejoint/><geom size=".1"/></body>
</worldbody>
<actuator><motor name="elbow" joint="elbow"/><general name="slide_int" joint="slide" dyntype="integrator"/>
  <motor name="slide" joint="slide"/><general name="elbow_int" joint="elbow" dyntype="integrator"/></actuator>
<sensor><jointpos joint="elbow"/><framepos objtype="site" objname="tip"/><velocimeter name="vel" site="tip"/>
  <jointvel joint="slide"/><subtreecom body="arm"/></sensor>
</mujoco>"""

MODELS = sorted(tm.XML) + sorted(f[:-len('.npz')] for f in os.listdir(tm._ASSETS) if f.endswith('.npz')) + ['ball_free']

# what the columns of one element are, from its joint type, sensor width or activation address
QPOS_WIDTH, DOF_WIDTH = {0: 7, 1: 4, 2: 1, 3: 1}, {0: 6, 1: 3, 2: 1, 3: 1}     # free, ball, slide, hinge
NV_FIELDS = ('qvel', 'qacc', 'qacc_warmstart', 'qfrc_bias', 'qfrc_passive', 'qfrc_actuator', 'qfrc_constraint', 'qfrc_applied')
RAGGED = {'joint': ('qpos',) + NV_FIELDS, 'sensor': ('sensordata',), 'actuator': ('act',)}


def _columns(m, kind, field, ids):
  if kind == 'joint':
    adr, width = (m.jnt_qposadr, QPOS_WIDTH) if field == 'qpos' else (m.jnt_dofadr, DOF_WIDTH)
    return [int(adr[j]) + k for j in ids for k in range(width[int(m.jnt_type[j])])]
  if kind == 'sensor':
    return [int(m.sensor_adr[s]) + k for s in ids for k in range(int(m.sensor_dim[s]))]
  return [int(m.actuator_actadr[a]) for a in ids if m.actuator_actadr[a] >= 0]


def test_table_is_the_io_struct():
  io = [(n, c) for n, c in blib.IO_FIELDS if n not in ('var_geom_pos', 'var_geom_size')]
  assert list(DATA_FIELDS) == [n for n, _ in io]
  assert list(DATA_FIELDS)[:5] == ['qpos', 'qvel', 'act', 'qacc_warmstart', 'time']
  for n, ctype in io:
    assert DATA_FIELDS[n].dtype == (torch.float64 if ctype._type_ is ctypes.c_double else torch.int32), n
  assert STATE_FIELDS == ('qpos', 'qvel', 'act', 'qacc_warmstart', 'time', 'ctrl')
  assert APPLIED_FIELDS == ('qfrc_applied', 'xfrc_applied')


@pytest.mark.parametrize('name', MODELS)
def test_bind_ragged_columns(name):
  m = mjcf_compile.compile_xml(BALL_FREE) if name == 'ball_free' else tm.load(name)
  B = 2
  data = types.SimpleNamespace()
  for f in {f for fields in RAGGED.values() for f in fields}:
    n = int(np.prod(DATA_FIELDS[f].shape(m), dtype=np.int64))
    setattr(data, f, torch.arange(B * n, dtype=torch.float64).reshape(B, n))
  phys = types.SimpleNamespace(model=m, data=data, device=torch.device('cpu'), batch=B, mark_as_dirty=lambda: None,
                               forward=lambda: None)
  for kind, fields in RAGGED.items():
    names = m.ordered_names.get(kind, [])
    selections = [[n] for n in names] + ([names[::-1]] if names else [])
    for sel in selections:
      ids = [m.name2id(n, kind) for n in sel]
      bound = binding.Binding(phys, kind, sel if len(sel) > 1 else sel[0])
      for field in fields:
        cols = _columns(m, kind, field, ids)
        t = getattr(data, field)
        assert torch.equal(getattr(bound, field), t[:, cols]), (kind, sel, field)
        if len(sel) > 1:
          before = t.clone()
          new = -1.0 - torch.arange(B * len(cols), dtype=torch.float64).reshape(B, len(cols))
          setattr(bound, field, new)
          before[:, cols] = new
          assert torch.equal(t, before), (kind, field)
