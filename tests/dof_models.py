"""Generated models with exactly the number of degrees of freedom asked for.

The fixture models reach only a few dof counts. The engine switches code paths on nv: one compile-time-size
acceleration kernel per entry of B200MJ_NV_LIST (6, 9, 12, 18, 22, 27), and in the runtime-size algebra one row per lane
below 32, two rows per lane from 32, and no spare row for a ride-along right-hand side at 64, the largest nv the
engine accepts. `model(nv)` builds a free-floating torso with limbs of ball, hinge and slide joints, spheres and
capsules only (closed-form contact pairs), a floor, and motors on some hinges. `initial_states(model, batch, seed)` gives seeded starts.
"""
from __future__ import annotations

import numpy as np

from dm_control_b200 import mjcf_compile

_CACHE = {}


def _limb_xml(joints, k, rs):
  """A chain of bodies, one joint each, hanging down and out from the torso; returns (xml, motorised joint names)."""
  ang = 2 * np.pi * k / 6 + rs.uniform(-0.2, 0.2)
  dx, dy = 0.12 * np.cos(ang), 0.12 * np.sin(ang)
  xml, close, motors = '', '', []
  for i, kind in enumerate(joints):
    name = f'j{k}_{i}'
    pos = f'{dx:.4f} {dy:.4f} -0.05' if i == 0 else f'{dx * 0.6:.4f} {dy * 0.6:.4f} -0.1'
    xml += f'<body name="b{k}_{i}" pos="{pos}">'
    if kind == 'ball':
      xml += f'<joint name="{name}" type="ball" damping="0.2" armature="0.01"/>'
    else:
      axis = rs.randn(3); axis /= np.linalg.norm(axis)
      xml += (f'<joint name="{name}" type="{kind}" axis="{axis[0]:.4f} {axis[1]:.4f} {axis[2]:.4f}" damping="0.3" '
              f'armature="0.01"/>')
      if kind == 'hinge' and i % 2 == 0:
        motors.append(name)
    if i % 2:
      xml += f'<geom type="sphere" size="{rs.uniform(0.03, 0.05):.3f}" mass="{rs.uniform(0.1, 0.5):.3f}"/>'
    else:
      xml += (f'<geom type="capsule" size="{rs.uniform(0.02, 0.035):.3f}" fromto="0 0 0 {dx * 0.6:.4f} {dy * 0.6:.4f} -0.1" '
              f'mass="{rs.uniform(0.1, 0.5):.3f}"/>')
    close += '</body>'
  return xml + close, motors


def xml(nv, seed=0):
  """MJCF of a model with exactly `nv` dofs: 6 of a free joint, the rest in up to six limbs."""
  assert nv >= 6
  rs = np.random.RandomState(seed * 1009 + nv)
  rest = nv - 6
  kinds = []
  while rest:                                    # balls while they fit, then hinges and slides
    if rest >= 3 and len(kinds) % 3 != 2:
      kinds.append('ball'); rest -= 3
    else:
      kinds.append('hinge' if len(kinds) % 4 else 'slide'); rest -= 1
  limbs = [kinds[k::6] for k in range(min(6, len(kinds)))]
  body, motors = '', []
  for k, joints in enumerate(limbs):
    x, m = _limb_xml(joints, k, rs)
    body += x; motors += m
  act = ''.join(f'<motor joint="{j}" gear="2" ctrlrange="-1 1" ctrllimited="true"/>' for j in motors)
  return (f'<mujoco model="dof{nv}"><option timestep="0.005"/>'
          f'<worldbody><geom name="floor" type="plane" size="5 5 .1"/>'
          f'<body name="torso" pos="0 0 0.6"><freejoint/><geom type="sphere" size="0.1" mass="2"/>{body}</body>'
          f'</worldbody><actuator>{act}</actuator></mujoco>')


def name(nv):
  return f'dof{nv}'


def model(nv):
  if nv not in _CACHE:
    _CACHE[nv] = mjcf_compile.compile_xml(xml(nv))
  return _CACHE[nv]


def initial_states(m, batch, seed=0):
  """Upside down (the limbs point up), the torso sphere 0 to 4 cm above the floor, a slightly random orientation and
  random joint velocities: the torso lands within the first tenth of a second and the limbs swing over it."""
  q = np.tile(m.qpos0, (batch, 1)).astype(np.float64)
  v = np.zeros((batch, m.nv))
  for e in range(batch):
    rs = np.random.RandomState(seed * 100003 + e)
    quat = np.array([0.0, 1.0, 0.0, 0.0]) + rs.uniform(-0.15, 0.15, 4)
    q[e, 2] = rs.uniform(0.1, 0.14)
    q[e, 3:7] = quat / np.linalg.norm(quat)
    v[e, 6:] = rs.uniform(-1, 1, m.nv - 6)
  return q, v


NV_TARGETS = (6, 9, 12, 18, 22, 27, 31, 32, 33, 63, 64)     # the compile-time-size kernels, the runtime-size boundaries


def load(name, batch, seed):
  """(model, qpos, qvel) for a fixture name (testing_models) or a generated `dofNN`."""
  if name.startswith('dof'):
    m = model(int(name[3:]))
    return (m,) + initial_states(m, batch, seed)
  from dm_control_b200 import testing_models as tm
  m = tm.load(name)
  return (m,) + tm.initial_states(m, name, batch, seed)
