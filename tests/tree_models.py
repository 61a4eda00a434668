"""Generated models for the tree shapes the fixtures never reach.

The engine walks a tree level by level with one lane per body and strides of 32, and runs one lane per body, joint,
geom, site, actuator and tendon elsewhere; the fixtures' widest level has 6 bodies. These models have levels wider
than a warp, chains deeper than one, more than 32 joints, sites, actuators and fixed tendons, welded (jointless)
bodies, bodies with several joints, and rotated body, inertial, geom and site frames with joint offsets. Every body
has an explicit inertial (some `diaginertia` with a rotated frame, some `fullinertia`); geoms do not collide.

`MODELS` maps a name to a generator; `model(name)` compiles (and caches) it with contacts disabled.
"""
from __future__ import annotations

import copy

import numpy as np

from dm_control_b200 import mjcf_compile

DSBL_CONTACT = 1 << 4
_CACHE = {}


def _v(rs, n, lo=-1.0, hi=1.0):
  return ' '.join(f'{x:.6g}' for x in rs.uniform(lo, hi, n))


def _unit(rs, n=3):
  x = rs.randn(n)
  return ' '.join(f'{v:.6g}' for v in x / np.linalg.norm(x))


def _inertial(rs, k):
  mass = rs.uniform(0.2, 2.0)
  if k % 3 == 2:        # fullinertia: a random SPD matrix well inside the triangle inequality
    A = rs.uniform(-0.3, 0.3, (3, 3)); I = 0.02 * (A @ A.T + np.eye(3))
    return (f'<inertial pos="{_v(rs, 3, -0.05, 0.05)}" mass="{mass:.4g}" fullinertia="{I[0,0]:.6g} {I[1,1]:.6g} '
            f'{I[2,2]:.6g} {I[0,1]:.6g} {I[0,2]:.6g} {I[1,2]:.6g}"/>')
  d = rs.uniform(0.02, 0.04, 3)          # any two at least the third
  return (f'<inertial pos="{_v(rs, 3, -0.05, 0.05)}" quat="{_unit(rs, 4)}" mass="{mass:.4g}" '
          f'diaginertia="{d[0]:.5g} {d[1]:.5g} {d[2]:.5g}"/>')


def _decor(rs, name):
  return (f'<geom type="sphere" size="0.03" pos="{_v(rs, 3, -0.1, 0.1)}" quat="{_unit(rs, 4)}" contype="0" '
          f'conaffinity="0"/><site name="s_{name}" pos="{_v(rs, 3, -0.1, 0.1)}" quat="{_unit(rs, 4)}"/>')


def _joint(rs, name, kind):
  if kind == 'ball':
    return f'<joint name="{name}" type="ball" pos="{_v(rs, 3, -0.05, 0.05)}" damping="{rs.uniform(0, 0.2):.3g}" armature="0.01"/>'
  ref = f' ref="{rs.uniform(-0.3, 0.3):.4g}"' if rs.rand() < 0.5 else ''
  return (f'<joint name="{name}" type="{kind}" pos="{_v(rs, 3, -0.05, 0.05)}" axis="{_unit(rs)}"{ref} '
          f'stiffness="{rs.uniform(0, 2):.3g}" springref="{rs.uniform(-0.2, 0.2):.3g}" damping="{rs.uniform(0, 0.3):.3g}" '
          f'armature="{rs.uniform(0.005, 0.05):.3g}"/>')


def _actuators(rs, joints, ntendon):
  """Motor, position, velocity and general (affine gain and bias, integrator / filter dynamics) in turn, on scalar
  joints and on tendons, with control and force limits."""
  out = []
  targets = [f'joint="{j}"' for j in joints] + [f'tendon="t{t}"' for t in range(ntendon)]
  for k, tgt in enumerate(targets):
    lim = f'ctrlrange="-1 1" ctrllimited="true"' if k % 2 == 0 else ''
    flim = f' forcerange="-0.6 0.8" forcelimited="true"' if k % 3 == 1 else ''
    kind = k % 4
    if kind == 0:
      out.append(f'<motor {tgt} gear="{rs.uniform(0.5, 3):.3g}" {lim}{flim}/>')
    elif kind == 1:
      out.append(f'<position {tgt} kp="{rs.uniform(1, 5):.3g}" {lim}{flim}/>')
    elif kind == 2:
      out.append(f'<velocity {tgt} kv="{rs.uniform(0.1, 1):.3g}" {lim}{flim}/>')
    else:
      dyn = ('dyntype="integrator" actrange="-0.5 0.7" actlimited="true"' if k % 8 == 3 else
             f'dyntype="filter" dynprm="{rs.uniform(0.02, 0.2):.3g}"')
      out.append(f'<general {tgt} {dyn} gaintype="affine" gainprm="{_v(rs, 3, 0.2, 1.5)}" biastype="affine" '
                 f'biasprm="{_v(rs, 3, -0.5, 0.5)}" gear="{rs.uniform(0.5, 2):.3g}" {lim}{flim}/>')
  return ''.join(out)


def _tendons(rs, joints, n):
  out = []
  for t in range(n):
    pick = rs.choice(len(joints), size=min(3, len(joints)), replace=False)
    terms = ''.join(f'<joint joint="{joints[i]}" coef="{rs.uniform(-1.5, 1.5):.3g}"/>' for i in pick)
    out.append(f'<fixed name="t{t}">{terms}</fixed>')
  return f'<tendon>{"".join(out)}</tendon>' if out else ''


def _wrap(name, body, joints, rs, ntendon=0, nact=None):
  act_joints = joints if nact is None else joints[:nact]
  return (f'<mujoco model="{name}"><compiler angle="radian"/><option timestep="0.004"/>'
          f'<worldbody>{body}</worldbody>{_tendons(rs, joints, ntendon)}'
          f'<actuator>{_actuators(rs, act_joints, ntendon)}</actuator></mujoco>')


def wide_free(nchild, seed=0):
  """A free root with `nchild` children on one level: the first min(nchild, 58) on slide joints, the rest welded."""
  rs = np.random.RandomState(seed + nchild)
  kids, joints = '', []
  for k in range(nchild):
    jt = ''
    if k < 58:
      joints.append(f'j{k}'); jt = _joint(rs, f'j{k}', 'slide')
    kids += (f'<body name="c{k}" pos="{_v(rs, 3, -0.5, 0.5)}" quat="{_unit(rs, 4)}">{jt}{_inertial(rs, k)}'
             f'{_decor(rs, f"c{k}")}</body>')
  body = (f'<body name="root" pos="0 0 1" quat="{_unit(rs, 4)}"><freejoint/>{_inertial(rs, 0)}{_decor(rs, "root")}'
          f'{kids}</body>')
  return _wrap(f'wide{nchild}', body, joints, rs, ntendon=34 if nchild >= 40 else 0)


def chain(n, seed=0):
  """n hinges in a chain, one body each, rotated frames and joint offsets."""
  rs = np.random.RandomState(seed + 1000 + n)
  body, close, joints = '', '', []
  for k in range(n):
    joints.append(f'h{k}')
    body += (f'<body name="l{k}" pos="{_v(rs, 3, -0.05, 0.05)} " quat="{_unit(rs, 4)}">{_joint(rs, f"h{k}", "hinge")}'
             f'{_inertial(rs, k)}{_decor(rs, f"l{k}")}')
    close += '</body>'
  return _wrap(f'chain{n}', body + close, joints, rs, nact=40)


def welded(nbody, nv, seed=0):
  """A free root and a random tree of nbody - 1 more bodies, of which only some carry a hinge or slide, so that nv
  stays at `nv`."""
  rs = np.random.RandomState(seed + 2000 + nbody)
  njoint = nv - 6
  jointed = set(rs.choice(np.arange(1, nbody), size=njoint, replace=False).tolist())
  parent = [-1] + [int(rs.randint(0, k)) for k in range(1, nbody)]
  children = {k: [] for k in range(nbody)}
  for k in range(1, nbody):
    children[parent[k]].append(k)
  joints = []

  def emit(k):
    if k == 0:
      inner = '<freejoint/>'
    elif k in jointed:
      joints.append(f'w{k}'); inner = _joint(rs, f'w{k}', 'hinge' if k % 3 else 'slide')
    else:
      inner = ''
    s = (f'<body name="b{k}" pos="{_v(rs, 3, -0.3, 0.3)}" quat="{_unit(rs, 4)}">{inner}{_inertial(rs, k)}'
         f'{_decor(rs, f"b{k}")}')
    return s + ''.join(emit(c) for c in children[k]) + '</body>'
  return _wrap(f'welded{nbody}', emit(0), joints, rs, ntendon=8)


def multi_joint(seed=0):
  """Bodies with two and three joints (hinge + slide + hinge, slide + hinge, hinge + ball), off-origin joints."""
  rs = np.random.RandomState(seed + 3000)
  groups = [('hinge', 'slide', 'hinge'), ('slide', 'hinge'), ('hinge', 'ball'), ('hinge', 'slide', 'hinge'),
            ('ball',), ('slide', 'slide', 'hinge')]
  body, close, joints = '', '', []
  for k, g in enumerate(groups):
    js = ''
    for i, kind in enumerate(g):
      js += _joint(rs, f'm{k}_{i}', kind)
      if kind != 'ball':
        joints.append(f'm{k}_{i}')
    body += f'<body name="g{k}" pos="{_v(rs, 3, -0.2, 0.2)}" quat="{_unit(rs, 4)}">{js}{_inertial(rs, k)}{_decor(rs, f"g{k}")}'
    close += '</body>'
  body = (f'<body name="root" pos="0 0.1 0.5" quat="{_unit(rs, 4)}"><freejoint/>{_inertial(rs, 1)}{_decor(rs, "root")}'
          f'{body}{close}</body>')
  return _wrap('multijoint', body, joints, rs, ntendon=3)


MODELS = {
    'wide33': lambda: wide_free(33), 'wide40': lambda: wide_free(40), 'wide64': lambda: wide_free(64),
    'chain64': lambda: chain(64), 'welded65': lambda: welded(65, 30), 'welded100': lambda: welded(100, 64),
    'multijoint': multi_joint,
}


def model(name):
  if name not in _CACHE:
    m = mjcf_compile.compile_xml(MODELS[name]())
    m.opt.disableflags = m.opt.disableflags | DSBL_CONTACT
    _CACHE[name] = m
  return copy.deepcopy(_CACHE[name])
