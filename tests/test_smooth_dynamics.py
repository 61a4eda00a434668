"""The engine's smooth dynamics, stage by stage, against first principles in extended precision (tests/smooth_reference.py).

Kinematics (body, inertial, geom and site frames), the subtree centres of mass, `cvel`, `subtree_linvel`, the
joint-space inertia `qM`, `qfrc_bias`, passive and actuator forces, the unconstrained `qacc`, and one Euler (explicit
and implicit-damping) or RK4 step, on generated trees wider than a warp (tests/tree_models.py), the dof-count models
and the fixtures, with contacts (and equality constraints) disabled and every joint inside its limits, so that no constraint row exists.

Two tiers run the same cases, as in test_dense_algebra.py:
  * `cpu`: the emulated kernels (tests/emu/b200mj_emu.EmuPhysics), no GPU needed;
  * `gpu` (`-m gpu`): `BatchedPhysics` on the device (or on the emulation under B200MJ_EMULATE_GPU=1).

Bounds. Forward quantities are held norm-wise, |x - x_ref|_max <= C (depth + nv) U scale(field), with `depth` the
number of tree levels and scale(field) the magnitude the field's terms can reach (smooth_reference.forward: tree
extent, speeds, force sums). `qacc` and the implicit Euler solve are held by backward error -- the residual of the
kernel's answer against the reference's M and force -- because the 64-hinge chain's M is ill-conditioned and a forward
error would measure the conditioning, not the kernel. One constant C holds everything. Set B200MJ_SMOOTH_REPORT to a
path to have the worst ratio err / ((depth + nv) U scale) per tier and field written there as JSON.
"""
from __future__ import annotations

import atexit
import copy
import json
import os
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, 'emu'))
import b200mj_emu as emu            # noqa: E402
import dof_models                   # noqa: E402
import smooth_reference as ref      # noqa: E402
import tree_models                  # noqa: E402
from dm_control_b200 import mjcf_compile             # noqa: E402
from dm_control_b200 import testing_models as tm     # noqa: E402

pytestmark = pytest.mark.timeout(900)

U = 2.0 ** -53
C = 8
LD = np.longdouble
DSBL_EQUALITY, DSBL_CONTACT, DSBL_PASSIVE, DSBL_GRAVITY, DSBL_CLAMPCTRL = 1 << 1, 1 << 4, 1 << 5, 1 << 6, 1 << 7
DSBL_ACTUATION, DSBL_EULERDAMP = 1 << 10, 1 << 14
TIERS = ['cpu', pytest.param('gpu', marks=pytest.mark.gpu)]

WORST = {}


def _report():
  path = os.environ.get('B200MJ_SMOOTH_REPORT')
  if path and WORST:
    with open(path, 'w') as f:
      json.dump({t: dict(sorted(v.items())) for t, v in WORST.items()}, f, indent=1)


atexit.register(_report)


# ------------------------------------------------------------------------------------------------------------------
# the two tiers behind one driver
# ------------------------------------------------------------------------------------------------------------------
class Run:
  """B environments of `model` on the emulated kernels (`cpu`) or through BatchedPhysics (`gpu`); numpy in and out."""

  def __init__(self, tier, model, B, legacy=True, applied=False, env_fields=()):
    self.tier = tier
    if tier == 'cpu':
      assert not env_fields
      self.p = emu.EmuPhysics(model, B, legacy_step=legacy, applied_forces=applied)
    else:
      import torch
      from dm_control_b200.physics import BatchedPhysics
      self.torch = torch
      self.p = BatchedPhysics(model, batch=B)
      self.p.legacy_step = legacy
      if applied:
        self.p.enable_applied_forces(True)
      if env_fields:
        self.p.set_env_model_fields(list(env_fields))

  def set(self, name, value):
    if self.tier == 'cpu':
      getattr(self.p.data, name)[:] = value
    else:
      t = getattr(self.p.data, name)
      t.copy_(self.torch.as_tensor(np.asarray(value), dtype=t.dtype).reshape(t.shape).to(t.device))

  def set_env(self, name, value):
    t = getattr(self.p.env_model, name)
    t.copy_(self.torch.as_tensor(np.asarray(value), dtype=t.dtype).reshape(t.shape).to(t.device))

  def get(self, name):
    a = getattr(self.p.data, name)
    return np.array(a) if self.tier == 'cpu' else a.detach().cpu().numpy().copy()

  def forward(self):
    self.p.forward()

  def step(self, n=1):
    self.p.step(n)


def no_contact(model):
  """Contacts off, and the quadruped's tendon equalities too: constraint rows are not this file's subject."""
  m = copy.deepcopy(model)
  m.opt.disableflags = int(m.opt.disableflags) | DSBL_CONTACT | DSBL_EQUALITY
  return m


def load(name):
  if name in tree_models.MODELS:
    return tree_models.model(name)
  if name.startswith('dof'):
    return no_contact(mjcf_compile.compile_xml(dof_models.xml(int(name[3:]))))
  return no_contact(tm.load(name))


def random_quat(rs):
  q = rs.randn(4)
  return q / np.linalg.norm(q)


def random_state(m, rs, vscale=1.0):
  """Random unit quaternions, hinge and slide joints inside their ranges where limited, controls beyond +-1 (so that
  control clamps act at both ends) and activations inside their ranges."""
  q = np.array(m.qpos0, np.float64)
  for j in range(m.njnt):
    t, qa = m.jnt_type[j], m.jnt_qposadr[j]
    if t == ref.FREE:
      q[qa:qa + 3] += rs.uniform(-0.5, 0.5, 3)
      q[qa + 3:qa + 7] = random_quat(rs)
    elif t == ref.BALL:
      q[qa:qa + 4] = random_quat(rs)
    elif m.jnt_limited[j]:
      lo, hi = m.jnt_range[j]
      q[qa] = rs.uniform(lo + 0.1 * (hi - lo), hi - 0.1 * (hi - lo))
    else:
      q[qa] += rs.uniform(-np.pi, np.pi) if t == ref.HINGE else rs.uniform(-0.3, 0.3)
  v = rs.uniform(-1, 1, m.nv) * vscale
  ctrl = rs.uniform(-1.5, 1.5, m.nu)
  act = np.zeros(m.na)
  for u in range(m.nu):
    aa = m.actuator_actadr[u]
    if aa >= 0:
      lo, hi = m.actuator_actrange[u] if m.actuator_actlimited[u] else (-1.0, 1.0)
      act[aa] = rs.uniform(lo, hi)
  return q, v, ctrl, act


def record(tier, field, ratio):
  WORST.setdefault(tier, {})
  WORST[tier][field] = max(WORST[tier].get(field, 0.0), float(ratio))


def check(tier, what, field, got, want, n, scale):
  got = np.asarray(got, np.float64).reshape(-1)
  want = np.asarray(want, LD).reshape(-1)
  assert got.shape == want.shape, (what, field, got.shape, want.shape)
  assert np.all(np.isfinite(got)), (what, field)
  err = float(np.max(np.abs(got.astype(LD) - want), initial=0))
  ratio = err / (n * U * scale) if scale > 0 else (0.0 if err == 0 else np.inf)
  record(tier, field, ratio)
  assert ratio <= C, f'{what}: {field} off by {err:.3e} = {ratio:.2f} x (depth + nv) U scale (scale {scale:.3e})'


def mat2quat(R):
  """Unit quaternion (w >= 0) of a rotation matrix, in long double (Shepperd)."""
  R = np.asarray(R, LD).reshape(3, 3)
  tr = R[0, 0] + R[1, 1] + R[2, 2]
  cands = [1 + tr, 1 + R[0, 0] - R[1, 1] - R[2, 2], 1 - R[0, 0] + R[1, 1] - R[2, 2], 1 - R[0, 0] - R[1, 1] + R[2, 2]]
  k = int(np.argmax(cands)); s = np.sqrt(cands[k]) * 2
  if k == 0:
    q = [s / 4, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s]
  elif k == 1:
    q = [(R[2, 1] - R[1, 2]) / s, s / 4, (R[0, 1] + R[1, 0]) / s, (R[0, 2] + R[2, 0]) / s]
  elif k == 2:
    q = [(R[0, 2] - R[2, 0]) / s, (R[0, 1] + R[1, 0]) / s, s / 4, (R[1, 2] + R[2, 1]) / s]
  else:
    q = [(R[1, 0] - R[0, 1]) / s, (R[0, 2] + R[2, 0]) / s, (R[1, 2] + R[2, 1]) / s, s / 4]
  q = np.array(q, LD)
  return -q if q[0] < 0 else q


def angle_factor(m, qpos):
  """A hinge angle a (from qpos0) is known to a U in double, and every configuration-dependent output inherits that:
  the bounds scale by the largest."""
  a = [abs(qpos[m.jnt_qposadr[j]] - m.qpos0[m.jnt_qposadr[j]]) for j in range(m.njnt) if m.jnt_type[j] == ref.HINGE]
  return max([1.0] + a)


POS_FIELDS = dict(xpos='pos', xipos='pos', geom_xpos='pos', site_xpos='pos', subtree_com='pos', xmat='rot',
                  geom_xmat='rot', site_xmat='rot', cvel='vel', subtree_linvel='vel', qM='M', qfrc_bias='bias',
                  qfrc_passive='passive', actuator_force='actuator_force', qfrc_actuator='qfrc_actuator')


def check_forward(tier, what, m, run, e, R, qpos):
  """Every forward output of environment e against the reference R."""
  n = R['depth'] + m.nv
  S = R['scales']
  af = angle_factor(m, qpos)
  for f, sk in POS_FIELDS.items():
    got = run.get(f)[e]
    if got.size == 0:
      continue
    check(tier, what, f, got, R[f], n, S[sk] * af)
  xq = run.get('xquat')[e].reshape(-1, 4)
  qr = np.array([mat2quat(x) for x in R['xmat']])
  sign = np.where(xq[:, :1] < 0, -1.0, 1.0)
  check(tier, what, 'xquat', xq * sign, qr, n, af)
  assert int(run.get('nefc')[e]) == 0, (what, 'constraint rows in a contact-free, in-range state')
  # qacc: backward error against the reference's M and force
  qacc = run.get('qacc')[e].astype(LD)
  res = R['qM'].dot(qacc) - R['qfrc_smooth']
  Mn = float(np.max(np.sum(np.abs(R['qM']), axis=1)))
  check(tier, what, 'qacc (residual)', res, np.zeros_like(res), n, af * (Mn * float(np.max(np.abs(qacc))) + S['force']))


# ------------------------------------------------------------------------------------------------------------------
# the reference on closed forms
# ------------------------------------------------------------------------------------------------------------------
def _compile(body, opt='', extra=''):
  return mjcf_compile.compile_xml(f'<mujoco><compiler angle="radian"/><option timestep="0.01" {opt}/>'
                                  f'<worldbody>{body}</worldbody>{extra}</mujoco>')


def _close(a, b, rel=1e-17, what=''):
  a, b = np.asarray(a, LD), np.asarray(b, LD)
  err = float(np.max(np.abs(a - b))); s = max(1.0, float(np.max(np.abs(b))))
  assert err <= rel * s, (what, err, s)


def test_reference_pendulum():
  m_, l, Iyy, arm = 1.3, 0.7, 0.02, 0.05
  m = _compile(f'<body><joint name="h" type="hinge" axis="0 1 0" armature="{arm}"/>'
               f'<inertial pos="0 0 {-l}" mass="{m_}" diaginertia="0.03 {Iyy} 0.01"/></body>')
  for th, w in ((0.3, 0.0), (-2.1, 1.7), (np.pi, -3.0)):
    R = ref.forward(m, [th], [w])
    g = -float(m.opt.gravity[2])
    _close(R['qM'], [[LD(m_) * LD(l) ** 2 + LD(Iyy) + LD(arm)]], what='M')
    _close(R['qfrc_bias'], [LD(m_) * LD(g) * LD(l) * np.sin(LD(th))], rel=1e-16, what='bias')


def test_reference_double_pendulum():
  m1, m2, l1, l2, I1, I2 = 1.1, 0.6, 0.5, 0.4, 0.01, 0.02
  m = _compile(f'<body><joint type="hinge" axis="0 1 0"/><inertial pos="0 0 {-l1}" mass="{m1}" diaginertia="0.01 {I1} 0.01"/>'
               f'<body pos="0 0 {-l1}"><joint type="hinge" axis="0 1 0"/>'
               f'<inertial pos="0 0 {-l2}" mass="{m2}" diaginertia="0.01 {I2} 0.01"/></body></body>')
  rs = np.random.RandomState(0)
  for _ in range(3):
    q, v = rs.uniform(-3, 3, 2), rs.uniform(-4, 4, 2)
    R = ref.forward(m, q, v)
    L1, L2, M1, M2, J1, J2 = (LD(x) for x in (l1, l2, m1, m2, I1, I2))
    c2, s2 = np.cos(LD(q[1])), np.sin(LD(q[1]))
    M = [[M1 * L1 ** 2 + M2 * (L1 ** 2 + L2 ** 2 + 2 * L1 * L2 * c2) + J1 + J2, M2 * (L2 ** 2 + L1 * L2 * c2) + J2],
         [M2 * (L2 ** 2 + L1 * L2 * c2) + J2, M2 * L2 ** 2 + J2]]
    g = LD(-float(m.opt.gravity[2]))
    s1, s12 = np.sin(LD(q[0])), np.sin(LD(q[0]) + LD(q[1]))
    w1, w2 = LD(v[0]), LD(v[1])
    bias = [-M2 * L1 * L2 * s2 * (2 * w1 * w2 + w2 * w2) + (M1 + M2) * g * L1 * s1 + M2 * g * L2 * s12,
            M2 * L1 * L2 * s2 * w1 * w1 + M2 * g * L2 * s12]
    _close(R['qM'], M, what='M')
    _close(R['qfrc_bias'], bias, rel=1e-16, what='bias')


def test_reference_free_body_gyroscopic_torque():
  a, b, c = 0.3, 0.5, 0.9
  m = _compile(f'<body><freejoint/><inertial pos="0 0 0" mass="2" diaginertia="{a} {b} {c}"/></body>',
               extra='<option><flag gravity="disable"/></option>')
  rs = np.random.RandomState(1)
  for _ in range(3):
    q = np.concatenate([rs.randn(3), random_quat(rs)])
    v = rs.uniform(-5, 5, 6)
    R = ref.forward(m, q, v, disable=DSBL_CONTACT | DSBL_GRAVITY)
    w = v[3:].astype(LD); I = np.array([a, b, c], LD)
    _close(R['qfrc_bias'][:3], np.zeros(3), rel=1e-16, what='linear')
    _close(R['qfrc_bias'][3:], np.cross(w, I * w), rel=1e-16, what='omega x I omega')
    _close(R['qM'], np.diag(np.array([2, 2, 2, a, b, c], LD)), what='M')


def _slide_chain(n=4, damp=True):
  rs = np.random.RandomState(2)
  body, close = '', ''
  ms, ks, ds, qs = rs.uniform(0.5, 2, n), rs.uniform(1, 20, n), rs.uniform(0.1, 2, n) if damp else np.zeros(n), rs.uniform(-0.1, 0.1, n)
  for i in range(n):
    body += (f'<body pos="0.1 0 0"><joint type="slide" axis="1 0 0" stiffness="{float(ks[i])!r}" damping="{float(ds[i])!r}" '
             f'springref="{float(qs[i])!r}"/><inertial pos="0 0 0" mass="{float(ms[i])!r}" diaginertia="0.1 0.1 0.1"/>')
    close += '</body>'
  m = _compile(body + close, opt='gravity="0 0 0" integrator="RK4"')
  M = np.array([[sum(LD(ms[b]) for b in range(max(i, j), n)) for j in range(n)] for i in range(n)], LD)
  return m, M, np.diag(ks.astype(LD)), np.diag(ds.astype(LD)), qs.astype(LD)


def test_reference_slide_chain_steps_in_closed_form():
  """Linear spring-damper chain: RK4 is the degree-4 Taylor polynomial of exp(hA), the Euler steps their closed forms."""
  m, M, K, D, qs = _slide_chain()
  n = m.nv
  Minv = np.array([ref.solve(M, np.eye(n, dtype=LD)[:, i]) for i in range(n)]).T
  A = np.block([[np.zeros((n, n), LD), np.eye(n, dtype=LD)], [-Minv.dot(K), -Minv.dot(D)]])
  h = LD(m.opt.timestep)
  rs = np.random.RandomState(3)
  q, v = rs.uniform(-0.2, 0.2, n), rs.uniform(-1, 1, n)
  x = np.concatenate([q.astype(LD) - qs, v.astype(LD)])
  T, P = np.eye(2 * n, dtype=LD), np.eye(2 * n, dtype=LD)
  for k in range(1, 5):
    P = P.dot(h * A) / k; T = T + P
  y = T.dot(x)
  R = ref.rk4_step(m, q, v)
  _close(np.asarray(R['qpos'], LD) - qs, y[:n], rel=1e-17, what='rk4 q'); _close(R['qvel'], y[n:], rel=1e-17, what='rk4 v')
  f = -K.dot(q.astype(LD) - qs) - D.dot(v.astype(LD))
  for implicit in (False, True):
    E = ref.euler_step(m, q, v, disable=DSBL_CONTACT | (0 if implicit else DSBL_EULERDAMP))
    assert E['implicit'] == implicit
    a = ref.solve(M + h * D, f) if implicit else Minv.dot(f)
    v1 = v.astype(LD) + h * a
    _close(E['qvel'], v1, rel=1e-17, what='euler v'); _close(E['qpos'], q.astype(LD) + h * v1, rel=1e-17, what='euler q')


# ------------------------------------------------------------------------------------------------------------------
# the kernels against the reference
# ------------------------------------------------------------------------------------------------------------------
TREES = list(tree_models.MODELS)
DOFS = [dof_models.name(nv) for nv in sorted(set(dof_models.NV_TARGETS))]
FIXTURES = ['humanoid', 'quadruped', 'cheetah', 'cartpole', 'cmu_humanoid']
B = 2


def _forward_case(tier, name, m, states, run=None, overrides=None, what=None):
  run = run or Run(tier, m, len(states))
  for k, fld in enumerate(('qpos', 'qvel', 'ctrl', 'act')):
    run.set(fld, np.stack([s[k] for s in states]))
  run.forward()
  qpos_after = run.get('qpos')
  for e, (q, v, c, a) in enumerate(states):
    R = ref.forward(m, q, v, c, a, overrides=None if overrides is None else overrides[e])
    check_forward(tier, what or f'{name}[{e}]', m, run, e, R, q)
  return run, qpos_after


@pytest.mark.parametrize('tier', TIERS)
@pytest.mark.parametrize('name', TREES + DOFS + FIXTURES)
def test_forward(tier, name):
  m = load(name)
  rs = np.random.RandomState(zlib.crc32(name.encode()))
  _forward_case(tier, name, m, [random_state(m, rs, vscale=3.0) for _ in range(B)])


@pytest.mark.parametrize('tier', TIERS)
def test_actuator_clamps_active_at_both_ends(tier):
  m = load('wide64')
  rs = np.random.RandomState(5)
  states = [random_state(m, rs, vscale=3.0) for _ in range(3)]
  run, _ = _forward_case(tier, 'wide64', m, states)
  f = run.get('actuator_force')
  lim = np.nonzero(m.actuator_forcelimited)[0]
  assert np.any(f[:, lim] == m.actuator_forcerange[lim, 0]) and np.any(f[:, lim] == m.actuator_forcerange[lim, 1])


@pytest.mark.parametrize('tier', TIERS)
@pytest.mark.parametrize('flag', ['gravity', 'passive', 'actuation', 'clampctrl'])
def test_disable_flags(tier, flag):
  bit = dict(gravity=DSBL_GRAVITY, passive=DSBL_PASSIVE, actuation=DSBL_ACTUATION, clampctrl=DSBL_CLAMPCTRL)[flag]
  for name in ('multijoint', 'wide40'):
    m = load(name)
    m.opt.disableflags = int(m.opt.disableflags) | bit
    rs = np.random.RandomState(7)
    _forward_case(tier, name, m, [random_state(m, rs) for _ in range(B)], what=f'{name} without {flag}')


def _kernel_step_check(tier, what, m, run, e, q, v, c, a, rk4=False, overrides=None):
  """One step of environment e: Euler by backward error of its velocity update and integratePos of its own new
  velocity; RK4 by forward error against the reference step, scaled by M's condition number."""
  q1, v1 = run.get('qpos')[e], run.get('qvel')[e]
  act1 = run.get('act')[e] if m.na else np.zeros(0)
  h = float(m.opt.timestep)
  depth_nv = int(m.nlevel) + m.nv
  if rk4:
    S = ref.rk4_step(m, q, v, c, a, overrides=overrides)
    F = ref.forward(m, q, v, c, a, overrides=overrides)
    kappa = float(np.linalg.cond(np.asarray(F['qM'], np.float64)))
    vs = float(np.max(np.abs(v))) + h * float(np.max(np.abs(np.asarray(F['qacc'], np.float64))))
    check(tier, what, 'rk4 qvel', v1, S['qvel'], depth_nv, kappa * max(vs, 1e-300))
    check(tier, what, 'rk4 qpos', q1, S['qpos'], depth_nv, kappa * (F['scales']['pos'] + h * vs))
    if m.na:
      check(tier, what, 'rk4 act', act1, S['act'], depth_nv, kappa * (1 + float(np.max(np.abs(a)))))
    return
  S = ref.euler_step(m, q, v, c, a, overrides=overrides)
  A, f = S['A'], S['F']['qfrc_smooth']
  x = (v1.astype(LD) - np.asarray(v, LD)) / LD(h)
  res = A.dot(x) - f
  An = float(np.max(np.sum(np.abs(A), axis=1)))
  vround = An * (float(np.max(np.abs(v1))) + float(np.max(np.abs(v)))) / h
  check(tier, what, 'euler solve (residual)', res, np.zeros_like(res), depth_nv,
        An * float(np.max(np.abs(x))) + S['F']['scales']['force'] + vround)
  qi = ref.integrate_pos(m, q, v1, h)
  check(tier, what, 'integratePos', q1, qi, depth_nv, S['F']['scales']['pos'] + h * float(np.max(np.abs(v1))))
  if m.na:
    check(tier, what, 'act', act1, S['act'], depth_nv, 1 + float(np.max(np.abs(S['act']))))


STEP_CASES = [('multijoint', 'split'), ('wide40', 'split'), ('chain64', 'split'), ('welded100', 'split'), ('dof12', 'split'),
              ('dof27', 'split'), ('dof33', 'split'), ('quadruped', 'split'), ('multijoint', 'nonlegacy'),
              ('wide64', 'nonlegacy'), ('dof18', 'tn0'), ('multijoint', 'nosplit'), ('dof22', 'nosplit'),
              ('multijoint', 'noeulerdamp'), ('cheetah', 'noeulerdamp')]


@pytest.mark.parametrize('tier', TIERS)
@pytest.mark.parametrize('name,path', STEP_CASES)
def test_euler_step(tier, name, path, monkeypatch):
  """step(1): with the legacy ordering on the split kernels (compile-time size for nv in B200MJ_NV_LIST, runtime size
  otherwise), with the non-legacy ordering on the fused kernel, with B200MJ_TN=0 and B200MJ_SPLIT=0 (read when the
  model is created), and with eulerdamp disabled."""
  m = load(name)
  if path == 'noeulerdamp':
    m.opt.disableflags = int(m.opt.disableflags) | DSBL_EULERDAMP
  if path == 'tn0':
    monkeypatch.setenv('B200MJ_TN', '0')
  if path == 'nosplit':
    monkeypatch.setenv('B200MJ_SPLIT', '0')
  rs = np.random.RandomState(11)
  states = [random_state(m, rs, vscale=2.0) for _ in range(B)]
  run = Run(tier, m, B, legacy=path != 'nonlegacy')
  for k, fld in enumerate(('qpos', 'qvel', 'ctrl', 'act')):
    run.set(fld, np.stack([s[k] for s in states]))
  run.step(1)
  for e, (q, v, c, a) in enumerate(states):
    _kernel_step_check(tier, f'{name}/{path}[{e}]', m, run, e, q, v, c, a)


@pytest.mark.parametrize('tier', TIERS)
@pytest.mark.parametrize('name', ['multijoint', 'wide33', 'cartpole', 'dof12', 'welded65'])
def test_rk4_step(tier, name):
  m = load(name)
  m.opt.integrator = 1
  rs = np.random.RandomState(13)
  states = [random_state(m, rs) for _ in range(B)]
  run = Run(tier, m, B)
  for k, fld in enumerate(('qpos', 'qvel', 'ctrl', 'act')):
    run.set(fld, np.stack([s[k] for s in states]))
  run.step(1)
  for e, (q, v, c, a) in enumerate(states):
    _kernel_step_check(tier, f'{name}/rk4[{e}]', m, run, e, q, v, c, a, rk4=True)


@pytest.mark.parametrize('tier', TIERS)
def test_applied_forces(tier):
  m = load('multijoint')
  rs = np.random.RandomState(17)
  states = [random_state(m, rs) for _ in range(B)]
  qf, xf = rs.uniform(-1, 1, (B, m.nv)), rs.uniform(-1, 1, (B, m.nbody, 6))
  run = Run(tier, m, B, applied=True)
  run.set('qfrc_applied', qf); run.set('xfrc_applied', xf)
  for k, fld in enumerate(('qpos', 'qvel', 'ctrl', 'act')):
    run.set(fld, np.stack([s[k] for s in states]))
  run.forward()
  for e, (q, v, c, a) in enumerate(states):
    R = ref.forward(m, q, v, c, a, qfrc_applied=qf[e], xfrc_applied=xf[e])
    check_forward(tier, f'applied[{e}]', m, run, e, R, q)


# ------------------------------------------------------------------------------------------------------------------
# states at the edges
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('tier', TIERS)
def test_quaternion_norms_and_write_back(tier):
  """normalize4 (mju_normalize4): a quaternion whose norm is within mjMINVAL of 1 is used and kept as it is; any other
  is divided by its norm and written back to qpos by forward(); a norm below mjMINVAL becomes (1, 0, 0, 0)."""
  m = load('multijoint')
  quat_adr = [m.jnt_qposadr[j] + (3 if m.jnt_type[j] == ref.FREE else 0) for j in range(m.njnt)
              if m.jnt_type[j] in (ref.FREE, ref.BALL)]
  rs = np.random.RandomState(19)
  states, scales = [], (1 + 2.2e-16, 1 - 1.1e-16, 1 + 1e-10, 1 - 1e-10, 1.3, 0.7, 0.0)
  for s in scales:
    q, v, c, a = random_state(m, rs)
    for qa in quat_adr:
      q[qa:qa + 4] *= s
    states.append((q, v, c, a))
  run = Run(tier, m, len(states))
  for k, fld in enumerate(('qpos', 'qvel', 'ctrl', 'act')):
    run.set(fld, np.stack([st[k] for st in states]))
  run.forward()
  qout = run.get('qpos')
  for e, (s, (q, v, c, a)) in enumerate(zip(scales, states)):
    for qa in quat_adr:
      got, given = qout[e, qa:qa + 4], q[qa:qa + 4]
      n = np.sqrt(np.sum(given.astype(LD) ** 2))
      if s == 0.0:
        np.testing.assert_array_equal(got, [1, 0, 0, 0])
      elif abs(float(n) - 1) <= ref.MINVAL:
        np.testing.assert_array_equal(got, given)
      else:
        assert float(np.max(np.abs(got.astype(LD) - given / n))) <= 4 * U, (s, got, given)
    qn = q.copy()
    for qa in quat_adr:
      qn[qa:qa + 4] = qout[e, qa:qa + 4]
    check_forward(tier, f'quaternion norm {s!r}', m, run, e, ref.forward(m, qn, v, c, a), qn)


@pytest.mark.parametrize('tier', TIERS)
def test_hinge_angles_at_the_edges(tier):
  m = load('chain64')
  rs = np.random.RandomState(23)
  states = []
  for ang in (0.0, np.pi, -np.pi, 1e4):
    q, v, c, a = random_state(m, rs)
    q[:] = np.asarray(m.qpos0) + ang
    states.append((q, v, c, a))
  _forward_case(tier, 'chain64 edge angles', m, states)


@pytest.mark.parametrize('tier', TIERS)
def test_quaternion_integration_edges(tier):
  """Free and ball angular speeds with |w| h = 0, 1e-12, about pi and beyond 2 pi, and speeds up to 1e3. The engine
  skips the update when |w| < mjMINVAL, where mju_quatIntegrate rotates by |w| h about (1, 0, 0) after normalising:
  the position stage has already normalised the quaternion in place, and the rotation, below 1e-17 rad, is under half
  an ulp of every component of a unit quaternion. So the step must leave such a quaternion bitwise as it was."""
  m = load('multijoint')
  m.opt.disableflags = int(m.opt.disableflags) | DSBL_GRAVITY
  h = float(m.opt.timestep)
  rs = np.random.RandomState(29)
  cases = [0.0, 1e-12 / h, 3.1 / h, 7.0 / h, 1e3, 1e-17]
  states = []
  for wn in cases:
    q, v, c, a = random_state(m, rs)
    for j in range(m.njnt):
      if m.jnt_type[j] in (ref.FREE, ref.BALL):
        da = m.jnt_dofadr[j] + (3 if m.jnt_type[j] == ref.FREE else 0)
        d = rs.randn(3); v[da:da + 3] = wn * d / np.linalg.norm(d)
    states.append((q, v, c, a))
  run = Run(tier, m, len(states), legacy=False)
  for k, fld in enumerate(('qpos', 'qvel', 'ctrl', 'act')):
    run.set(fld, np.stack([st[k] for st in states]))
  run.step(1)
  for e, (wn, (q, v, c, a)) in enumerate(zip(cases, states)):
    _kernel_step_check(tier, f'|w| = {wn!r}', m, run, e, q, v, c, a)
  # a state with only tiny angular speeds: the quaternions after one step are those the position stage normalised
  q, v, c, a = random_state(m, rs)
  v[:] = 0
  for j in range(m.njnt):
    if m.jnt_type[j] in (ref.FREE, ref.BALL):
      da = m.jnt_dofadr[j] + (3 if m.jnt_type[j] == ref.FREE else 0)
      v[da:da + 3] = [1e-17, -3e-18, 0.0]
  m2 = copy.deepcopy(m)
  m2.opt.disableflags = int(m2.opt.disableflags) | DSBL_PASSIVE | DSBL_ACTUATION
  run = Run(tier, m2, 1, legacy=False)
  run.set('qpos', q[None]); run.set('qvel', v[None])
  run.forward()
  qn = run.get('qpos')[0]
  run.set('qvel', v[None])
  run.step(1)
  q1 = run.get('qpos')[0]
  for j in range(m.njnt):
    if m.jnt_type[j] in (ref.FREE, ref.BALL):
      qa = m.jnt_qposadr[j] + (3 if m.jnt_type[j] == ref.FREE else 0)
      np.testing.assert_array_equal(q1[qa:qa + 4], qn[qa:qa + 4])


# ------------------------------------------------------------------------------------------------------------------
# per-environment model fields
# ------------------------------------------------------------------------------------------------------------------
ENV_FIELDS = ('body_mass', 'body_inertia', 'body_ipos', 'geom_friction', 'geom_solref', 'geom_solimp', 'dof_damping',
              'dof_armature', 'jnt_stiffness', 'actuator_gainprm', 'actuator_biasprm')


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['multijoint', 'wide40', 'dof27'])
def test_env_model_fields(name):
  """All eleven per-environment fields randomised per environment; the reference reads each environment's rows and,
  like the engine, the model's shared body_subtreemass."""
  m = load(name)
  rs = np.random.RandomState(31)
  Bn = 3
  over = []
  for e in range(Bn):
    o = {}
    for f in ENV_FIELDS:
      base = np.asarray(getattr(m, f), np.float64)
      o[f] = base * rs.uniform(0.8, 1.2, base.shape) if f != 'body_ipos' else base + rs.uniform(-0.02, 0.02, base.shape)
    o['dof_damping'][rs.rand(m.nv) < 0.3] = 0
    over.append(o)
  run = Run('gpu', m, Bn, env_fields=ENV_FIELDS)
  for f in ENV_FIELDS:
    run.set_env(f, np.stack([o[f] for o in over]))
  states = [random_state(m, rs) for _ in range(Bn)]
  _forward_case('gpu', name, m, states, run=run, overrides=over, what=f'{name} per-environment')
  for k, fld in enumerate(('qpos', 'qvel', 'ctrl', 'act')):
    run.set(fld, np.stack([s[k] for s in states]))
  run.step(1)
  for e, (q, v, c, a) in enumerate(states):
    _kernel_step_check('gpu', f'{name} per-environment step[{e}]', m, run, e, q, v, c, a, overrides=over[e])
