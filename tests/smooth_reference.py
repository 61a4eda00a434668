"""Smooth dynamics from first principles, in extended precision, read from a compiled `Model`'s tables.

This is the yardstick `tests/test_smooth_dynamics.py` holds the kernels to. It shares no code and no recursion with the
engine or with `oracle/mjoracle.cpp`: there are no motion subspaces (`cdof`), no composite inertias and no recursive
Newton-Euler. Each body's frame is composed directly, each body's Jacobians are written down joint by joint, and

    M         = sum_b  m_b Jv_b^T Jv_b + Jw_b^T I_b Jw_b  +  diag(armature)
    qfrc_bias = sum_b  Jv_b^T m_b (Jdot_v qdot - g)  +  Jw_b^T (I_b Jdot_w qdot + w_b x I_b w_b)

with Jv_b the Jacobian of the body's centre of mass `xipos`, Jw_b its angular Jacobian and I_b its inertia about the
centre of mass in world axes. `Jdot qdot` is the derivative of the body's velocity along q(t) = integratePos(q, t qdot),
taken by central differences in mpmath at 50 digits: the second derivative of `xipos` and the first of the angular
velocity.

MuJoCo's coordinate conventions, which the reference follows:
  * hinge and slide joints are measured from `qpos0`; a fixed tendon's length is sum(coef * qpos), not from `qpos0`;
  * a free joint's linear velocity is in the world frame, its angular velocity in the body frame;
  * a ball joint's angular velocity is in the frame of its body (the ball is the body's last joint), its axes the
    columns of the body's final rotation;
  * `cvel` is [angular; linear] velocity of the body, the linear part at the subtree centre of mass of the body's root;
  * quaternions are normalised when read (mju_normalize4) and integrated as q <- q * exp(h w / 2) with w in the body
    frame (mju_quatIntegrate);
  * `subtree_com` and `subtree_linvel` divide by the model's `body_subtreemass`, which per-environment masses do not
    change (nothing derived is recomputed), and a subtree lighter than mjMINVAL takes the body's own `xipos`.

Arithmetic is np.longdouble (x86-64 extended, 64-bit mantissa); solves are Gaussian elimination with partial pivoting
in the same type.
"""
from __future__ import annotations

import mpmath
import numpy as np

LD = np.longdouble
assert np.finfo(LD).nmant >= 63, 'the reference needs x86-64 extended precision (64-bit long double)'

MINVAL = 1e-15
FREE, BALL, SLIDE, HINGE = 0, 1, 2, 3
DSBL_PASSIVE, DSBL_GRAVITY, DSBL_CLAMPCTRL, DSBL_ACTUATION, DSBL_EULERDAMP = 1 << 5, 1 << 6, 1 << 7, 1 << 10, 1 << 14
MP_DPS = 50


class _Num:
  """Scalar backend: np.longdouble arrays, or numpy object arrays of mpmath numbers."""

  def __init__(self, mp):
    self.mp = mp
    if mp:
      self.sin, self.cos, self.sqrt = mpmath.sin, mpmath.cos, mpmath.sqrt
    else:
      self.sin, self.cos, self.sqrt = np.sin, np.cos, np.sqrt

  def arr(self, x):
    x = np.asarray(x)
    if not self.mp:
      return x.astype(LD)
    return np.array([mpmath.mpf(float(v)) if x.dtype != object else mpmath.mpf(v) for v in x.reshape(-1)],
                    dtype=object).reshape(x.shape)

  def eye(self):
    return self.arr(np.eye(3))


_LDN, _MPN = _Num(False), _Num(True)


class Params:
  """The model's tables, with this environment's own rows for the per-environment fields where given."""

  def __init__(self, model, overrides=None):
    self.model, self.over = model, dict(overrides or {})

  def __getattr__(self, name):
    if name in ('model', 'over'):
      raise AttributeError(name)
    if name in self.over:
      return np.asarray(self.over[name], np.float64).reshape(np.shape(getattr(self.model, name)))
    return getattr(self.model, name)


def _unit_quat_mat(N, q):
  n = N.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
  w, x, y, z = q[0] / n, q[1] / n, q[2] / n, q[3] / n
  return N.arr(np.zeros((3, 3))) + np.array(
      [[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
       [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
       [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]], dtype=object if N.mp else LD)


def _rodrigues(N, axis, angle):
  """Rotation by `angle` about the direction of `axis`: I + sin K + (1 - cos) K^2 with K the cross-product matrix of
  the unit axis. (Normalised here: a composed rotation that is off orthogonal by e tilts the next axis' length by e,
  and Rodrigues' formula with that axis squares the defect, so along a chain it would grow geometrically.)"""
  axis = axis / N.sqrt(axis[0] * axis[0] + axis[1] * axis[1] + axis[2] * axis[2])
  K = N.arr(np.zeros((3, 3)))
  K[0, 1], K[0, 2], K[1, 0], K[1, 2], K[2, 0], K[2, 1] = -axis[2], axis[1], axis[2], -axis[0], -axis[1], axis[0]
  return N.eye() + N.sin(angle) * K + (1 - N.cos(angle)) * K.dot(K)


def _quat_normalize(N, q):
  n = N.sqrt(sum(v * v for v in q))
  return q / n


def kinematics(P, qpos, N=_LDN):
  """Frames of every body, joint, geom and site. Returns a dict of arrays (backend N)."""
  m = P.model
  nb, nj = m.nbody, m.njnt
  q = N.arr(qpos)
  q0 = N.arr(m.qpos0)
  R = [N.eye() for _ in range(nb)]
  x = [N.arr(np.zeros(3)) for _ in range(nb)]
  anchor = [None] * nj
  axis = [None] * nj
  for b in range(1, nb):
    p = m.body_parentid[b]
    Rb = R[p].dot(_unit_quat_mat(N, N.arr(m.body_quat[b])))
    xb = x[p] + R[p].dot(N.arr(m.body_pos[b]))
    for j in range(m.body_jntadr[b], m.body_jntadr[b] + m.body_jntnum[b]):
      t, qa = m.jnt_type[j], m.jnt_qposadr[j]
      jp, ja = N.arr(m.jnt_pos[j]), N.arr(m.jnt_axis[j])
      if t == FREE:
        xb, Rb = q[qa:qa + 3].copy(), _unit_quat_mat(N, q[qa + 3:qa + 7])
        anchor[j], axis[j] = xb.copy(), Rb.dot(ja)
        continue
      a = xb + Rb.dot(jp)
      anchor[j], axis[j] = a, Rb.dot(ja)
      if t == SLIDE:
        xb = xb + axis[j] * (q[qa] - q0[qa])
      elif t == HINGE:
        Q = _rodrigues(N, axis[j], q[qa] - q0[qa])
        Rb, xb = Q.dot(Rb), a + Q.dot(xb - a)
      else:
        Rb = Rb.dot(_unit_quat_mat(N, q[qa:qa + 4]))
        xb = a - Rb.dot(jp)
    R[b], x[b] = Rb, xb
  ipos = N.arr(P.body_ipos)
  xipos = [x[b] + R[b].dot(ipos[b]) for b in range(nb)]
  ximat = [R[b].dot(_unit_quat_mat(N, N.arr(m.body_iquat[b]))) for b in range(nb)]
  out = dict(R=R, x=x, anchor=anchor, axis=axis, xipos=xipos, ximat=ximat)
  for kind in ('geom', 'site'):
    bid = getattr(m, f'{kind}_bodyid')
    pos, quat = getattr(m, f'{kind}_pos'), getattr(m, f'{kind}_quat')
    out[f'{kind}_xpos'] = [x[bid[g]] + R[bid[g]].dot(N.arr(pos[g])) for g in range(len(bid))]
    out[f'{kind}_xmat'] = [R[bid[g]].dot(_unit_quat_mat(N, N.arr(quat[g]))) for g in range(len(bid))]
  return out


def dof_directions(m, K, N=_LDN):
  """Per dof: (angular direction w, translation direction t, point a), so that the dof's unit velocity moves a point p
  of a body it carries with linear velocity t + w x (p - a) and angular velocity w."""
  z = N.arr(np.zeros(3))
  W, T, A = [z] * m.nv, [z] * m.nv, [z] * m.nv
  for j in range(m.njnt):
    t, da, b = m.jnt_type[j], m.jnt_dofadr[j], m.jnt_bodyid[j]
    if t == FREE:
      for k in range(3):
        e = N.arr(np.eye(3)[k])
        T[da + k] = e
        W[da + 3 + k], A[da + 3 + k] = K['R'][b][:, k].copy(), K['anchor'][j]
    elif t == BALL:
      for k in range(3):
        W[da + k], A[da + k] = K['R'][b][:, k].copy(), K['anchor'][j]
    elif t == SLIDE:
      T[da] = K['axis'][j]
    else:
      W[da], A[da] = K['axis'][j], K['anchor'][j]
  return W, T, A


def ancestors_mask(m):
  """mask[b, i]: dof i moves body b (its joint's body is b or an ancestor of b)."""
  mask = np.zeros((m.nbody, m.nv), bool)
  for b in range(1, m.nbody):
    a = b
    while a > 0:
      d0, dn = m.body_dofadr[a], m.body_dofnum[a]
      mask[b, d0:d0 + dn] = True
      a = m.body_parentid[a]
  return mask


def jacobians(m, K, point_of_body):
  """(Jv[b] at point_of_body[b], Jw[b]) as [nbody, 3, nv] longdouble arrays."""
  W, T, A = (np.array([v for v in lst], LD).reshape(m.nv, 3) for lst in dof_directions(m, K))
  mask = ancestors_mask(m)
  Jv = np.zeros((m.nbody, 3, m.nv), LD)
  Jw = np.zeros((m.nbody, 3, m.nv), LD)
  for b in range(1, m.nbody):
    p = np.asarray(point_of_body[b], LD)
    cols = T + np.cross(W, p[None, :] - A)
    Jv[b] = (cols * mask[b][:, None]).T
    Jw[b] = (W * mask[b][:, None]).T
  return Jv, Jw


def body_inertia_world(P, K):
  inert = np.asarray(P.body_inertia, np.float64)
  return [K['ximat'][b].dot(np.diag(inert[b].astype(LD))).dot(K['ximat'][b].T) for b in range(P.model.nbody)]


def integrate_pos(m, qpos, qvel, h, N=_LDN):
  """mj_integratePos: hinge / slide q + h v; free position + h v; quaternions q * exp(h w / 2), w in the body frame."""
  q, v = N.arr(qpos).copy(), N.arr(qvel)
  h = N.arr(np.array(h)) if not isinstance(h, (mpmath.mpf,)) else h
  for j in range(m.njnt):
    t, qa, da = m.jnt_type[j], m.jnt_qposadr[j], m.jnt_dofadr[j]
    if t in (SLIDE, HINGE):
      q[qa] = q[qa] + h * v[da]
      continue
    if t == FREE:
      q[qa:qa + 3] = q[qa:qa + 3] + h * v[da:da + 3]
      qa, da = qa + 3, da + 3
    w = v[da:da + 3]
    nw = N.sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2])
    quat = _quat_normalize(N, q[qa:qa + 4])
    if nw == 0:
      q[qa:qa + 4] = quat
      continue
    half = h * nw / 2
    s, c = N.sin(half), N.cos(half)
    r = [c, s * w[0] / nw, s * w[1] / nw, s * w[2] / nw]
    a = quat
    q[qa:qa + 4] = [a[0] * r[0] - a[1] * r[1] - a[2] * r[2] - a[3] * r[3],
                    a[0] * r[1] + a[1] * r[0] + a[2] * r[3] - a[3] * r[2],
                    a[0] * r[2] - a[1] * r[3] + a[2] * r[0] + a[3] * r[1],
                    a[0] * r[3] + a[1] * r[2] - a[2] * r[1] + a[3] * r[0]]
  return q


def _body_motion_mp(P, qpos, qvel, t):
  """(xipos[b], angular velocity[b]) at q(t) = integratePos(q, t qdot), in mpmath."""
  m = P.model
  N = _MPN
  qt = integrate_pos(m, qpos, qvel, t, N)
  K = kinematics(P, qt, N)
  W, T, A = dof_directions(m, K, N)
  v = N.arr(qvel)
  mask = ancestors_mask(m)
  om = [sum((W[i] * v[i] for i in np.nonzero(mask[b])[0]), N.arr(np.zeros(3))) for b in range(m.nbody)]
  return K['xipos'], om


def jdot_qdot(P, qpos, qvel):
  """Per body: (d^2/dt^2 xipos, d/dt omega) along q(t) = integratePos(q, t qdot), central differences at 50 digits."""
  m = P.model
  with mpmath.workdps(MP_DPS):
    eps = mpmath.mpf(10) ** -14 / (1 + float(np.max(np.abs(qvel), initial=0)))
    xp, wp = _body_motion_mp(P, qpos, qvel, eps)
    x0, _ = _body_motion_mp(P, qpos, qvel, mpmath.mpf(0))
    xm, wm = _body_motion_mp(P, qpos, qvel, -eps)
    acc = np.array([[LD(str((xp[b][k] - 2 * x0[b][k] + xm[b][k]) / eps ** 2)) for k in range(3)] for b in range(m.nbody)])
    alp = np.array([[LD(str((wp[b][k] - wm[b][k]) / (2 * eps))) for k in range(3)] for b in range(m.nbody)])
  return acc, alp


def solve(A, b):
  """Gaussian elimination with partial pivoting in long double."""
  A = np.array(A, LD); x = np.array(b, LD)
  n = len(x)
  for k in range(n):
    p = k + int(np.argmax(np.abs(A[k:, k])))
    if p != k:
      A[[k, p]] = A[[p, k]]; x[[k, p]] = x[[p, k]]
    f = A[k + 1:, k] / A[k, k]
    A[k + 1:, k:] -= f[:, None] * A[k, k:][None, :]
    x[k + 1:] -= f * x[k]
  for k in range(n - 1, -1, -1):
    x[k] = (x[k] - A[k, k + 1:].dot(x[k + 1:])) / A[k, k]
  return x


def tendon_rows(m):
  """Fixed tendons' Jacobians [ntendon, nv] (coefficients on their joints' dofs) and qpos coefficients [ntendon, nq]."""
  Jt = np.zeros((m.ntendon, m.nv), LD)
  Lt = np.zeros((m.ntendon, m.nq), LD)
  for t in range(m.ntendon):
    for w in range(m.tendon_adr[t], m.tendon_adr[t] + m.tendon_num[t]):
      j = m.wrap_objid[w]
      Jt[t, m.jnt_dofadr[j]] += LD(m.wrap_prm[w])
      Lt[t, m.jnt_qposadr[j]] += LD(m.wrap_prm[w])
  return Jt, Lt


def actuation(P, qpos, qvel, ctrl, act, disable):
  """(actuator_force, qfrc_actuator, act_dot, and their absolute-value scales) per mj_fwdActuation."""
  m = P.model
  nu = m.nu
  force = np.zeros(nu, LD); actdot = np.zeros(m.na, LD); fscale = np.zeros(nu, LD)
  moment = np.zeros((nu, m.nv), LD)
  Jt, Lt = tendon_rows(m)
  q, v = np.asarray(qpos, LD), np.asarray(qvel, LD)
  gp, bp = np.asarray(P.actuator_gainprm, np.float64).reshape(nu, 3), np.asarray(P.actuator_biasprm, np.float64).reshape(nu, 3)
  for a in range(nu):
    gear = LD(m.actuator_gear[a] if np.ndim(m.actuator_gear[a]) == 0 else m.actuator_gear[a][0])
    if m.actuator_trntype[a] == 0:
      j = m.actuator_trnid[a]
      moment[a, m.jnt_dofadr[j]] = gear
      length = gear * q[m.jnt_qposadr[j]]
    else:
      moment[a] = gear * Jt[m.actuator_trnid[a]]
      length = gear * Lt[m.actuator_trnid[a]].dot(q)
    vel = moment[a].dot(v)
    if disable & DSBL_ACTUATION:
      continue
    c = LD(ctrl[a])
    if m.actuator_ctrllimited[a] and not disable & DSBL_CLAMPCTRL:
      c = min(max(c, LD(m.actuator_ctrlrange[a][0])), LD(m.actuator_ctrlrange[a][1]))
    aa, dt = m.actuator_actadr[a], m.actuator_dyntype[a]
    inp = c
    if dt == 1:
      actdot[aa], inp = c, LD(act[aa])
    elif dt == 2:
      actdot[aa], inp = (c - LD(act[aa])) / max(LD(MINVAL), LD(m.actuator_dynprm[a] if np.ndim(m.actuator_dynprm[a]) == 0
                                                                  else m.actuator_dynprm[a][0])), LD(act[aa])
    gain, gsc = LD(gp[a, 0]), abs(LD(gp[a, 0]))
    if m.actuator_gaintype[a] == 1:
      gain += LD(gp[a, 1]) * length + LD(gp[a, 2]) * vel
      gsc += abs(LD(gp[a, 1]) * length) + abs(LD(gp[a, 2]) * vel)
    bias = bsc = LD(0)
    if m.actuator_biastype[a] == 1:
      bias = LD(bp[a, 0]) + LD(bp[a, 1]) * length + LD(bp[a, 2]) * vel
      bsc = abs(LD(bp[a, 0])) + abs(LD(bp[a, 1]) * length) + abs(LD(bp[a, 2]) * vel)
    f = gain * inp + bias
    fscale[a] = gsc * abs(inp) + bsc
    if m.actuator_forcelimited[a]:
      f = min(max(f, LD(m.actuator_forcerange[a][0])), LD(m.actuator_forcerange[a][1]))
    force[a] = f
  return force, moment.T.dot(force), actdot, fscale, np.abs(moment).T.dot(fscale)


def forward(model, qpos, qvel, ctrl=None, act=None, qfrc_applied=None, xfrc_applied=None, disable=None, overrides=None):
  """Every smooth output of mj_forward with contacts off, plus the scales the tests' bounds use."""
  P = Params(model, overrides)
  m = model
  disable = int(m.opt.disableflags if disable is None else disable)
  ctrl = np.zeros(m.nu) if ctrl is None else ctrl
  act = np.zeros(m.na) if act is None else act
  qpos, qvel = np.asarray(qpos, np.float64), np.asarray(qvel, np.float64)
  K = kinematics(P, qpos)
  nb, nv = m.nbody, m.nv
  mass = np.asarray(P.body_mass, np.float64).astype(LD)
  Jv, Jw = jacobians(m, K, K['xipos'])
  Iw = body_inertia_world(P, K)
  M = np.diag(np.asarray(P.dof_armature, np.float64).astype(LD))
  for b in range(1, nb):
    M += mass[b] * Jv[b].T.dot(Jv[b]) + Jw[b].T.dot(Iw[b]).dot(Jw[b])
  v = qvel.astype(LD)
  om = np.array([Jw[b].dot(v) for b in range(nb)])
  vcom = np.array([Jv[b].dot(v) for b in range(nb)])
  g = np.zeros(3, LD) if disable & DSBL_GRAVITY else np.asarray(m.opt.gravity, np.float64).astype(LD)
  acc, alp = jdot_qdot(P, qpos, qvel)
  bias = np.zeros(nv, LD)
  for b in range(1, nb):
    Io = Iw[b].dot(om[b])
    bias += Jv[b].T.dot(mass[b] * (acc[b] - g)) + Jw[b].T.dot(Iw[b].dot(alp[b]) + np.cross(om[b], Io))
  # subtree centres of mass and linear momenta, divided by the model's subtree masses
  xipos = np.array(K['xipos'], LD)
  stm = np.asarray(m.body_subtreemass, np.float64)
  mx, mv = mass[:, None] * xipos, mass[:, None] * vcom
  mx[0] = mv[0] = 0
  smx, smv = mx.copy(), mv.copy()
  for b in range(nb - 1, 0, -1):
    smx[m.body_parentid[b]] += smx[b]; smv[m.body_parentid[b]] += smv[b]
  scom = np.array([xipos[b] if stm[b] < MINVAL else smx[b] / LD(stm[b]) for b in range(nb)])
  slinvel = smv / np.maximum(LD(MINVAL), stm.astype(LD))[:, None]
  cvel = np.zeros((nb, 6), LD)
  for b in range(1, nb):
    r = scom[m.body_rootid[b]]
    cvel[b, :3] = om[b]
    cvel[b, 3:] = vcom[b] + np.cross(om[b], r - xipos[b])
  # passive forces: springs about qpos_spring (hinge, slide), dof damping
  passive = np.zeros(nv, LD); pscale = np.zeros(nv, LD)
  if not disable & DSBL_PASSIVE:
    stiff, damp = np.asarray(P.jnt_stiffness, np.float64), np.asarray(P.dof_damping, np.float64)
    for i in range(nv):
      j = m.dof_jntid[i]
      if m.jnt_type[j] in (SLIDE, HINGE) and stiff[j] != 0:
        qa = m.jnt_qposadr[j]
        s = LD(stiff[j]) * (LD(qpos[qa]) - LD(m.qpos_spring[qa]))
        passive[i] -= s; pscale[i] += abs(s)
      passive[i] -= LD(damp[i]) * v[i]; pscale[i] += abs(LD(damp[i]) * v[i])
  force, qfrc_act, actdot, fscale, qascale = actuation(P, qpos, qvel, ctrl, act, disable)
  applied = np.zeros(nv, LD)
  if qfrc_applied is not None:
    applied += np.asarray(qfrc_applied, LD)
  if xfrc_applied is not None:
    xf = np.asarray(xfrc_applied, LD).reshape(nb, 6)
    for b in range(1, nb):
      applied += Jv[b].T.dot(xf[b, :3]) + Jw[b].T.dot(xf[b, 3:])
  f = passive - bias + qfrc_act + applied
  qacc = solve(M, f)
  # scales of the bounds: extent L of the tree, speed V, and absolute-value sums of the forces
  L = 1 + max(float(np.max(np.abs(xipos))), float(np.max(np.abs(np.array(K['x'], LD)))),
              max((float(np.max(np.abs(np.array(K[k], LD)))) for k in ('geom_xpos', 'site_xpos') if len(K[k])), default=0))
  W = float(np.sum(np.abs(qvel)))
  V = W * L
  Itr = sum(float(np.sum(np.asarray(P.body_inertia, np.float64)[b])) for b in range(nb))
  mtot = float(np.sum(mass))
  S_bias = mtot * (float(np.max(np.abs(g))) * L + V * V) + Itr * W * W
  scales = dict(pos=L, rot=1.0, vel=max(V, 1e-300), M=float(np.max(np.abs(np.diag(M)))), bias=max(S_bias, 1e-300),
                passive=float(np.max(pscale, initial=0)), actuator_force=float(np.max(fscale, initial=0)),
                qfrc_actuator=float(np.max(qascale, initial=0)),
                force=S_bias + float(np.max(pscale, initial=0)) + float(np.max(qascale, initial=0)) +
                float(np.max(np.abs(applied), initial=0)))
  return dict(xpos=np.array(K['x'], LD), xmat=np.array([R.reshape(9) for R in K['R']]), xipos=xipos,
              geom_xpos=np.array(K['geom_xpos'], LD).reshape(-1, 3), geom_xmat=np.array([R.reshape(9) for R in K['geom_xmat']], LD).reshape(-1, 9),
              site_xpos=np.array(K['site_xpos'], LD).reshape(-1, 3), site_xmat=np.array([R.reshape(9) for R in K['site_xmat']], LD).reshape(-1, 9),
              subtree_com=scom, subtree_linvel=slinvel, cvel=cvel, qM=M, qfrc_bias=bias, qfrc_passive=passive,
              actuator_force=force, qfrc_actuator=qfrc_act, act_dot=actdot, qfrc_smooth=f, qacc=qacc, scales=scales,
              depth=int(m.nlevel), kin=K)


def euler_step(model, qpos, qvel, ctrl=None, act=None, disable=None, overrides=None, **kw):
  """mj_Euler: act + h act_dot (clamped to actrange), qvel + h qacc -- or, when some dof is damped and eulerdamp is on,
  qvel + h (M + h diag(damping))^-1 f -- then qpos by integratePos with the new velocity."""
  m = model
  P = Params(model, overrides)
  disable = int(m.opt.disableflags if disable is None else disable)
  act = np.zeros(m.na) if act is None else act
  F = forward(model, qpos, qvel, ctrl, act, disable=disable, overrides=overrides, **kw)
  h = LD(m.opt.timestep)
  damp = np.asarray(P.dof_damping, np.float64)
  implicit = bool(np.any(damp > 0)) and not disable & DSBL_EULERDAMP
  A = F['qM'] + (h * np.diag(damp.astype(LD)) if implicit else 0)
  acc = solve(A, F['qfrc_smooth']) if implicit else F['qacc']
  v1 = np.asarray(qvel, LD) + h * acc
  q1 = integrate_pos(m, qpos, v1, h)
  return dict(qpos=q1, qvel=v1, act=_advance_act(m, act, F['act_dot'], h), implicit=implicit, A=A, F=F)


def _advance_act(m, act, actdot, h):
  a = np.asarray(act, LD) + h * actdot
  for u in range(m.nu):
    aa = m.actuator_actadr[u]
    if aa >= 0 and m.actuator_actlimited[u]:
      a[aa] = min(max(a[aa], LD(m.actuator_actrange[u][0])), LD(m.actuator_actrange[u][1]))
  return a


def rk4_step(model, qpos, qvel, ctrl=None, act=None, disable=None, overrides=None):
  """mj_RK4: the classical tableau (stage weights 1/2, 1/2, 1; final weights 1/6, 1/3, 1/3, 1/6). Stage i starts from
  X0 advanced by a_i h F_{i-1}: positions by integratePos of the start positions with the previous stage's velocity,
  velocities and activations linearly; the final positions integratePos the start positions with the weighted sum of
  the four stage velocities."""
  m = model
  act = np.zeros(m.na) if act is None else np.asarray(act, np.float64)
  h = LD(m.opt.timestep)
  q0, v0, a0 = np.asarray(qpos, np.float64), np.asarray(qvel, LD), np.asarray(act, LD)
  A, B = (0.5, 0.5, 1.0), (1 / LD(6), 1 / LD(3), 1 / LD(3), 1 / LD(6))
  q, v, a = q0, v0, a0
  Fv, Fa, Fd = [], [], []
  for i in range(4):
    F = forward(m, np.asarray(q, np.float64), np.asarray(v, np.float64), ctrl, np.asarray(a, np.float64), disable=disable,
                overrides=overrides)
    Fv.append(v); Fa.append(F['qacc']); Fd.append(F['act_dot'])
    if i < 3:
      s = LD(A[i])
      q = integrate_pos(m, q0, s * v, h)
      v = v0 + h * s * F['qacc']
      a = _advance_act(m, a0, s * F['act_dot'], h)
  dv = sum(B[i] * Fv[i] for i in range(4))
  return dict(qpos=integrate_pos(m, q0, dv, h), qvel=v0 + h * sum(B[i] * Fa[i] for i in range(4)),
              act=_advance_act(m, a0, sum(B[i] * Fd[i] for i in range(4)), h))
