"""Per-environment model fields (BatchedPhysics.set_env_model_fields, b200mj_model_set_env_fields) and the batched
PhysicsVariator. The contract every engine test here checks: environment e of a batch with per-environment values v_e
equals, bit for bit, environment 0 of a BatchedPhysics built on a copy of the model with v_e written through
`model.set` — nothing derived is recomputed, and the implicit-damping choice of mj_Euler is made per environment."""
import os
import pickle
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import DEV, EMULATE                   # noqa: E402  ('cuda'; 'cpu' only under B200MJ_EMULATE_GPU=1)
from dm_control_b200 import lib                     # noqa: E402
from dm_control_b200 import mjcf_compile            # noqa: E402
from dm_control_b200 import testing_models as tm    # noqa: E402
from dm_control_b200.physics import ENV_MODEL_FIELDS, BatchedPhysics   # noqa: E402
from dm_control_b200.variation import PhysicsVariator                 # noqa: E402

STEPS = 3 if EMULATE else 20          # control steps (of NSUB physics steps) in the bitwise comparisons
NSUB = 2
OUTS = ('qpos', 'qvel', 'act', 'qacc', 'sensordata', 'ncon', 'nefc', 'efc_force', 'contact_geom', 'contact_pos',
        'contact_dist', 'contact_frame', 'warning', 'qfrc_passive', 'qfrc_actuator', 'subtree_linvel', 'xipos')


def _outputs(phys, envs=None):
  out = {n: getattr(phys.data, n).clone() for n in OUTS}
  return out if envs is None else {n: t[envs] for n, t in out.items()}


def _assert_equal(a, b, what):
  for n in OUTS:
    assert torch.equal(a[n], b[n]), (what, n, (a[n].double() - b[n].double()).abs().max().item())


def _start(model, name, B, seed=0):
  base = name.split(':')[0]
  q, v = tm.initial_states(model, base if base in ('humanoid', 'quadruped', 'cheetah', 'cartpole', 'cmu_humanoid') else base, B, seed)
  return torch.as_tensor(q), torch.as_tensor(v)


def _make(model, B, q, v, variant=None, var_geoms=None):
  phys = BatchedPhysics(model, batch=B)
  if variant == 'applied':
    phys.enable_applied_forces(True)
    g = torch.Generator().manual_seed(3)
    phys.data.qfrc_applied.copy_((torch.rand(B, model.nv, generator=g, dtype=torch.float64) - 0.5).to(DEV))
  if variant == 'nonlegacy':
    phys.legacy_step = False
  if var_geoms is not None:
    phys.set_variable_geoms(var_geoms)
  phys.data.qpos.copy_(q.to(DEV)); phys.data.qvel.copy_(v.to(DEV)); phys.forward()
  return phys


def _run(phys, steps, seed=1):
  g = torch.Generator().manual_seed(seed)
  for _ in range(steps):
    phys.set_control((torch.rand(phys.batch, phys.model.nu, generator=g, dtype=torch.float64) * 2 - 1).to(DEV))
    phys.step(NSUB)


def _load(name):
  if name.endswith(':pgs'):
    return mjcf_compile.compile_xml(tm.XML['pendulum_free'].replace('<option ', '<option solver="PGS" iterations="100" '),
                                    nconmax=16, njmax=64)
  return tm.load(name.split(':')[0])


def _walls(model):
  return [g for g in range(model.ngeom) if int(model.geom_bodyid[g]) == 0 and int(model.geom_type[g]) == 6]


INERT = ['humanoid', 'quadruped', 'cheetah', 'cartpole', 'convex_zoo', 'cmu_humanoid', 'pendulum_free:pgs',
         'pendulum_free:applied', 'pendulum_free:nonlegacy']


@pytest.mark.parametrize('name', INERT)
def test_per_environment_fields_holding_the_models_values_are_inert(name):
  model = _load(name)
  variant = name.split(':')[1] if name.count(':') and not name.endswith(':pgs') else None
  B = 4
  q, v = _start(model, name, B)
  walls = _walls(model) if name == 'cmu_humanoid' else None
  ref = _make(model, B, q, v, variant, walls)
  phys = _make(model, B, q, v, variant, walls)
  if walls:
    for p in (ref, phys):     # per-environment walls (the corridor arenas): shifted differently in every environment
      p.data.var_geom_pos[:, :, 0] += torch.arange(B, dtype=torch.float64, device=p.device)[:, None] * 0.1
  phys.set_env_model_fields(ENV_MODEL_FIELDS)
  ref.forward(); phys.forward()
  _assert_equal(_outputs(ref), _outputs(phys), 'forward')
  _run(ref, STEPS); _run(phys, STEPS)
  _assert_equal(_outputs(ref), _outputs(phys), 'step')


def _draw(model, B, seed, lo=0.5, hi=1.5):
  """Independent per-environment values of every supported field: scales in [lo, hi], solref time constants,
  gains; environment 0 gets an all-zero dof_damping row and environment 1 a damped one (both damping crossings)."""
  rs = np.random.RandomState(seed)
  vals = {}
  for f in ENV_MODEL_FIELDS:
    base = np.asarray(model.fields[f], dtype=np.float64)
    vals[f] = base[None] * rs.uniform(lo, hi, (B,) + base.shape)
  vals['geom_solref'][..., 0] = rs.uniform(0.01, 0.04, vals['geom_solref'].shape[:-1])
  vals['geom_solimp'] = np.broadcast_to(np.asarray(model.fields['geom_solimp']), (B,) + model.fields['geom_solimp'].shape).copy()
  vals['geom_solimp'][..., 0] = rs.uniform(0.85, 0.95, vals['geom_solimp'].shape[:-1])
  vals['dof_damping'][0] = 0
  vals['dof_damping'][1] = rs.uniform(0.2, 1.0, model.nv)
  return vals


def _single(model, vals, e, q, v, B=1):
  m = model.copy()
  for f, a in vals.items():
    m.set(f, a[e])
  p = BatchedPhysics(m, batch=B)
  p.data.qpos.copy_(q[e:e + 1].to(DEV).expand(B, -1)); p.data.qvel.copy_(v[e:e + 1].to(DEV).expand(B, -1)); p.forward()
  return p


@pytest.mark.parametrize('hook', [None, 'B200MJ_TN', 'B200MJ_SPLIT'])
@pytest.mark.parametrize('name', ['pendulum_free', 'humanoid', 'quadruped', 'convex_zoo'])
def test_each_environment_equals_a_model_with_its_values(name, hook, monkeypatch):
  if hook:
    monkeypatch.setenv(hook, '0')
  model = tm.load(name)
  B = 6
  q, v = _start(model, name, B)
  vals = _draw(model, B, 11)
  phys = BatchedPhysics(model, batch=B)
  phys.set_env_model_fields(ENV_MODEL_FIELDS)
  for f, a in vals.items():
    getattr(phys.env_model, f).copy_(torch.as_tensor(a).to(DEV))
  phys.data.qpos.copy_(q.to(DEV)); phys.data.qvel.copy_(v.to(DEV)); phys.forward()
  singles = [_single(model, vals, e, q, v) for e in range(B)]
  for e, s in enumerate(singles):
    _assert_equal(_outputs(phys, [e]), _outputs(s), (e, 'forward'))
  steps = STEPS if name != 'humanoid' or not EMULATE else 2
  _run(phys, steps, seed=5)
  g = torch.Generator().manual_seed(5)
  ctrls = [(torch.rand(B, model.nu, generator=g, dtype=torch.float64) * 2 - 1) for _ in range(steps)]
  for e, s in enumerate(singles):
    for c in ctrls:
      s.set_control(c[e:e + 1].to(DEV)); s.step(NSUB)
    _assert_equal(_outputs(phys, [e]), _outputs(s), (e, 'step'))
  cf = phys.contact_force(0)
  for e, s in enumerate(singles):
    assert torch.equal(cf[e:e + 1], s.contact_force(0)), (e, 'contact_force')
  phys.subtree_vel()
  for e, s in enumerate(singles):
    s.subtree_vel()
    _assert_equal(_outputs(phys, [e]), _outputs(s), (e, 'subtree_vel'))
  mask = torch.tensor([1, 0, 1, 0, 1, 1], dtype=torch.bool)
  before = _outputs(phys)
  phys.reset(env_mask=mask.to(DEV)); phys.after_reset(env_mask=mask.to(DEV))
  after = _outputs(phys)
  for e, s in enumerate(singles):
    if mask[e]:
      s.reset(); s.after_reset()
      _assert_equal({n: t[[e]] for n, t in after.items()}, _outputs(s), (e, 'reset'))
    else:
      _assert_equal({n: t[[e]] for n, t in after.items()}, {n: t[[e]] for n, t in before.items()}, (e, 'untouched by reset'))


@pytest.mark.parametrize('name', ['humanoid', 'quadruped'])
def test_per_environment_models_match_the_oracle(name, oracle_mod):
  model = tm.load(name)
  B = 2 if EMULATE else 3
  nctl = 4 if EMULATE else 25
  q, v = _start(model, name, B, seed=2)
  # scales in [0.8, 1.2]. With [0.5, 1.5] the quadruped's environment 1 gets contacts with a solref time constant of
  # 0.0108 s at h = 0.005 s (near MuJoCo's 2h floor) and halved masses: there qacc amplifies a 1e-13 difference in qpos
  # to 1e-8 within six physics steps (same ncon, nefc and Newton iterations on both sides), and on the seventh qacc
  # differs by 2e2 (|dqpos| 5e-3) — a jump, as when a constraint row changes state on one side only. Every field varied
  # alone stays within 1e-14.
  # That is the conditioning of the model, not a per-environment effect: the engine equals its model-copy twin bitwise.
  vals = _draw(model, B, 21, 0.8, 1.2)
  phys = BatchedPhysics(model, batch=B)
  phys.set_env_model_fields(ENV_MODEL_FIELDS)
  for f, a in vals.items():
    getattr(phys.env_model, f).copy_(torch.as_tensor(a).to(DEV))
  phys.data.qpos.copy_(q.to(DEV)); phys.data.qvel.copy_(v.to(DEV)); phys.forward()
  ctrl = np.random.RandomState(3).uniform(-1, 1, (B, model.nu))
  phys.set_control(torch.as_tensor(ctrl).to(DEV))
  for _ in range(nctl):
    phys.step(NSUB)
  for e in range(B):
    m = model.copy()
    for f, a in vals.items():
      m.set(f, a[e])
    o = oracle_mod.OraclePhysics(m)
    o.qpos[:] = q[e].numpy(); o.qvel[:] = v[e].numpy(); o.forward(); o.ctrl[:] = ctrl[e]
    for _ in range(nctl):
      o.control_step(NSUB)
    assert np.abs(phys.data.qpos[e].cpu().numpy() - o.qpos).max() < 1e-9, e
    assert np.abs(phys.data.qvel[e].cpu().numpy() - o.qvel).max() < 1e-9, e


TILT = """
<mujoco><option timestep="0.002"/>
<default><geom solimp="0.99 0.99 0.001" solref="0.004 1"/></default>
<worldbody>
  <geom name="slope" type="plane" size="5 5 .1" euler="0 {deg} 0" friction="0.1"/>
  <body name="box" pos="{x} 0 {z}" euler="0 {deg} 0"><freejoint/><geom name="box" type="box" size=".1 .1 .1" friction="0.1"/></body>
</worldbody></mujoco>"""


def test_box_on_a_slope_slides_exactly_where_friction_is_below_the_tangent():
  """tan(theta) = 0.5: per-environment friction 0.3 and 0.45 slide down, 0.55 and 0.8 hold (mixing takes the larger
  of the two geoms' coefficients, so both geoms get the environment's value). MuJoCo's soft contacts regularise
  friction, so a held box creeps: with stiff contacts (solimp 0.99) by well under a millimetre in half a second,
  against more than 10 cm for the sliding ones — and less the further friction is above the tangent."""
  th = np.arctan(0.5)
  n = np.array([np.sin(th), 0, np.cos(th)])      # slope normal (the plane's z axis after the rotation about y)
  c = 0.1 * n
  model = mjcf_compile.compile_xml(TILT.format(deg=np.degrees(th), x=c[0], z=c[2]))
  mus = [0.3, 0.45, 0.55, 0.8]
  B = len(mus)
  phys = BatchedPhysics(model, batch=B)
  phys.set_env_model_fields(['geom_friction'])
  phys.env_model.geom_friction[:, :, 0] = torch.tensor(mus, dtype=torch.float64, device=phys.device)[:, None]
  phys.mark_as_dirty()
  phys.step(250)                  # settle onto the slope
  p0 = phys.data.qpos[:, :3].clone()
  phys.step(250)
  d = (phys.data.qpos[:, :3] - p0).cpu().numpy()
  down = d @ np.array([np.cos(th), 0, -np.sin(th)])         # displacement down the slope
  for k, mu in enumerate(mus):
    if mu < 0.5:
      assert down[k] > 0.1, (mu, down[k])
    else:
      assert np.abs(d[k]).max() < 1e-3, (mu, d[k])
  assert np.abs(d[3]).max() < np.abs(d[2]).max()


PEND = """
<mujoco><option timestep="0.0005" gravity="0 0 -9.81"/>
<worldbody><body name="bob" pos="0 0 1"><joint name="hinge" type="hinge" axis="0 1 0"/>
  <inertial pos="0 0 -.5" mass="1" diaginertia=".01 .01 .01"/></body></worldbody></mujoco>"""


def test_pendulum_period_follows_per_environment_mass_and_armature():
  model = mjcf_compile.compile_xml(PEND)
  mass = [0.5, 1.0, 2.0, 1.0]
  arm = [0.0, 0.0, 0.1, 0.5]
  B = len(mass)
  phys = BatchedPhysics(model, batch=B)
  phys.set_env_model_fields(['body_mass', 'dof_armature'])
  phys.bind('body', 'bob').mass = torch.tensor(mass, dtype=torch.float64)[:, None]
  phys.named.model.dof_armature['hinge'] = torch.tensor(arm, dtype=torch.float64, device=phys.device)[:, None]
  phys.data.qpos[:] = 0.01
  phys.forward()
  h, l, g = model.opt.timestep, 0.5, 9.81
  T = [2 * np.pi * np.sqrt((0.01 + m * l * l + a) / (m * g * l)) for m, a in zip(mass, arm)]
  n = int(1.6 * max(T) / h)
  qs = []
  for _ in range(n // 50):
    phys.step(50)
    qs.append(phys.data.qpos[:, 0].cpu().numpy().copy())
  qs = np.array(qs)
  t = (np.arange(len(qs)) + 1) * 50 * h
  for e in range(B):
    x = qs[:, e]
    cross = [t[i] - x[i] * (t[i + 1] - t[i]) / (x[i + 1] - x[i]) for i in range(len(x) - 1) if x[i] > 0 >= x[i + 1]]
    assert len(cross) >= 1
    # first downward zero crossing from the release at rest at +amplitude: a quarter period
    assert abs(cross[0] * 4 - T[e]) / T[e] < 1e-3, (e, cross[0] * 4, T[e])


def test_bind_and_named_model_address_only_their_rows():
  model = tm.load('pendulum_free')
  B = 3
  phys = BatchedPhysics(model, batch=B)
  phys.set_env_model_fields(['geom_friction', 'body_mass', 'jnt_stiffness'])
  fr = phys.bind('geom', ['a', 's']).friction
  assert tuple(fr.shape) == (B, 2, 3)
  assert tuple(phys.bind('geom', 'a').friction.shape) == (B, 3)
  assert tuple(phys.bind('body', ['a', 'b']).mass.shape) == (B, 2)
  assert tuple(phys.bind('body', 'a').mass.shape) == (B,)
  base = phys.env_model.geom_friction.clone()
  phys._pos_current = True
  phys.bind('geom', ['a', 's']).friction = torch.tensor([.9, .01, .001], dtype=torch.float64)      # [w]: every environment
  assert not phys._pos_current and phys.is_dirty
  ga, gs = model.name2id('a', 'geom'), model.name2id('s', 'geom')
  want = base.clone(); want[:, [ga, gs]] = torch.tensor([.9, .01, .001], dtype=torch.float64, device=phys.device)
  assert torch.equal(phys.env_model.geom_friction, want)
  per_env = torch.arange(B * 2 * 3, dtype=torch.float64).reshape(B, 2, 3)
  phys.bind('geom', ['a', 's']).friction = per_env                                                  # [B, k, w]
  assert torch.equal(phys.env_model.geom_friction[:, [ga, gs]].cpu(), per_env)
  phys.bind('body', 'b').mass = 2.5                                                                  # scalar
  bb = model.name2id('b', 'body')
  assert torch.all(phys.env_model.body_mass[:, bb] == 2.5)
  others = [i for i in range(model.nbody) if i != bb]
  assert torch.equal(phys.env_model.body_mass[:, others].cpu(), torch.as_tensor(model.body_mass[others])[None].expand(B, -1))
  st = phys.named.model.jnt_stiffness['h2'].clone()                                               # [B, 1]
  st[1] = 7.0
  phys.named.model.jnt_stiffness['h2'] = st
  j = model.name2id('h2', 'joint')
  assert phys.env_model.jnt_stiffness[:, j].tolist() == [float(model.jnt_stiffness[j]), 7.0, float(model.jnt_stiffness[j])]
  assert tuple(phys.named.model.geom_friction['a'].shape) == (B, 3)
  assert float(model.jnt_stiffness[j]) != 7.0          # the shared model is untouched


def test_fields_survive_a_model_reupload_pickling_and_copy():
  model = tm.load('pendulum_free').copy()
  B = 3
  q, v = _start(model, 'pendulum_free', B)
  vals = _draw(model, B, 5)
  phys = BatchedPhysics(model, batch=B)
  phys.set_env_model_fields(ENV_MODEL_FIELDS)
  for f, a in vals.items():
    getattr(phys.env_model, f).copy_(torch.as_tensor(a).to(DEV))
  phys.data.qpos.copy_(q.to(DEV)); phys.data.qvel.copy_(v.to(DEV)); phys.forward()
  _run(phys, 2)
  model.set('geom_margin', 0.0)       # a shared-model write: the next call re-uploads the model
  twin = phys.copy()
  pick = pickle.loads(pickle.dumps(phys))
  assert twin.env_model_fields == ENV_MODEL_FIELDS and pick.env_model_fields == ENV_MODEL_FIELDS
  for other in (twin, pick):
    assert torch.equal(other.env_model.dof_damping, phys.env_model.dof_damping)
  for p in (phys, twin, pick):
    p.forward()
    _run(p, 2, seed=8)
  _assert_equal(_outputs(phys), _outputs(twin), 'copy')
  _assert_equal(_outputs(phys), _outputs(pick), 'pickle')
  s0 = _single(model, vals, 0, phys.data.qpos.cpu(), phys.data.qvel.cpu())
  s0.data.ctrl.copy_(phys.data.ctrl[:1]); s0.forward()
  phys.forward()
  for n in ('qacc', 'qfrc_passive', 'qfrc_actuator', 'sensordata', 'ncon', 'nefc', 'xipos', 'subtree_linvel'):
    assert torch.equal(getattr(phys.data, n)[:1], getattr(s0.data, n)), n      # (contact slots past ncon hold history)
  phys.set_env_model_fields(())
  assert phys.env_model is None and phys.env_model_fields == ()
  phys.forward()


@pytest.mark.parametrize('field', ['actuator_gear', 'geom_size', 'geom_condim', 'body_mas'])
def test_unsupported_fields_are_refused_by_name(field):
  phys = BatchedPhysics(tm.load('pendulum_free'), batch=2)
  with pytest.raises(ValueError, match=field):
    phys.set_env_model_fields(['body_mass', field])
  with pytest.raises(ValueError, match='body_mass'):
    phys.set_env_model_fields(['body_mass', 'body_mass'])
  kind, attr = field.split('_', 1)
  with pytest.raises(ValueError, match=field):
    PhysicsVariator().bind_attributes({'actuator': 'actuator', 'geom': 'geom', 'body': 'body'}[kind], 'a', **{attr: 1.0})


def test_the_abi_refuses_bad_field_lists_and_batches_beyond_the_rows():
  import ctypes
  from dm_control_b200 import model as _model
  fid = {n: k for k, (n, _) in enumerate(_model.FIELDS)}
  phys = BatchedPhysics(tm.load('pendulum_free'), batch=2)
  L, h = phys._L, phys._handle
  rows = torch.zeros(4, 64, dtype=torch.float64, device=phys.device)
  ptr = ctypes.c_void_p(rows.data_ptr())

  def ids(*names):
    a = (ctypes.c_int32 * len(names))(*[fid[n] for n in names])
    return ctypes.cast(a, ctypes.POINTER(ctypes.c_int32))
  assert L.b200mj_model_set_env_fields(h, ids('actuator_gear'), 1, ptr, 2) == -6
  assert L.b200mj_model_set_env_fields(h, ids('geom_condim'), 1, ptr, 2) == -6
  assert L.b200mj_model_set_env_fields(h, ids('body_mass', 'body_mass'), 2, ptr, 2) == -7
  assert L.b200mj_model_set_env_fields(h, ids('body_mass'), 1, ctypes.c_void_p(None), 2) == -8
  assert L.b200mj_model_set_env_fields(h, ids('body_mass'), 1, ptr, 0) == -9
  for code in (-6, -7, -8, -9, -10):
    assert b'per-environment' in L.b200mj_error_string(code) or b'per environment' in L.b200mj_error_string(code)
  assert L.b200mj_model_set_env_fields(h, ids('body_mass'), 1, ptr, 1) == 0          # rows for one environment
  io, st = ctypes.byref(phys._io), phys._stream()
  assert L.b200mj_step(h, io, 2, 1, phys._flags(), st) == -10
  assert L.b200mj_forward(h, io, 2, 0, 0, st) == -10
  assert L.b200mj_forward_masked(h, io, 2, None, 0, 0, st) == -10
  assert L.b200mj_reset(h, io, 2, None, -1, st) == -10
  assert L.b200mj_subtree_vel(h, io, 2, 0, st) == -10
  assert L.b200mj_contact_force(h, io, 2, 0, ptr, st) == -10
  assert L.b200mj_model_set_env_fields(h, None, 0, None, 0) == 0                     # off again
  assert L.b200mj_forward(h, io, 2, 0, 0, st) == 0


def test_variator_changes_only_the_masked_rows():
  model = tm.load('pendulum_free')
  B = 5
  phys = BatchedPhysics(model, batch=B)
  phys.set_env_model_fields(['jnt_stiffness'])
  phys.env_model.jnt_stiffness[:, 0] = 3.0                 # kept: already per-environment
  var = PhysicsVariator()
  g = torch.Generator(device=phys.device).manual_seed(0)
  scale = lambda init, cur, gen, n: init * (0.5 + torch.rand(init.shape, generator=gen, dtype=init.dtype, device=init.device))
  var.bind_attributes('geom', ['a', 'b'], friction=scale)
  var.bind_attributes('body', 'a', mass=lambda init, cur, gen, n: cur + 1.0)
  var.bind_attributes('actuator', 'm2', gainprm=4.0)
  var.bind_attributes('joint', ['h1', 'sl'], damping=lambda init, cur, gen, n: init + torch.arange(n, dtype=init.dtype, device=init.device)[:, None])
  mask = torch.tensor([1, 0, 1, 0, 0], dtype=torch.bool, device=phys.device)
  var.apply_variations(phys, g, env_mask=mask)
  assert set(phys.env_model_fields) == {'jnt_stiffness', 'geom_friction', 'body_mass', 'actuator_gainprm', 'dof_damping'}
  d1, dsl = model.jnt_dofadr[model.name2id('h1', 'joint')], model.jnt_dofadr[model.name2id('sl', 'joint')]
  dd = phys.env_model.dof_damping.cpu()
  base = torch.as_tensor(np.array(model.dof_damping))
  assert torch.equal(dd[[1, 3, 4]], base[None].expand(3, -1))                     # unmasked rows untouched
  assert dd[0, d1] == base[d1] and dd[2, d1] == base[d1] + 1 and dd[2, dsl] == base[dsl] + 1
  assert tuple(phys.bind('joint', ['h1', 'sl']).damping.shape) == (B, 2)          # one column per dof
  assert tuple(phys.bind('joint', 'a').armature.shape) == (6,)                     # shared here; a free joint: six dofs
  assert torch.all(phys.env_model.jnt_stiffness[:, 0] == 3.0)
  ga, gb, ba = model.name2id('a', 'geom'), model.name2id('b', 'geom'), model.name2id('a', 'body')
  m2 = model.name2id('m2', 'actuator')
  fr0 = torch.as_tensor(np.asarray(model.geom_friction), device=phys.device)
  fr = phys.env_model.geom_friction
  for e in range(B):
    changed = not torch.equal(fr[e], fr0)
    assert changed == bool(mask[e]), e
    assert torch.equal(fr[e, [i for i in range(model.ngeom) if i not in (ga, gb)]], fr0[[i for i in range(model.ngeom) if i not in (ga, gb)]])
    ratio = fr[e, [ga, gb]] / fr0[[ga, gb]]
    assert bool(((ratio >= 0.5) & (ratio <= 1.5)).all())
    assert float(phys.env_model.body_mass[e, ba]) == float(model.body_mass[ba]) + (1.0 if mask[e] else 0.0)
    assert torch.all(phys.env_model.actuator_gainprm[e, m2] == (4.0 if mask[e] else torch.as_tensor(model.actuator_gainprm[m2], device=phys.device)))
  # initial values are remembered: a second application scales the first application's value again, not the current one
  var.apply_variations(phys, g, env_mask=mask)
  ratio = phys.env_model.geom_friction[0, [ga, gb]] / fr0[[ga, gb]]
  assert bool(((ratio >= 0.5) & (ratio <= 1.5)).all())
  assert float(phys.env_model.body_mass[0, ba]) == float(model.body_mass[ba]) + 2.0     # `current` is the row's value
  phys.forward()
  phys.step(2)
  var.clear()
  var.apply_variations(phys, g)                            # nothing bound: nothing changes
  assert float(phys.env_model.body_mass[0, ba]) == float(model.body_mass[ba]) + 2.0


@pytest.mark.skipif(DEV != 'cuda', reason='CUDA graphs: device only')
def test_graph_replays_read_rows_rewritten_in_place():
  from dm_control_b200 import suite
  B, nu = 32, 21
  outs = []
  for graphed, rewrite in ((False, True), (True, True), (False, False)):
    env = suite.load('humanoid', 'run', batch=B, seed=4)
    env.physics.check_errors = False
    env._graph_step = graphed
    env.reset()
    g = torch.Generator(device=DEV).manual_seed(9)
    rows = []
    for t in range(12):
      if t == 3:      # fields enabled after steps were captured: the graphs must be re-captured, not replayed stale
        env.physics.set_env_model_fields(ENV_MODEL_FIELDS)
      if t == 5 and rewrite:
        env.physics.env_model.body_mass.mul_(1.3)
        env.physics.env_model.dof_damping[::2] = 0.7
        env.physics.env_model.geom_friction[1::2, :, 0] = 0.2
        env.physics.mark_as_dirty()
      a = torch.rand(B, nu, generator=g, device=DEV, dtype=torch.float64) * 2 - 1
      ts = env.step(a)
      rows.append(torch.cat([v.reshape(B, -1) for v in ts.observation.values()] + [ts.reward[:, None]], dim=1).clone())
    outs.append(torch.stack(rows))
    if graphed:
      assert any(isinstance(v, tuple) for v in env._step_graphs.values())
  assert torch.equal(outs[0], outs[1])                     # graph == eager, bit for bit
  assert torch.equal(outs[0][:5], outs[2][:5]) and not torch.equal(outs[0][5:], outs[2][5:])   # the rewrite took effect
