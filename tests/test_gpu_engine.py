"""-m gpu: engine semantics the reference's own engine tests pin, exercised on the CUDA path."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
from conftest import DEV, EMULATE                   # noqa: E402  ('cuda'; 'cpu' only under B200MJ_EMULATE_GPU=1)
from dm_control_b200 import testing_models as tm   # noqa: E402
from dm_control_b200 import mjcf_compile as mc    # noqa: E402
import os, sys   # noqa: E402
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dof_models   # noqa: E402


def _phys(name, B, **kw):
  from dm_control_b200.physics import BatchedPhysics
  return BatchedPhysics(tm.load(name), batch=B, **kw)


def _seed(phys, name, seed=0):
  q0, v0 = tm.initial_states(phys.model, name, phys.batch, seed)
  phys.data.qpos.copy_(torch.as_tensor(q0)); phys.data.qvel.copy_(torch.as_tensor(v0))
  phys.forward()


def test_readme_known_answer_on_gpu():
  # dm_control/mujoco/README.md:25-50
  phys = _phys('slide_box', 3)
  with phys.reset_context():
    phys.data.qpos[:, 0] = 0.5
  np.testing.assert_allclose(phys.data.geom_xpos[0, 1].cpu().numpy(), [0, 0, 0.8], atol=1e-12)
  while float(phys.time()[0]) < 1.0:
    phys.step()
  z = phys.data.geom_xpos[:, 1:3, 2].cpu().numpy()
  assert np.all(np.abs(z - np.array([0.19996362, 0.39996362])) < 5e-9)


def test_contact_force_equals_weight_on_gpu():
  # dm_control/mujoco/wrapper/core_test.py:393-416: sum of contact normal forces == weight (7 places)
  phys = _phys('free_box', 2)
  phys.step(500)
  d = phys.data
  assert d.ncon.tolist() == [4, 4]
  # mj_contactForce through the C ABI (b200mj_contact_force), as the reference test calls it per contact
  forces = torch.stack([phys.contact_force(i) for i in range(4)])          # [4, B, 6]
  total = forces[:, :, 0].sum(0)
  assert float((total - 9.81 * phys.model.body_mass[1]).abs().max()) < 5e-8
  assert float(forces[:, :, 3:].abs().max()) == 0.0                          # condim 3: no contact torque (core_test.py:426-462)
  assert float(phys.contact_force(7).abs().max()) == 0.0                    # beyond ncon: zeros
  for i in range(4):      # and it is the pyramid decoding of efc_force
    a = int(d.contact_efc_address[0, i])
    assert abs(float(d.efc_force[0, a:a + 4].sum()) - float(forces[i, 0, 0])) < 1e-12


@pytest.mark.parametrize('name,nstep', [('cheetah', 4), ('cartpole', 4), ('humanoid', 4), ('cheetah', 70)],
                         ids=['cheetah', 'cartpole', 'humanoid', 'cheetah-70'])
def test_nstep_equals_repeated_step_bitwise(name, nstep):
  # dm_control/mujoco/engine_test.py:627-663 (Euler for cheetah/humanoid, RK4 for cartpole); 70: a call of more than 64 physics steps
  a, b = _phys(name, 8), _phys(name, 8)
  a.legacy_step = b.legacy_step = True
  for p in (a, b):
    _seed(p, name, 4)
    p.set_control(torch.full((p.model.nu,), 0.25, dtype=torch.float64))
  a.step(nstep)
  for _ in range(nstep):
    b.step()
  assert torch.equal(a.get_state(), b.get_state())
  assert torch.equal(a.data.qacc_warmstart, b.data.qacc_warmstart)


def test_run_to_run_determinism_and_batch_invariance():
  # suite/suite_test.py:169-185 (same seed + actions => identical trajectories), extended across batch sizes:
  # env i of a B=4096 launch must equal env i of a B=64 launch bit for bit
  big, small, again = _phys('humanoid', 4096), _phys('humanoid', 64), _phys('humanoid', 4096)
  for p in (big, small, again):
    _seed(p, 'humanoid', 9)
  tape = torch.as_tensor(np.random.RandomState(3).uniform(-1, 1, (10, 4096, 21)), device=DEV)
  for t in range(10):
    big.set_control(tape[t]); again.set_control(tape[t]); small.set_control(tape[t, :64])
    big.step(5); again.step(5); small.step(5)
  assert torch.equal(big.get_state(), again.get_state())
  assert torch.equal(big.get_state()[:64], small.get_state())
  assert torch.equal(big.data.xpos[:64], small.data.xpos)
  assert bool(torch.isfinite(big.get_state()).all())


def test_actuation_disabled_in_after_reset():
  # dm_control/mujoco/engine_test.py:599-604
  phys = _phys('cartpole', 2)
  phys.data.ctrl[:, 0] = 1.0
  phys.after_reset()
  assert float(phys.data.actuator_force.abs().max()) == 0.0
  phys.forward()
  assert phys.data.actuator_force[:, 0].tolist() == [1.0, 1.0]


def test_bad_control_and_bad_state_raise_physics_error():
  # dm_control/mujoco/engine_test.py:487-547
  from dm_control_b200.physics import PhysicsError
  phys = _phys('cartpole', 4)
  phys.data.ctrl[2, 0] = float('nan')
  with pytest.raises(PhysicsError, match='mjWARN_BADCTRL'):
    phys.step()
  phys.data.ctrl.zero_()
  phys.step()                      # recovers
  phys.data.qpos[1, 0] = float('inf')
  with pytest.raises(PhysicsError, match='mjWARN_BADQPOS'):
    phys.step()
  assert bool(torch.isfinite(phys.data.qpos).all())   # offending env was reset in place
  phys.data.qpos[0, 0] = 1e15
  with phys.suppress_physics_errors():
    phys.step()                    # suppressed: logged only


@pytest.mark.skipif(EMULATE, reason='BASELINE-size batch: device only')
def test_sampled_environments_of_the_8192_batch_match_live_oracles(oracle_mod):
  """BASELINE.json batch size against the oracle: 64 environments sampled across the 8 192 (both environment groups,
  every row bucket) are re-run on the CPU oracle from the same start state and action tape; states, contact counts
  and the ordered contact-pair lists must agree after 6 control steps of 5 physics steps."""
  from oracle import oracle as om
  B, nstep = 8192, 6
  phys = _phys('humanoid', B)
  _seed(phys, 'humanoid', 13)
  q0, v0 = phys.data.qpos.cpu().numpy().copy(), phys.data.qvel.cpu().numpy().copy()
  tape = np.random.RandomState(17).uniform(-1, 1, (nstep, B, 21))
  for t in range(nstep):
    phys.set_control(torch.as_tensor(tape[t], device=DEV)); phys.step(5)
  q, v = phys.data.qpos.cpu().numpy(), phys.data.qvel.cpu().numpy()
  ncon = phys.data.ncon.cpu().numpy(); cg = phys.data.contact_geom.cpu().numpy().reshape(B, -1, 2)
  picks = np.unique(np.concatenate([np.random.RandomState(5).choice(B, 60, replace=False), [0, 4095, 4096, 8191]]))
  in_contact = 0
  for e in picks:
    o = om.OraclePhysics(phys.model)
    o.qpos[:] = q0[e]; o.qvel[:] = v0[e]; o.forward()
    for t in range(nstep):
      o.ctrl[:] = tape[t, e]; o.control_step(5)
    assert np.abs(q[e] - o.qpos).max() < 1e-7 and np.abs(v[e] - o.qvel).max() < 1e-6, int(e)
    assert int(ncon[e]) == o.ncon, int(e)
    assert [(int(a), int(b)) for a, b in cg[e, :ncon[e]]] == [(c.geom1, c.geom2) for c in o.contact], int(e)
    in_contact += o.ncon > 0
  assert in_contact >= 5     # the sample must exercise the contact path


@pytest.mark.skipif(EMULATE, reason='BASELINE-size batch: device only')
def test_full_batch_properties_humanoid_8192():
  """BASELINE.json size: properties that need no oracle (finite, bounded, contacts present, clock exact)."""
  phys = _phys('humanoid', 8192, outputs=('xpos', 'subtree_com', 'sensordata', 'ncon'))
  _seed(phys, 'humanoid', 1)
  g = torch.Generator(device=DEV).manual_seed(0)
  for _ in range(40):
    phys.data.ctrl.uniform_(-1, 1, generator=g)
    phys.step(5)
  d = phys.data
  assert bool(torch.isfinite(d.qpos).all()) and bool(torch.isfinite(d.qvel).all())
  np.testing.assert_allclose(d.time.cpu().numpy(), 40 * 5 * 0.005, rtol=0, atol=1e-9)
  quat = d.qpos[:, 3:7]
  assert float((quat.norm(dim=1) - 1).abs().max()) < 1e-9         # free-joint quaternion stays unit
  assert float(d.qpos[:, 2].min()) > -0.05                        # nobody tunnels through the floor
  assert float(d.ncon.float().mean()) > 0.5                       # they are lying on it
  assert int(d.warning.sum()) == 0


def test_compile_and_step_inline_model():
  phys = mc and __import__('dm_control_b200.physics', fromlist=['BatchedPhysics']).BatchedPhysics.from_xml_string(
      tm.XML['pendulum_free'], batch=5)
  phys.step(10)
  assert bool(torch.isfinite(phys.data.qpos).all())


def test_step_host_equals_step():
  """The HOST-buffer entry point (b200mj_step_host) gives the same state as set_control + step on device tensors."""
  a, b = _phys('cheetah', 16), _phys('cheetah', 16)
  for p in (a, b):
    _seed(p, 'cheetah', 2)
  ctrl = torch.rand(16, 6, dtype=torch.float64).mul_(2).sub_(1).pin_memory()
  obs_host = torch.empty(16, 3, dtype=torch.float64).pin_memory()
  for _ in range(5):
    a.set_control(ctrl.to(DEV)); a.step(3)
    b.step_host(ctrl, b.data.sensordata, obs_host, nstep=3)
  assert torch.equal(a.get_state(), b.get_state())
  assert torch.equal(obs_host, a.data.sensordata.cpu())


@pytest.mark.skipif(EMULATE, reason='spawns fresh interpreters on the device; tests/test_emu_kernel_parity.py has the emulated twin')
def test_fused_and_split_paths_agree_bitwise(monkeypatch):
  """B200MJ_SPLIT=0 (one fused kernel) and the default split path are the same arithmetic."""
  import subprocess, sys, os, json
  code = ("import sys, json, torch; sys.path.insert(0, %r);"
          "from dm_control_b200 import testing_models as tm; from dm_control_b200.physics import BatchedPhysics;"
          "m = tm.load('humanoid'); q, v = tm.initial_states(m, 'humanoid', 32, 5); p = BatchedPhysics(m, batch=32);"
          "p.data.qpos.copy_(torch.as_tensor(q)); p.data.qvel.copy_(torch.as_tensor(v)); p.forward();"
          "g = torch.Generator(device='cuda').manual_seed(0);"
          "[ (p.data.ctrl.uniform_(-1, 1, generator=g), p.step(5)) for _ in range(6) ];"
          "print(json.dumps(dict(q=p.data.qpos.cpu().tolist(), s=p.data.sensordata.cpu().tolist(), n=p.data.ncon.cpu().tolist())))"
          ) % os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  outs = []
  # B200MJ_TN=0: runtime-size acceleration kernels (they share their arithmetic with the fused kernel); the last run is the
  # default path, acceleration kernels with nv fixed at compile time (other summation order: equal to rounding noise only)
  for split, tn in (('0', '0'), ('1', '0'), ('1', '1')):
    env = dict(os.environ, B200MJ_SPLIT=split, B200MJ_TN=tn)
    r = subprocess.run([sys.executable, '-c', code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    outs.append(json.loads(r.stdout.strip().splitlines()[-1]))
  assert outs[0] == outs[1]
  import numpy as np
  assert outs[2]['n'] == outs[1]['n']
  for f in ('q', 's'):
    a, b = np.asarray(outs[2][f]), np.asarray(outs[1][f])
    assert np.abs(a - b).max() <= 1e-8 * (1 + np.abs(b).max()), (f, np.abs(a - b).max())


@pytest.mark.parametrize('nv', [6, 9, 12, 18, 22, 27])
def test_compile_time_size_kernels_match_runtime_size_path(nv, monkeypatch):
  """For every nv with a compile-time-size acceleration kernel (B200MJ_NV_LIST), a contact rollout of a generated model
  agrees to 1e-8 with the runtime-size kernels that B200MJ_TN=0 selects at model creation."""
  from dm_control_b200.physics import BatchedPhysics
  import numpy as np
  B = 13
  model, q0, v0 = dof_models.load(dof_models.name(nv), B, 0)
  tape = np.random.RandomState(1).uniform(-1, 1, (12, B, model.nu))

  def run():
    p = BatchedPhysics(model, batch=B)
    p.data.qpos.copy_(torch.as_tensor(q0)); p.data.qvel.copy_(torch.as_tensor(v0)); p.forward()
    ncon = 0
    for t in range(len(tape)):
      p.set_control(torch.as_tensor(tape[t])); p.step(2)
      ncon += int(p.data.ncon.sum())
    assert int(p.data.warning.sum()) == 0
    return p.data.qpos.cpu().numpy(), p.data.qvel.cpu().numpy(), ncon

  qa, va, na = run()
  monkeypatch.setenv('B200MJ_TN', '0')
  qb, vb, nb = run()
  assert na == nb and na > 0
  for a, b in ((qa, qb), (va, vb)):
    assert np.abs(a - b).max() <= 1e-8 * max(1.0, np.abs(b).max()), (nv, np.abs(a - b).max())


SLIDING_CUBE = """
<mujoco><option gravity="0 0 -9.81"/><worldbody>
  <geom name="floor" type="plane" pos="0 0 0" size="10 10 0.1"/>
  <body name="cube" pos="0 0 0.1"><geom type="box" size="0.1 0.1 0.1" mass="1"/>
    <site name="cube_site" type="box" size="0.1 0.1 0.1"/><joint type="slide"/></body>
</worldbody><sensor><touch name="touch_sensor" site="cube_site"/></sensor></mujoco>"""


def test_disable_flags_on_gpu():
  # dm_control/mujoco/wrapper/core_test.py:291-330 through model.disable(...) on the CUDA path
  from dm_control_b200.physics import BatchedPhysics
  phys = BatchedPhysics.from_xml_string(SLIDING_CUBE, batch=2)
  phys.step(100)
  assert float(phys.data.qvel.abs().max()) < 5e-5
  assert float((phys.data.sensordata[:, 0] - 9.81).abs().max()) < 5e-3
  with phys.model.disable('contact', 'gravity'):
    phys.step()
  assert float(phys.data.qvel.abs().max()) < 5e-5
  assert float(phys.data.sensordata.abs().max()) == 0.0
  with phys.model.disable(1 << 4):
    phys.step(10)
  assert float(phys.data.qvel.max()) < -0.1


def test_copy_then_lockstep():
  # dm_control/mujoco/engine_test.py:549-572: a copy stepped in lock-step stays bit-equal
  a = _phys('cheetah', 8)
  _seed(a, 'cheetah', 6)
  a.set_control(torch.full((6,), 0.3, dtype=torch.float64)); a.step(10)
  b = a.copy()
  for p in (a, b):
    p.set_control(torch.full((6,), -0.2, dtype=torch.float64))
  a.step(10); b.step(10)
  assert torch.equal(a.get_state(), b.get_state())
  a.free(); a.free()       # idempotent (engine_test.py:203-205)


def test_masked_reset_leaves_the_other_environments_alone():
  """b200mj_reset with an env_mask (engine.py:306-327 for some environments): masked ones go back to qpos0 with fresh
  outputs, the others keep state AND outputs (sensordata, actuator_force, xpos) bit for bit."""
  phys = _phys('cheetah', 6)
  _seed(phys, 'cheetah', 3)
  phys.set_control(torch.full((6,), 0.4, dtype=torch.float64)); phys.step(7)
  before = {k: getattr(phys.data, k).clone() for k in ('qpos', 'qvel', 'time', 'sensordata', 'actuator_force', 'xpos', 'qacc', 'ctrl')}
  mask = torch.tensor([True, False, False, True, False, False], device=DEV)
  phys.reset(env_mask=mask)
  keep = ~mask
  for k, v in before.items():
    assert torch.equal(getattr(phys.data, k)[keep], v[keep]), k
  q0 = torch.as_tensor(np.asarray(phys.model.qpos0), device=DEV)
  assert torch.equal(phys.data.qpos[mask], q0.expand(2, -1)) and float(phys.data.qvel[mask].abs().max()) == 0.0
  assert float(phys.data.time[mask].abs().max()) == 0.0 and float(phys.data.ctrl[mask].abs().max()) == 0.0
  assert float(phys.data.actuator_force[mask].abs().max()) == 0.0          # forward ran with actuation disabled
  fresh = _phys('cheetah', 2)
  assert torch.equal(phys.data.xpos[mask], fresh.data.xpos)
  # keyframes through the same entry point
  with pytest.raises(ValueError):
    phys.reset(keyframe_id=5)


def test_subtree_vel_entry_point_matches_forward():
  """b200mj_subtree_vel (mj_subtreeVel after a hand-written state, legacy_base.py:179-186) against mj_forward's output."""
  a, b = _phys('humanoid', 4), _phys('humanoid', 4)
  for p in (a, b):
    _seed(p, 'humanoid', 8)
  q0, v0 = tm.initial_states(a.model, 'humanoid', 4, 9)
  for p in (a, b):
    p.data.qpos.copy_(torch.as_tensor(q0)); p.data.qvel.copy_(torch.as_tensor(v0))
  a.forward(); b.subtree_vel()
  assert torch.equal(a.data.subtree_linvel, b.data.subtree_linvel) and torch.equal(a.data.xpos, b.data.xpos)
  assert torch.equal(a.data.qvel, b.data.qvel)


VAR_GEOM = """
<mujoco><worldbody>
  <geom name="floor" type="plane" size="5 5 .1"/>
  <geom name="step" type="box" pos="0 0 .1" size=".3 .3 .1"/>
  <body name="ball" pos="0 0 .6"><freejoint/><geom name="ball" type="sphere" size=".1"/></body>
</worldbody></mujoco>"""


def test_per_environment_geoms(oracle_mod):
  """set_variable_geoms: every environment has its own platform box (height / half-size); each must behave like a model
  COMPILED with that box (what the reference does per episode, composer/environment.py:378-383) — checked against the
  oracle on per-environment models."""
  from dm_control_b200 import mjcf_compile
  from dm_control_b200.physics import BatchedPhysics
  from oracle import oracle as om
  model = mjcf_compile.compile_xml(VAR_GEOM)
  B = 3
  phys = BatchedPhysics(model, batch=B)
  gid = model.name2id('step', 'geom')
  phys.set_variable_geoms([gid])
  pos = torch.tensor([[0, 0, .1], [0, 0, .25], [.05, 0, .05]], dtype=torch.float64)
  size = torch.tensor([[.3, .3, .1], [.3, .3, .25], [.2, .2, .05]], dtype=torch.float64)
  phys.data.var_geom_pos[:, 0] = pos.to(DEV); phys.data.var_geom_size[:, 0] = size.to(DEV)
  phys.forward()
  phys.step(400)
  z = phys.data.qpos[:, 2].cpu().numpy()
  for e in range(B):
    m = model.copy()
    m.fields['geom_pos'].reshape(-1, 3)[gid] = pos[e].numpy(); m.fields['geom_size'].reshape(-1, 3)[gid] = size[e].numpy()
    m.fields['geom_rbound'].reshape(-1)[gid] = float(np.linalg.norm(size[e].numpy())); m.touch()
    o = om.OraclePhysics(m); o.forward()
    for _ in range(400):
      o.control_step(1)
    assert abs(z[e] - o.qpos[2]) < 1e-9, (e, z[e], o.qpos[2])
  assert z[1] - z[0] > 0.29 and z[0] - z[2] > 0.09          # resting on platforms of different heights


@pytest.mark.parametrize('feature,xml', [
    ('condim 4 (torsional friction)', '<mujoco><worldbody><geom type="plane" size="1 1 .1"/><body pos="0 0 .2"><freejoint/><geom size=".1" condim="4"/></body></worldbody></mujoco>'),
    ('condim 6 (rolling friction)', '<mujoco><worldbody><geom type="plane" size="1 1 .1"/><body pos="0 0 .2"><freejoint/><geom size=".1" condim="6"/></body></worldbody></mujoco>'),
    ('CG solver', '<mujoco><option solver="CG"/><worldbody><geom type="plane" size="1 1 .1"/><body pos="0 0 .2"><freejoint/><geom size=".1"/></body></worldbody></mujoco>'),
    ('elliptic cones', '<mujoco><option cone="elliptic"/><worldbody><geom type="plane" size="1 1 .1"/><body pos="0 0 .2"><freejoint/><geom size=".1"/></body></worldbody></mujoco>'),
    ('nv = 65, one more than the largest supported', dof_models.xml(65)),
])
def test_unsupported_features_are_refused_not_approximated(feature, xml):
  """wrapper/core_test.py:426-462 pins contact torques for condim 4 / 6: this engine has condim 1 / 3 only, and a model
  that asks for more must be refused at model creation (error -3), never run with silently different physics."""
  from dm_control_b200 import lib, mjcf_compile
  from dm_control_b200.physics import BatchedPhysics
  try:
    model = mjcf_compile.compile_xml(xml)
  except (NotImplementedError, ValueError):
    return                                  # refused by the compiler already
  with pytest.raises(lib.EngineError, match='-3'):
    BatchedPhysics(model, batch=2)
