"""-m gpu: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs.

Bar (BASELINE.json north_star): qpos/qvel within 1e-5 relative after a fixed horizon, contact-pair indexing
bit-exact. Measured agreement is ~1e-11, so the assertions use 1e-8 to catch regressions early.
The oracle itself is pinned only by the reference's analytic known-answers (tests/test_oracle_kat.py).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')
from dm_control_b200 import testing_models as tm   # noqa: E402

import os, sys   # noqa: E402
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dof_models   # noqa: E402

TOL = 1e-8          # asserted; north_star bar is 1e-5
FIELD_TOL = 1e-10


def relerr(a, b):
  a, b = np.asarray(a), np.asarray(b)
  return float(np.max(np.abs(a - b)) / max(1.0, np.max(np.abs(b)))) if a.size else 0.0


def _setup(name, B, seed, oracle_mod):
  from dm_control_b200.physics import BatchedPhysics
  model, q0, v0 = dof_models.load(name, B, seed)
  phys = BatchedPhysics(model, batch=B)
  phys.data.qpos.copy_(torch.as_tensor(q0))
  phys.data.qvel.copy_(torch.as_tensor(v0))
  phys.forward()
  oracles = []
  for e in range(B):
    o = oracle_mod.OraclePhysics(model)
    o.qpos[:] = q0[e]
    o.qvel[:] = v0[e]
    o.forward()
    oracles.append(o)
  return model, phys, oracles


@pytest.mark.parametrize('name,B', [('cartpole', 8), ('pendulum_free', 8), ('cheetah', 16), ('humanoid', 16),
                                    ('slide_box', 4), ('free_box', 4), ('cmu_humanoid', 4)])
def test_forward_fields_match_oracle(name, B, oracle_mod):
  model, phys, oracles = _setup(name, B, 11, oracle_mod)
  for f in ('xpos', 'xquat', 'xmat', 'xipos', 'geom_xpos', 'geom_xmat', 'site_xpos', 'site_xmat', 'subtree_com',
            'cvel', 'qfrc_bias', 'qfrc_passive', 'qacc', 'qfrc_constraint', 'qfrc_actuator', 'sensordata',
            'subtree_linvel'):
    if f == 'subtree_linvel':
      for o in oracles:
        o.subtree_vel()
    g = getattr(phys.data, f).cpu().numpy().reshape(B, -1)
    o = np.stack([np.asarray(getattr(oo, f)).reshape(-1) for oo in oracles])
    assert relerr(g, o) < FIELD_TOL, (name, f, relerr(g, o))
  gM = phys.data.qM.cpu().numpy()
  oM = np.stack([oo.M_dense() for oo in oracles])
  assert relerr(gM, oM) < 1e-13
  np.testing.assert_array_equal(phys.data.ncon.cpu().numpy(), [o.ncon for o in oracles])
  np.testing.assert_array_equal(phys.data.nefc.cpu().numpy(), [o.nefc for o in oracles])
  for e, o in enumerate(oracles):
    n = o.nefc
    np.testing.assert_allclose(phys.data.efc_force[e, :n].cpu().numpy(), o.efc('efc_force'), rtol=1e-7, atol=1e-7)


@pytest.mark.parametrize('name,B,ncontrol,nsub', [('cartpole', 16, 60, 1), ('pendulum_free', 8, 50, 2),
                                                   ('cheetah', 32, 100, 1), ('humanoid', 32, 20, 5),
                                                   ('quadruped', 16, 15, 4), ('cmu_humanoid', 6, 6, 6)] +
                         # generated models (tests/dof_models.py) at the dof counts no fixture has: the compile-time-size
                         # kernels and the runtime-size boundaries; B = 13 leaves the last 4-warp and 5-warp CTAs partly filled
                         [(dof_models.name(nv), B, 12, 2) for nv in dof_models.NV_TARGETS for B in (8, 13)])
def test_rollout_matches_oracle(name, B, ncontrol, nsub, oracle_mod):
  """Fixed recorded action tape, legacy step ordering; compare every control step."""
  model, phys, oracles = _setup(name, B, 0, oracle_mod)
  tape = np.random.RandomState(1).uniform(-1, 1, (ncontrol, B, model.nu))
  saw_contact = 0
  for t in range(ncontrol):
    phys.set_control(torch.as_tensor(tape[t]))
    phys.step(nsub)
    gq, gv = phys.data.qpos.cpu().numpy(), phys.data.qvel.cpu().numpy()
    gn, gg = phys.data.ncon.cpu().numpy(), phys.data.contact_geom.cpu().numpy()
    for e, o in enumerate(oracles):
      o.ctrl[:] = tape[t, e]
      o.control_step(nsub)
    oq, ov = np.stack([o.qpos for o in oracles]), np.stack([o.qvel for o in oracles])
    assert relerr(gq, oq) < TOL and relerr(gv, ov) < TOL, (name, t, relerr(gq, oq), relerr(gv, ov))
    for e, o in enumerate(oracles):
      cs = o.contact
      assert len(cs) == gn[e], (name, t, e)
      assert [(c.geom1, c.geom2) for c in cs] == [tuple(x) for x in gg[e, :gn[e]]], (name, t, e)
      saw_contact += len(cs)
    np.testing.assert_allclose(phys.data.time.cpu().numpy(), [o.time for o in oracles], rtol=0, atol=1e-12)
  if name != 'cartpole':
    assert saw_contact > 0, 'horizon never touched the contact path'
  assert int(phys.data.warning.sum()) == 0


def test_quadruped_smooth_dynamics_match_oracle(oracle_mod):
  """Tendons, tendon equalities, filter-dynamics actuators (na=12), acc-stage sensors: airborne horizon."""
  from dm_control_b200.physics import BatchedPhysics
  model = tm.load('quadruped')
  B = 8
  q0, v0 = tm.initial_states(model, 'quadruped', B, 2)
  q0[:, 2] = 3.0   # keep it off the floor for the horizon (convex-pair collisions are not in the subset)
  phys = BatchedPhysics(model, batch=B)
  phys.data.qpos.copy_(torch.as_tensor(q0)); phys.data.qvel.copy_(torch.as_tensor(v0)); phys.forward()
  oracles = []
  for e in range(B):
    o = oracle_mod.OraclePhysics(model); o.qpos[:] = q0[e]; o.qvel[:] = v0[e]; o.forward(); oracles.append(o)
  tape = np.random.RandomState(5).uniform(-1, 1, (15, B, model.nu))
  for t in range(15):
    phys.set_control(torch.as_tensor(tape[t])); phys.step(4)
    for e, o in enumerate(oracles):
      o.ctrl[:] = tape[t, e]; o.control_step(4)
    for f in ('qpos', 'qvel', 'act', 'sensordata'):
      g = getattr(phys.data, f).cpu().numpy()
      o = np.stack([getattr(oo, f) for oo in oracles])
      assert relerr(g, o) < TOL, (f, t, relerr(g, o))
