"""The CUDA engine's own source (dm_control_b200/csrc/b200mj.cu), compiled for the CPU with the lock-step emulation
of tests/emu/cuda_emu.h, against the oracle — no GPU needed.

This is NOT a product path (nothing in dm_control_b200/ loads the emulation build, and `BatchedPhysics` still refuses
to run without CUDA); it exists so that the round's CPU test tier exercises the kernels' logic — layouts and aliasing,
the packed Cholesky, collision/constraint assembly, the split-kernel handover and the launch orchestration behind the
C ABI — and not only the host code around them. The `-m gpu` tests remain the parity tests proper: the emulation says
nothing about races, memory spaces or performance, and `rsqrt` is `1/sqrt` here.
"""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'emu'))
import b200mj_emu as emu   # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dof_models   # noqa: E402

from dm_control_b200 import testing_models as tm   # noqa: E402

pytestmark = pytest.mark.timeout(600)
TOL = 1e-8


def relerr(a, b):
  a, b = np.asarray(a), np.asarray(b)
  return float(np.max(np.abs(a - b)) / max(1.0, np.max(np.abs(b)))) if a.size else 0.0


def _setup(name, B, seed, oracle_mod, **kw):
  model, q0, v0 = dof_models.load(name, B, seed)
  p = emu.EmuPhysics(model, B, **kw)
  p.data.qpos[:] = q0; p.data.qvel[:] = v0
  p.forward()
  oracles = []
  for e in range(B):
    o = oracle_mod.OraclePhysics(model)
    o.qpos[:] = q0[e]; o.qvel[:] = v0[e]; o.forward()
    oracles.append(o)
  return model, p, oracles


@pytest.mark.parametrize('name,B', [('cartpole', 8), ('pendulum_free', 8), ('cheetah', 16), ('humanoid', 16),
                                    ('quadruped', 8), ('slide_box', 4), ('free_box', 4), ('cmu_humanoid', 4)])
def test_forward_fields(name, B, oracle_mod):
  model, p, oracles = _setup(name, B, 11, oracle_mod)
  for f in ('xpos', 'xquat', 'xmat', 'xipos', 'geom_xpos', 'geom_xmat', 'site_xpos', 'site_xmat', 'subtree_com', 'cvel',
            'qfrc_bias', 'qfrc_passive', 'qacc', 'qfrc_constraint', 'qfrc_actuator', 'sensordata'):
    g = getattr(p.data, f).reshape(B, -1)
    o = np.stack([np.asarray(getattr(oo, f)).reshape(-1) for oo in oracles])
    assert relerr(g, o) < 1e-10, (name, f, relerr(g, o))
  assert relerr(p.data.qM, np.stack([oo.M_dense() for oo in oracles])) < 1e-13       # packed triangle -> dense output
  np.testing.assert_array_equal(p.data.ncon, [o.ncon for o in oracles])
  np.testing.assert_array_equal(p.data.nefc, [o.nefc for o in oracles])
  for e, o in enumerate(oracles):
    np.testing.assert_allclose(p.data.efc_force[e, :o.nefc], o.efc('efc_force'), rtol=1e-7, atol=1e-7)


@pytest.mark.parametrize('name,B,ncontrol,nsub', [('cartpole', 8, 60, 1), ('pendulum_free', 8, 50, 2), ('cheetah', 16, 100, 1),
                                                   ('humanoid', 16, 20, 5), ('quadruped', 8, 15, 4), ('cmu_humanoid', 4, 6, 6)] +
                         [(dof_models.name(nv), 3, 8, 2) for nv in dof_models.NV_TARGETS])      # tests/dof_models.py
def test_rollout(name, B, ncontrol, nsub, oracle_mod):
  """Fixed action tape, legacy step ordering (engine.py:147-162); every control step is compared: state to 1e-8,
  contact count and geom pairs exactly, sensors to 1e-7."""
  model, p, oracles = _setup(name, B, 0, oracle_mod)
  tape = np.random.RandomState(1).uniform(-1, 1, (ncontrol, B, model.nu))
  saw_contact = 0
  for t in range(ncontrol):
    p.data.ctrl[:] = tape[t]
    p.step(nsub)
    for e, o in enumerate(oracles):
      o.ctrl[:] = tape[t, e]
      o.control_step(nsub)
      assert relerr(p.data.qpos[e], o.qpos) < TOL and relerr(p.data.qvel[e], o.qvel) < TOL, (name, t, e)
      assert int(p.data.ncon[e]) == o.ncon, (name, t, e)
      pairs = [(c.geom1, c.geom2) for c in o.contact]
      assert [tuple(x) for x in p.data.contact_geom[e, :o.ncon]] == pairs, (name, t, e)
      saw_contact += o.ncon
      if model.nsensordata:
        o.subtree_vel()
        assert relerr(p.data.sensordata[e], o.sensordata) < 1e-7, (name, t, e)
      assert relerr(p.data.subtree_com[e], o.subtree_com) < 1e-9
  if name not in ('cartpole',):
    assert saw_contact > 0, 'the rollout should exercise the contact path'
  assert not p.data.warning.any()


def test_nstep_equals_repeated_steps_and_batch_independence(oracle_mod):
  """engine_test.py:627-663 on the emulated kernels: step(3) is bitwise 3 x step(1), and a call of more than 64
  physics steps, step(70), bitwise 2 x step(35); an environment's trajectory does not depend on which batch it sits in."""
  for name, whole, chunks in (('humanoid', [3], [1, 1, 1]), ('cheetah', [70], [35, 35])):
    model = tm.load(name)
    q0, v0 = tm.initial_states(model, name, 3, 5)
    ctrl = np.random.RandomState(2).uniform(-1, 1, (3, model.nu))
    def run(sel, chunks):
      p = emu.EmuPhysics(model, len(sel))
      p.data.qpos[:] = q0[sel]; p.data.qvel[:] = v0[sel]; p.forward(); p.data.ctrl[:] = ctrl[sel]
      for n in chunks:
        p.step(n)
      return p.data.qpos.copy(), p.data.qvel.copy(), p.data.sensordata.copy()
    a = run([0, 1, 2], whole)
    b = run([0, 1, 2], chunks)
    c = run([1], whole)
    for x, y in zip(a, b):
      np.testing.assert_array_equal(x, y)
    for x, y in zip(a, c):
      np.testing.assert_array_equal(x[1:2], y)


def test_bad_control_and_divergence_warnings():
  """engine_test.py:487-547 semantics at the C ABI: NaN ctrl -> BADCTRL counter (ctrl treated as 0), a huge qpos ->
  BADQPOS and an in-place reset to qpos0."""
  model = tm.load('cheetah')
  p = emu.EmuPhysics(model, 3)
  p.forward()
  p.data.ctrl[1, 0] = np.nan
  p.data.qpos[2, 0] = 1e15
  p.step(1)
  w = p.data.warning
  BADQPOS, BADCTRL = 4, 7                         # mjtWarning indices (include/b200mj_model_fields.h)
  assert w[0].sum() == 0
  assert w[1, BADCTRL] == 1 and w[1].sum() == 1
  assert w[2, BADQPOS] == 1
  assert np.isfinite(p.data.qpos).all() and abs(p.data.qpos[2, 0]) < 1.0


def test_workspaces_fit_and_buckets_are_described():
  p = emu.EmuPhysics(tm.load('humanoid'), 1)
  d = p.describe()
  assert d['pos_envs_per_cta'] == 5 and d['pos_workspace_bytes'] * 5 <= 227 * 1024
  rows = [b['rows'] for b in d['acc_buckets']]
  assert rows == sorted(rows) and rows[-1] == p.model.njmax
  assert all(b['workspace_bytes'] <= b['last_step_workspace_bytes'] <= 227 * 1024 for b in d['acc_buckets'])
  # packed M/H: the smallest bucket holds 16 environments per SM (1 KB reserved per CTA)
  assert (227 * 1024) // (d['acc_buckets'][0]['workspace_bytes'] + 1024) >= 16


def test_environment_groups_and_large_batch(oracle_mod):
  """Batches of 2048 and more are split into two environment groups on separate streams (b200mj_step); the split
  must not change any environment's result. 2050 cheetahs against the same states stepped as three smaller batches
  and, for a sample, against the oracle."""
  model = tm.load('cheetah')
  B = 2050
  q0, v0 = tm.initial_states(model, 'cheetah', B, 3)
  ctrl = np.random.RandomState(4).uniform(-1, 1, (B, model.nu))
  def run(sel):
    p = emu.EmuPhysics(model, len(sel))
    p.data.qpos[:] = q0[sel]; p.data.qvel[:] = v0[sel]; p.forward(); p.data.ctrl[:] = ctrl[sel]
    for _ in range(3):
      p.step(2)
    return p.data.qpos.copy(), p.data.qvel.copy(), p.data.ncon.copy()
  big = run(np.arange(B))
  for lo, hi in ((0, 700), (700, 1500), (1500, B)):
    part = run(np.arange(lo, hi))
    for x, y in zip(big, part):
      np.testing.assert_array_equal(x[lo:hi], y)
  for e in (0, 1024, 1025, 2049):
    o = oracle_mod.OraclePhysics(model)
    o.qpos[:] = q0[e]; o.qvel[:] = v0[e]; o.forward(); o.ctrl[:] = ctrl[e]
    for _ in range(3):
      o.control_step(2)
    assert relerr(big[0][e], o.qpos) < TOL and relerr(big[1][e], o.qvel) < TOL and int(big[2][e]) == o.ncon


_KNOB_SCRIPT = r'''
import hashlib, os, sys
import numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], 'tests', 'emu'))
import b200mj_emu as emu
from dm_control_b200 import testing_models as tm
h = hashlib.sha256()
for name, B, nsteps, nsub in (('humanoid', 6, 6, 5), ('quadruped', 4, 5, 4), ('pendulum_free', 4, 20, 2)):
  model = tm.load(name)
  q0, v0 = tm.initial_states(model, name, B, 0)
  p = emu.EmuPhysics(model, B)
  p.data.qpos[:] = q0; p.data.qvel[:] = v0; p.forward()
  tape = np.random.RandomState(9).uniform(-1, 1, (nsteps, B, model.nu))
  for t in range(nsteps):
    p.data.ctrl[:] = tape[t]; p.step(nsub)
    for f in ('qpos', 'qvel', 'sensordata', 'xpos', 'subtree_linvel', 'ncon', 'contact_geom', 'qacc', 'efc_force'):
      h.update(np.ascontiguousarray(getattr(p.data, f)).tobytes())
print(h.hexdigest())
'''


def test_launch_knobs_do_not_change_results():
  """The fused and the split path, any row-bucket partition, the CTA widths of every kernel and the convex-pair
  dispatch are scheduling choices: every one of them must reproduce the default path bit for bit (states, sensors,
  contacts, constraint forces, over rollouts with contacts)."""
  import subprocess
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  def digest(**env):
    e = dict(os.environ); e.update(env)
    out = subprocess.run([sys.executable, '-c', _KNOB_SCRIPT, root], env=e, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    return out.stdout.strip().splitlines()[-1]
  # the default path: acceleration kernels with nv fixed at compile time (register-resident algebra)
  from concurrent.futures import ThreadPoolExecutor      # the variants are independent child processes: run them side by side
  pool = ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 2))
  ref_f = pool.submit(digest)
  variants = (dict(B200MJ_BUCKETS='4,16'), dict(B200MJ_BUCKETS='6,12,24'), dict(B200MJ_EPB_POS='2'),
                # acceleration launches: unsynchronised one-warp CTAs, phase-aligned CTAs of 2 warps (4: the default)
                dict(B200MJ_ACC_WARPS='1'), dict(B200MJ_ACC_WARPS='2'),
                # the emulator running the lanes of every block in descending instead of ascending order: a cross-lane
                # dependency through shared memory that no collective or barrier separates would change the result
                dict(B200MJ_EMU_ORDER='reverse'),
                # convex pairs one per lane instead of by the whole warp (cvx_pair vs cvx_pair_warp): the same contact to the last bit
                dict(B200MJ_CVX_WARP='0'))
  futs = [(k, pool.submit(digest, **k)) for k in variants]
  # B200MJ_TN=0: the runtime-size acceleration kernels share their arithmetic with the fused kernel, so there the
  # fused and the split path must agree bit for bit as well
  ref0_f = pool.submit(digest, B200MJ_TN='0')
  variants0 = (dict(B200MJ_SPLIT='0'), dict(B200MJ_BUCKETS='4,16'), dict(B200MJ_ENVS_PER_BLOCK='2', B200MJ_SPLIT='0'),
               dict(B200MJ_EMU_ORDER='reverse', B200MJ_SPLIT='0'))
  futs0 = [(k, pool.submit(digest, B200MJ_TN='0', **k)) for k in variants0]
  ref, ref0 = ref_f.result(), ref0_f.result()
  for knobs, f in futs:
    assert f.result() == ref, knobs
  for knobs, f in futs0:
    assert f.result() == ref0, knobs
  pool.shutdown()


_TN_SCRIPT = r'''
import os, sys, json
import numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], 'tests', 'emu'))
import b200mj_emu as emu
from dm_control_b200 import testing_models as tm
out = {}
for name, B, nsteps, nsub in (('humanoid', 6, 6, 5), ('quadruped', 4, 5, 4), ('cheetah', 4, 8, 3)):
  model = tm.load(name)
  q0, v0 = tm.initial_states(model, name, B, 0)
  p = emu.EmuPhysics(model, B)
  p.data.qpos[:] = q0; p.data.qvel[:] = v0; p.forward()
  tape = np.random.RandomState(9).uniform(-1, 1, (nsteps, B, model.nu))
  for t in range(nsteps):
    p.data.ctrl[:] = tape[t]; p.step(nsub)
  out[name] = dict(qpos=p.data.qpos.tolist(), qvel=p.data.qvel.tolist(), ncon=p.data.ncon.tolist(), sens=p.data.sensordata.tolist())
print(json.dumps(out))
'''


def test_compile_time_size_kernels_match_runtime_size_kernels():
  """The acceleration kernels with nv fixed at compile time (tn_* algebra: other summation order, other Cholesky
  variant) against the runtime-size kernels on the same rollouts: same contacts, states equal to rounding noise."""
  import subprocess, json
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  res = []
  for tn in ('1', '0'):
    e = dict(os.environ, B200MJ_TN=tn)
    out = subprocess.run([sys.executable, '-c', _TN_SCRIPT, root], env=e, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    res.append(json.loads(out.stdout.strip().splitlines()[-1]))
  for name in res[0]:
    a, b = res[0][name], res[1][name]
    assert a['ncon'] == b['ncon'], name
    for f in ('qpos', 'qvel', 'sens'):
      x, y = np.asarray(a[f]), np.asarray(b[f])
      assert np.abs(x - y).max() <= 1e-8 * (1 + np.abs(y).max()), (name, f, np.abs(x - y).max())


def test_malformed_blob_is_refused_and_capacity_change_reallocates(oracle_mod):
  """b200mj_model_create validates the directory of the blob; b200mj_model_set_capacity drops handover rows sized for
  the old capacities (the next step reallocates) — exercised through the emulated library's own host code."""
  import ctypes
  L = emu.load()
  model = tm.load('cheetah')
  idata, rdata = model.pack()
  def create(i, r):
    h = ctypes.c_void_p()
    rc = L.b200mj_model_create(i.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), i.size,
                               r.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), r.size, ctypes.byref(h))
    if rc == 0:
      L.b200mj_model_destroy(h)
    return rc
  assert create(idata, rdata) == 0
  bad = idata.copy(); bad[1] = idata.size + 5            # first field's length runs past the blob
  assert create(bad, rdata) == -1
  bad = idata.copy(); bad[0] = -3
  assert create(bad, rdata) == -1
  assert create(idata[:20].copy(), rdata) == -1          # directory truncated
  # capacity change between steps
  L.b200mj_model_set_capacity.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
  p = emu.EmuPhysics(model, 2)
  q0, v0 = tm.initial_states(model, 'cheetah', 2, 0)
  p.data.qpos[:] = q0; p.data.qvel[:] = v0; p.forward(); p.step(2)
  assert L.b200mj_model_set_capacity(p._h, int(model.nconmax) + 7, int(model.njmax) + 40) == 0
  # io arrays sized by the old capacities stay valid for the fields that do not depend on them; re-bind the others
  m2 = model.copy(); m2.set_capacity(int(model.nconmax) + 7, int(model.njmax) + 40)
  p2 = emu.EmuPhysics(m2, 2)
  p2.data.qpos[:] = q0; p2.data.qvel[:] = v0; p2.forward(); p2.step(2)
  for name in ('efc_force', 'contact_dist', 'contact_pos', 'contact_frame', 'contact_geom', 'contact_efc_address'):
    a = getattr(p2.data, name)
    setattr(p.data, name, np.zeros_like(a))
    setattr(p._io, name, ctypes.cast(getattr(p.data, name).ctypes.data, dict(emu.blib.IO_FIELDS)[name]))
  p.step(2); p2.step(2)
  np.testing.assert_array_equal(p.data.qpos, p2.data.qpos)
  np.testing.assert_array_equal(p.data.qvel, p2.data.qvel)


@pytest.mark.parametrize('nconmax,njmax', [(2, 96), (32, 6), (1, 3)])
def test_capacity_overflow_raises_warnings_like_the_oracle(nconmax, njmax, oracle_mod):
  """Too small <size nconmax njmax>: contacts / rows beyond the capacity are dropped with mjWARN_CONTACTFULL /
  mjWARN_CNSTRFULL; kernel and oracle must drop the same ones, keep running, and agree on the state."""
  model = tm.load('humanoid').copy()
  model.set_capacity(nconmax, njmax)
  B = 4
  q0, v0 = tm.initial_states(model, 'humanoid', B, 0)
  q0[:, 2] = 0.12                                  # lying low: many floor contacts at once
  p = emu.EmuPhysics(model, B)
  p.data.qpos[:] = q0; p.data.qvel[:] = v0; p.forward()
  oracles = []
  for e in range(B):
    o = oracle_mod.OraclePhysics(model)
    o.qpos[:] = q0[e]; o.qvel[:] = v0[e]; o.forward()
    oracles.append(o)
  CONTACTFULL, CNSTRFULL = 1, 2
  for t in range(6):
    p.step(2)
    for e, o in enumerate(oracles):
      o.control_step(2)
      assert int(p.data.ncon[e]) == o.ncon <= nconmax and int(p.data.nefc[e]) == o.nefc <= njmax
      assert relerr(p.data.qpos[e], o.qpos) < 1e-7 and relerr(p.data.qvel[e], o.qvel) < 1e-6, (t, e)
  wk = p.data.warning
  wo = np.stack([np.asarray(o.warning)[:8] for o in oracles])
  assert wk[:, CONTACTFULL].sum() + wk[:, CNSTRFULL].sum() > 0, 'the capacities should have overflowed'
  np.testing.assert_array_equal(wk[:, CONTACTFULL] > 0, wo[:, CONTACTFULL] > 0)
  np.testing.assert_array_equal(wk[:, CNSTRFULL] > 0, wo[:, CNSTRFULL] > 0)


@pytest.mark.parametrize('name', ['humanoid', 'pendulum_free', 'quadruped'])
def test_non_legacy_ordering_and_applied_forces(name, oracle_mod):
  """`legacy_step = False` (engine.py:176: mj_step x n, nothing recomputed afterwards) and user forces
  (`qfrc_applied`, `xfrc_applied`) are served by the fused kernel: against the oracle's mj_step."""
  model = tm.load(name)
  B = 3
  q0, v0 = tm.initial_states(model, name, B, 2)
  p = emu.EmuPhysics(model, B, legacy_step=False, applied_forces=True)
  p.data.qpos[:] = q0; p.data.qvel[:] = v0
  rs = np.random.RandomState(6)
  p.data.qfrc_applied[:] = rs.uniform(-2, 2, p.data.qfrc_applied.shape)
  p.data.xfrc_applied[:, 1:] = rs.uniform(-5, 5, p.data.xfrc_applied[:, 1:].shape)
  p.forward()
  oracles = []
  for e in range(B):
    o = oracle_mod.OraclePhysics(model)
    o.qpos[:] = q0[e]; o.qvel[:] = v0[e]
    o.qfrc_applied[:] = p.data.qfrc_applied[e]; o.xfrc_applied[:] = p.data.xfrc_applied[e]
    o.forward()
    oracles.append(o)
    assert relerr(p.data.qacc[e], o.qacc) < 1e-9
  for t in range(8):
    ctrl = rs.uniform(-1, 1, (B, model.nu))
    p.data.ctrl[:] = ctrl
    p.step(3)
    for e, o in enumerate(oracles):
      o.ctrl[:] = ctrl[e]
      o.step(3)
      assert relerr(p.data.qpos[e], o.qpos) < TOL and relerr(p.data.qvel[e], o.qvel) < TOL, (name, t, e)


def test_step_host_and_disable_flags(oracle_mod):
  """b200mj_step_host (host action buffer in, observation block out) equals b200mj_step on the same inputs;
  b200mj_model_set_disableflags / the extra flags of b200mj_forward act like `model.disable()` (core.py:389-426)."""
  model = tm.load('cheetah')
  B = 4
  q0, v0 = tm.initial_states(model, 'cheetah', B, 1)
  a, b = emu.EmuPhysics(model, B), emu.EmuPhysics(model, B)
  for p in (a, b):
    p.data.qpos[:] = q0; p.data.qvel[:] = v0; p.forward()
  ctrl = np.random.RandomState(3).uniform(-1, 1, (B, model.nu))
  obs_host = np.zeros((B, model.nq))
  a.step_host(ctrl.copy(), a.data.qpos, obs_host, nstep=2)
  b.data.ctrl[:] = ctrl; b.step(2)
  np.testing.assert_array_equal(a.data.qpos, b.data.qpos)
  np.testing.assert_array_equal(obs_host, b.data.qpos)
  np.testing.assert_array_equal(a.data.ctrl, ctrl)
  # gravity + contact disabled: a resting cheetah with zero control does not accelerate
  c = emu.EmuPhysics(model, 1)
  c.set_disableflags((1 << 4) | (1 << 6))
  c.forward()
  assert np.abs(c.data.qacc).max() < 1e-12 and int(c.data.ncon[0]) == 0
  # actuation disabled only for this forward (reset()/after_reset(), engine.py:325-333)
  d = emu.EmuPhysics(model, 1)
  d.data.ctrl[:] = 1.0
  d.forward(extra_disableflags=1 << 10)
  assert np.abs(d.data.actuator_force).max() == 0
  d.forward()
  assert np.abs(d.data.actuator_force).max() > 0


@pytest.mark.parametrize('name,nsub', [('humanoid', 5), ('quadruped', 4), ('cartpole', 1), ('pendulum_free', 2)])
@pytest.mark.parametrize('outputs,sensors,full_final', [((), False, False), (('sensordata',), True, False), (('xpos', 'ncon'), False, True)])
def test_null_outputs_and_flag_combinations_leave_the_state_alone(name, nsub, outputs, sensors, full_final):
  """Any output pointer may be NULL and the sensor / full-final work is optional (include/b200mj.h): whatever subset
  is requested, the state trajectory is bit-identical to the run that materialises everything, and the requested
  outputs carry the same values."""
  model = tm.load(name)
  B = 3
  q0, v0 = tm.initial_states(model, name, B, 0)
  tape = np.random.RandomState(12).uniform(-1, 1, (6, B, model.nu))
  def run(**kw):
    p = emu.EmuPhysics(model, B, **kw)
    p.data.qpos[:] = q0; p.data.qvel[:] = v0; p.forward()
    for t in range(6):
      p.data.ctrl[:] = tape[t]; p.step(nsub)
    return p
  full = run()
  part = run(outputs=outputs, sensors=sensors, full_final=full_final)
  for f in ('qpos', 'qvel', 'act', 'qacc_warmstart', 'time'):
    np.testing.assert_array_equal(getattr(part.data, f), getattr(full.data, f))
  for f in outputs:
    if f == 'ncon' and not full_final:
      continue
    np.testing.assert_array_equal(getattr(part.data, f), getattr(full.data, f))


_ASAN_SCRIPT = r'''
import os, sys
import numpy as np
root = sys.argv[1]
sys.path.insert(0, root); sys.path.insert(0, os.path.join(root, 'tests', 'emu'))
import b200mj_emu as emu
emu._SO = sys.argv[2]
emu.build = lambda force=False: emu._SO
from dm_control_b200 import testing_models as tm
for name, B, nsteps, nsub in (('humanoid', 4, 6, 5), ('quadruped', 3, 4, 4), ('pendulum_free', 4, 16, 2), ('cartpole', 3, 8, 1),
                               ('cmu_humanoid', 2, 2, 6), ('cheetah', 2050, 2, 1)):
  model = tm.load(name)
  q0, v0 = tm.initial_states(model, name, B, 0)
  p = emu.EmuPhysics(model, B)
  p.data.qpos[:] = q0; p.data.qvel[:] = v0; p.forward()
  tape = np.random.RandomState(9).uniform(-1, 1, (nsteps, B, model.nu))
  for t in range(nsteps):
    p.data.ctrl[:] = tape[t]; p.step(nsub)
print('ASAN RUN COMPLETE')
'''


def test_address_sanitizer_finds_nothing():
  """memcheck without a GPU: the kernel source built with -fsanitize=address under the emulation. Every "device"
  buffer (model blob, io arrays, handover rows) is a heap allocation with red zones, so an out-of-bounds access of the
  kernels is reported with file:line; a deliberately undersized output buffer is the positive control."""
  import shutil, subprocess
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  libasan = subprocess.run(['g++', '-print-file-name=libasan.so'], capture_output=True, text=True).stdout.strip()
  if not os.path.isabs(libasan) or not os.path.exists(libasan):
    pytest.skip('libasan not available')
  so = os.path.join(root, 'tests', 'emu', '_build', 'libb200mj_emu_asan.so')
  if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in emu._DEPS):
    os.makedirs(os.path.dirname(so), exist_ok=True)
    subprocess.check_call(['g++', '-std=c++20', '-O1', '-g', '-fno-omit-frame-pointer', '-fsanitize=address', '-fPIC', '-shared',
                           '-pthread', '-x', 'c++', '-DB200MJ_CPU_EMU', '-Wno-unknown-pragmas', '-I' + emu._HERE, '-o', so, emu._SRC])
  env = dict(os.environ, LD_PRELOAD=libasan, ASAN_OPTIONS='detect_leaks=0:detect_stack_use_after_return=0')
  out = subprocess.run([sys.executable, '-c', _ASAN_SCRIPT, root, so], env=env, capture_output=True, text=True, timeout=900)
  assert 'ERROR: AddressSanitizer' not in out.stderr, out.stderr[-3000:]
  assert out.returncode == 0 and 'ASAN RUN COMPLETE' in out.stdout, (out.returncode, out.stderr[-2000:])
  control = _ASAN_SCRIPT.split("for name, B")[0] + '''
import ctypes
model = tm.load('cheetah'); p = emu.EmuPhysics(model, 4)
small = np.zeros((3, model.nv))
p._io.qacc = ctypes.cast(small.ctypes.data, dict(emu.blib.IO_FIELDS)['qacc'])
p.forward()
'''
  out = subprocess.run([sys.executable, '-c', control, root, so], env=env, capture_output=True, text=True, timeout=300)
  assert 'heap-buffer-overflow' in out.stderr and 'write_outputs' in out.stderr


@pytest.mark.parametrize('name,B,ncalls', [('humanoid', 6, 12), ('quadruped', 4, 8), ('pendulum_free', 4, 30), ('cheetah', 2050, 3)])
def test_reuse_of_trailing_position_stage_is_bit_identical(name, B, ncalls):
  """B200MJ_STEP_REUSE_POS: skipping the leading position kernel when the previous call's trailing mj_step1 already
  produced its handover must not change a single bit — states, sensors, contacts, warnings — for calls of 1..3 steps."""
  model = tm.load(name)
  q0, v0 = tm.initial_states(model, name, B, 0)
  rs = np.random.RandomState(8)
  tape = rs.uniform(-1, 1, (ncalls, B, model.nu)); ns = rs.choice([1, 2, 3], ncalls)
  def run(reuse):
    p = emu.EmuPhysics(model, B, reuse_pos=reuse)
    p.data.qpos[:] = q0; p.data.qvel[:] = v0; p.forward()
    out = []
    for t in range(ncalls):
      p.data.ctrl[:] = tape[t]; p.step(int(ns[t]))
      out.append([np.array(getattr(p.data, f)) for f in ('qpos', 'qvel', 'sensordata', 'ncon', 'nefc', 'contact_geom', 'qacc', 'efc_force', 'xpos', 'subtree_linvel', 'warning')])
    return out, emu.load().b200mj_launch_count()
  L = emu.load(); L.b200mj_launch_count.restype = ctypes.c_int64
  n0 = L.b200mj_launch_count(); a, n1 = run(False); b, n2 = run(True)
  for x, y in zip(a, b):
    for u, v in zip(x, y):
      np.testing.assert_array_equal(u, v)
  groups = 2 if B >= 2048 else 1
  # one position launch saved per call and group after the first — except for a one-step call that follows a longer one:
  # the trailing mj_step1 dumps what the acceleration-stage sensors need only after one-step calls, so that call
  # recomputes its position stage
  saved = sum(1 for t in range(1, ncalls) if not (ns[t] == 1 and ns[t - 1] > 1 and model.nsensordata > 0))
  assert (n1 - n0) - (n2 - n1) == saved * groups
