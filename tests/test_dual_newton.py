"""Dual (Woodbury) form of the Newton direction in the runtime-size acceleration kernels (b200mj.cu: dual_prepare,
newton_direction_dual, chol_solve_multi) against the oracle's primal Newton solver (MuJoCo's form, mj_solNewton).

The dual form is on by default for nv >= 32 and row buckets of at most 32 rows (the CMU humanoid); the tests force it
onto the 27-dof humanoid as well (B200MJ_TN=0 B200MJ_DUAL_MIN_NV=1), whose contacts are all closed-form primitives, so the
comparison with the oracle runs through tens of contact-rich control steps without a discontinuous convex pair ending
it. Tolerance: 1e-8 on qpos (north star: 1e-5 relative); contact pairs exact.
"""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_CHILD = r'''
import sys, json, numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, %(root)r + '/tests/emu')
from dm_control_b200 import testing_models as tm
from oracle import oracle as om
om.build()
name, B, ncontrol, nsub, emulate = %(name)r, %(B)d, %(ncontrol)d, %(nsub)d, %(emulate)d
model = tm.load(name)
q0, v0 = tm.initial_states(model, name, B, 3)
if emulate:
  import b200mj_emu as emu
  p = emu.EmuPhysics(model, B)
  p.data.qpos[:] = q0; p.data.qvel[:] = v0
  get = lambda x: np.asarray(x)
else:
  import torch
  from dm_control_b200.physics import BatchedPhysics
  p = BatchedPhysics(model, batch=B)
  p.data.qpos.copy_(torch.as_tensor(q0)); p.data.qvel.copy_(torch.as_tensor(v0))
  get = lambda x: x.cpu().numpy()
p.forward()
oracles = []
for e in range(B):
  o = om.OraclePhysics(model); o.qpos[:] = q0[e]; o.qvel[:] = v0[e]; o.forward(); oracles.append(o)
tape = np.random.RandomState(1).uniform(-1, 1, (ncontrol, B, model.nu))
worst, contacts, pairs_ok, rows = 0.0, 0, True, 0
gtype = np.asarray(model.geom_type)
tainted = [False] * B      # a convex pair resolved by MPR is a discontinuous function of the pose (DESIGN.md 3): stop comparing there
for t in range(ncontrol):
  if emulate: p.data.ctrl[:] = tape[t]
  else: p.data.ctrl.copy_(torch.as_tensor(tape[t]))
  p.step(nsub)
  q, v, ncon, cg, nefc = get(p.data.qpos), get(p.data.qvel), get(p.data.ncon).reshape(-1), get(p.data.contact_geom), get(p.data.nefc).reshape(-1)
  for e, o in enumerate(oracles):
    o.ctrl[:] = tape[t, e]; o.control_step(nsub)
    tainted[e] |= any(gtype[c.geom1] != 0 and (gtype[c.geom1] > 3 or gtype[c.geom2] > 3) for c in o.contact)
    if tainted[e]: continue
    worst = max(worst, float(np.abs(q[e] - o.qpos).max()), float(np.abs(v[e] - o.qvel).max()) / 10)
    pairs_ok &= int(ncon[e]) == o.ncon and [tuple(int(x) for x in r) for r in cg[e, :o.ncon]] == [(c.geom1, c.geom2) for c in o.contact]
    contacts += o.ncon
  rows = max(rows, int(nefc.max()))
print(json.dumps(dict(worst=worst, contacts=contacts, pairs_ok=bool(pairs_ok), max_nefc=rows)))
'''


def _run(name, B, ncontrol, nsub, emulate, **env):
  code = _CHILD % dict(root=ROOT, name=name, B=B, ncontrol=ncontrol, nsub=nsub, emulate=emulate)
  r = subprocess.run([sys.executable, '-c', code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=1500)
  assert r.returncode == 0, r.stderr[-3000:]
  return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.timeout(1800)
def test_dual_direction_matches_oracle_emulated():
  """Kernel source on the CPU emulation, dual form forced onto the humanoid: 20 control steps x 5 substeps in contact."""
  out = _run('humanoid', 6, 20, 5, 1, B200MJ_TN='0', B200MJ_DUAL_MIN_NV='1')
  assert out['pairs_ok'] and out['contacts'] > 50 and out['max_nefc'] > 10, out
  assert out['worst'] < 1e-8, out
  # the primal form of the same kernels on the same tape is the control: the dual form may not be much further away
  ref = _run('humanoid', 6, 20, 5, 1, B200MJ_TN='0', B200MJ_DUAL_MIN_NV='0')
  assert ref['pairs_ok'] and ref['worst'] < 1e-9, ref


@pytest.mark.gpu
@pytest.mark.parametrize('name,B,ncontrol,nsub,env', [
    ('humanoid', 32, 30, 5, dict(B200MJ_TN='0', B200MJ_DUAL_MIN_NV='1')),      # dual form forced on (runtime-size kernels)
    ('cmu_humanoid', 16, 5, 6, dict()),                                          # default: dual form for nv = 62
])
def test_dual_direction_matches_oracle_on_gpu(name, B, ncontrol, nsub, env):
  if os.environ.get('B200MJ_EMULATE_GPU') == '1':
    pytest.skip('spawns fresh interpreters on the device; the emulated twin is above')
  out = _run(name, B, ncontrol, nsub, 0, **env)
  assert out['pairs_ok'] and out['contacts'] > 0, out
  assert out['worst'] < 1e-7, out
