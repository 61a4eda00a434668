"""Cost of per-environment model fields on the flagship workload (suite.humanoid:run, BatchedEnvironment.step with
graphs), in three arms alternated in one process:

  (a) no per-environment fields
  (b) all eleven fields per environment, holding the model's own values
  (c) all eleven fields per environment, randomised (scales in [0.8, 1.2]; the same draw every round)

Prints one JSON line: env-steps/s (graph-replayed control steps, CUDA events around the timed window) and the median
time of the physics kernel group (eager steps with CUDA events around the b200mj_step call) per arm and round, the
card's name and power limit read in the same run, and whether (a) and (b) produced bitwise-equal observations.

  python tools/env_model_cost.py [--batch 8192] [--steps 200] [--warmup 50] [--rounds 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from dm_control_b200 import suite  # noqa: E402
from dm_control_b200.physics import ENV_MODEL_FIELDS  # noqa: E402


def _card():
  name = torch.cuda.get_device_name(0)
  try:
    out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = 'unavailable'
  return name, out


def _env(arm, batch):
  env = suite.load('humanoid', 'run', batch=batch, seed=0)
  env.physics.check_errors = False
  env._graph_step = True
  p = env.physics
  if arm != 'a':
    p.set_env_model_fields(ENV_MODEL_FIELDS)
    if arm == 'c':
      g = torch.Generator(device=p.device).manual_seed(1)
      for f in ENV_MODEL_FIELDS:
        t = getattr(p.env_model, f)
        t.mul_(0.8 + 0.4 * torch.rand(t.shape, generator=g, dtype=t.dtype, device=t.device))
      p.mark_as_dirty()
  env.reset()
  return env


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, default=8192)
  ap.add_argument('--steps', type=int, default=200)
  ap.add_argument('--warmup', type=int, default=50)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--kernel-steps', type=int, default=8)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('env_model_cost.py measures on the GPU; no CUDA device found')
  B, arms = a.batch, ('a', 'b', 'c')
  nu = 21
  g = torch.Generator(device='cuda').manual_seed(7)
  actions = [torch.rand(B, nu, generator=g, device='cuda', dtype=torch.float64) * 2 - 1 for _ in range(8)]
  envs = {arm: _env(arm, B) for arm in arms}
  res = {arm: dict(env_steps_per_s=[], kernel_group_ms=[]) for arm in arms}
  obs_equal = True
  for arm in arms:
    for i in range(a.warmup):
      envs[arm].step(actions[i % 8])
  for _ in range(a.rounds):
    last = {}
    for arm in arms:
      env = envs[arm]
      torch.cuda.synchronize()
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for i in range(a.steps):
        ts = env.step(actions[i % 8])
      e1.record()
      torch.cuda.synchronize()
      res[arm]['env_steps_per_s'].append(B * a.steps / (e0.elapsed_time(e1) / 1e3))
      last[arm] = torch.cat([v.reshape(B, -1) for v in ts.observation.values()], dim=1).clone()
      kev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.kernel_steps)]
      for i in range(a.kernel_steps):
        env.step(actions[i % 8], timing=kev[i])
      torch.cuda.synchronize()
      res[arm]['kernel_group_ms'].append(statistics.median(s.elapsed_time(t) for s, t in kev))
    obs_equal = obs_equal and torch.equal(last['a'], last['b'])
  name, power = _card()
  out = dict(workload='suite.humanoid:run', batch=B, steps=a.steps, rounds=a.rounds, card=name,
             power_limit_and_max_sm_clock=power, obs_bitwise_equal_a_b=obs_equal,
             arms={arm: dict(env_steps_per_s=[round(x) for x in r['env_steps_per_s']],
                             median_env_steps_per_s=round(statistics.median(r['env_steps_per_s'])),
                             kernel_group_ms=[round(x, 4) for x in r['kernel_group_ms']],
                             median_kernel_group_ms=round(statistics.median(r['kernel_group_ms']), 4)) for arm, r in res.items()})
  print(json.dumps(out))
  assert obs_equal, '(a) and (b) observations differ'


if __name__ == '__main__':
  main()
