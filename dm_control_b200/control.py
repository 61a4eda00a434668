"""`BatchedEnvironment`: B lock-stepped copies of `dm_control.rl.control.Environment` (rl/control.py:35-153).

Same call order per step (`before_step` -> `physics.step(n_sub_steps)` -> `after_step` -> reward -> observation),
same sub-step arithmetic (`compute_n_steps`, control.py:168-194), same time-limit rule, but every quantity has a
leading batch axis and stays on the device. Episodes that hit the time limit (or whose physics diverged) are reset
in place on the next `step`, per environment (the reference resets the single env on the next call, control.py:102).
"""
from __future__ import annotations

import collections

import torch


def compute_n_steps(control_timestep, physics_timestep, tolerance=1e-8):
  """Reference: rl/control.py:168-194 (same error text)."""
  if control_timestep < physics_timestep:
    raise ValueError('Control timestep ({}) cannot be smaller than physics timestep ({}).'.format(
        control_timestep, physics_timestep))
  if abs((control_timestep / physics_timestep - round(control_timestep / physics_timestep))) > tolerance:
    raise ValueError('Control timestep ({}) must be an integer multiple of physics timestep ({})'.format(
        control_timestep, physics_timestep))
  return int(round(control_timestep / physics_timestep))


TimeStep = collections.namedtuple('TimeStep', ['step_type', 'reward', 'discount', 'observation'])
FIRST, MID, LAST = 0, 1, 2


class BatchedEnvironment:

  def __init__(self, physics, task, time_limit=float('inf'), control_timestep=None, n_sub_steps=None,
               legacy_step=True, auto_reset=True, graph_task_ops=False, graph_step=False):
    self._physics, self._task = physics, task
    physics.legacy_step = legacy_step
    if n_sub_steps is not None and control_timestep is not None:
      raise ValueError('Both n_sub_steps and control_timestep were supplied.')
    if n_sub_steps is not None:
      self._n_sub_steps = n_sub_steps
    elif control_timestep is not None:
      self._n_sub_steps = compute_n_steps(control_timestep, physics.timestep())
    else:
      self._n_sub_steps = 1
    self._step_limit = float('inf') if time_limit == float('inf') else time_limit / (physics.timestep() * self._n_sub_steps)
    self._step_count = torch.zeros(physics.batch, dtype=torch.int64, device=physics.device)
    self._reset_next = torch.ones(physics.batch, dtype=torch.bool, device=physics.device)
    self._auto_reset = auto_reset
    # host-side upper bound of every environment's step count: while it is below the step limit no environment can
    # be LAST, so step() need not read `_reset_next` back (a device->host sync per step otherwise)
    self._count_ub = float('inf')     # unknown until the first check
    # Optional: replay the task's reward/observation torch ops (~80 tiny launches) as one CUDA graph. The returned
    # reward / observation tensors are then static buffers that the next step overwrites.
    self._graph_task_ops = graph_task_ops
    self._graph = None
    self._graph_out = None
    # Optional: the WHOLE control step — before_step, the physics call (its ~40 kernel launches on the engine's
    # streams), after_step, reward, observation, step counters — captured once per physics-flag combination and
    # replayed as one CUDA graph: one launch per step from the host, so a busy host cannot starve the GPU. Needs
    # `physics.check_errors = False` (the warning check is a device->host sync); the action is copied into a static
    # buffer; returned tensors are static buffers that the next step overwrites.
    self._graph_step = graph_step
    self._step_graphs = {}
    self._graph_epoch = None          # the physics' _launch_epoch the graphs were captured at
    # Optional device-side epilogue of a control step, `hook(reward, observation, discount)`: runs (and is captured)
    # with the step — e.g. packing the observation dict into one [B, k] block for a single device->host copy.
    self.post_step_hook = None

  @property
  def physics(self):
    return self._physics

  @property
  def task(self):
    return self._task

  @property
  def n_sub_steps(self):
    return self._n_sub_steps

  def control_timestep(self):
    return self._physics.timestep() * self._n_sub_steps

  def reset(self):
    self._task.initialize_episode(self._physics, None)
    self._step_count.zero_()
    self._reset_next.zero_()
    self._count_ub = 0
    obs = self._task.get_observation(self._physics)
    B = self._physics.batch
    return TimeStep(torch.full((B,), FIRST, device=self._physics.device), None, None, obs)

  def _reward_and_observation(self):
    if not self._graph_task_ops:
      return self._task.get_reward(self._physics), self._task.get_observation(self._physics)
    if self._graph is None:
      # warm up eagerly on a side stream (allocator + lazy module loads), then capture once
      s = torch.cuda.Stream(device=self._physics.device)
      s.wait_stream(torch.cuda.current_stream(self._physics.device))
      with torch.cuda.stream(s):
        for _ in range(2):
          self._task.get_reward(self._physics); self._task.get_observation(self._physics)
      torch.cuda.current_stream(self._physics.device).wait_stream(s)
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g):
        out = (self._task.get_reward(self._physics), self._task.get_observation(self._physics))
      self._graph, self._graph_out = g, out
    self._graph.replay()
    return self._graph_out

  def _device_step(self, action, timing=None, eager_task_ops=False):
    """Everything of a control step that runs on the device (capturable: no host reads)."""
    self._task.before_step(action, self._physics)
    if timing is not None:
      timing[0].record()
    self._physics.step(self._n_sub_steps)
    if timing is not None:
      timing[1].record()
    self._task.after_step(self._physics)
    if eager_task_ops:
      reward, obs = self._task.get_reward(self._physics), self._task.get_observation(self._physics)
    else:
      reward, obs = self._reward_and_observation()
    self._step_count += 1
    last = self._step_count >= self._step_limit
    discount = torch.ones_like(reward)
    # task termination (control.py:113-118): None = the task never terminates; otherwise a [B] tensor holding the
    # terminal discount for the environments that end now and NaN for the others. The time limit wins (discount 1).
    get_term = getattr(self._task, 'get_termination', None)
    term = get_term(self._physics) if get_term is not None else None
    if term is not None:
      ended = ~torch.isnan(term)
      discount = torch.where(ended & ~last, term, discount)
      last = last | ended
    step_type = torch.where(last, LAST, MID)
    if self.post_step_hook is not None:
      self.post_step_hook(reward, obs, discount)
    return reward, obs, discount, last, step_type, term is not None

  def _graphed_step(self, action):
    phys = self._physics
    phys._sync_model()
    if self._graph_epoch != phys._launch_epoch:
      # a captured step launches with the model, io and per-environment tables of its capture: re-capture after any change
      self._step_graphs.clear()
      self._graph_epoch = phys._launch_epoch
    key = phys._flags()
    entry = self._step_graphs.get(key)
    if entry is None:
      # first call with this flag combination: run eagerly (allocations, lazy module loads), capture on the next one
      self._step_graphs[key] = 'warm'
      return self._device_step(action, eager_task_ops=True)
    if entry == 'warm':
      static_action = torch.empty_like(action)
      static_action.copy_(action)
      pos_current = phys._pos_current
      g = torch.cuda.CUDAGraph()
      torch.cuda.synchronize(phys.device)
      with torch.cuda.graph(g):
        out = self._device_step(static_action, eager_task_ops=True)
      # the capture did not execute anything: restore the facade's bookkeeping and the step counter's value, then replay
      after = phys._pos_current
      phys._pos_current = pos_current
      entry = self._step_graphs[key] = (g, static_action, out, after)
    g, static_action, out, after = entry
    static_action.copy_(action)
    g.replay()
    phys._pos_current = after
    return out

  def step(self, action, timing=None):
    """One control step for every environment. `timing`: optional (start, end) CUDA events recorded around the
    physics call (bench.py times the step's kernel group with them); no effect on the result."""
    if self._auto_reset and self._count_ub >= self._step_limit:
      if bool(self._reset_next.any()):
        mask = self._reset_next
        self._task.initialize_episode(self._physics, mask)
        self._step_count[mask] = 0
        self._reset_next = torch.zeros_like(mask)
      self._count_ub = int(self._step_count.max())      # slow path only: one more readback, then exact again
    if self._graph_step and timing is None and not self._physics.check_errors:
      reward, obs, discount, last, step_type, may_end = self._graphed_step(action)
    else:
      reward, obs, discount, last, step_type, may_end = self._device_step(action, timing)
    self._count_ub += 1
    if may_end:
      self._count_ub = float('inf')       # episodes may end at any step: check the flags on the next call
    self._reset_next = last
    return TimeStep(step_type, reward, discount, obs)
