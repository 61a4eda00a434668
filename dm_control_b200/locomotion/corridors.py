"""CMU humanoid + WallsCorridor + RunThroughCorridor, batched (BASELINE.json config 5).

Reference: locomotion/examples/basic_cmu_2019.py:34-63 (`cmu_humanoid_run_walls`), locomotion/tasks/corridors.py:33-158,
locomotion/arenas/corridors.py:94-175 (planes), :330-440 (walls), locomotion/walkers/{cmu_humanoid,legacy_base,base}.py
(observables). The model is the compiled fixture `assets/cmu_corridor_walls.npz` (tools/make_model_fixtures.py builds it
from the reference XML); the 25 wall boxes are per-environment geoms re-drawn every episode.
"""
from __future__ import annotations

import collections
import math

import numpy as np
import torch

from .. import rewards, testing_models
from ..physics import BatchedPhysics
from . import composer

N_WALLS = 25
_CORRIDOR_WIDTH, _WALL_GAP, _WALL_HEIGHT, _WALL_THICKNESS, _X_PADDING = 10.0, 4.0, 3.0, 0.16, 2.0
_WALL_WIDTH_RANGE = (1.0, 7.0)                 # distributions.Uniform(1, 7), basic_cmu_2019.py:44
_TARGET_VELOCITY, _TERMINATE_AT_HEIGHT = 3.0, -0.5
_PHYSICS_TIMESTEP, _CONTROL_TIMESTEP, _TIME_LIMIT = 0.005, 0.03, 30
_TOUCH_THRESHOLD, _TORQUE_THRESHOLD = 1e-3, 60   # legacy_base.py:29, cmu_humanoid.py:183

OUTPUTS = ('xpos', 'xmat', 'subtree_linvel', 'sensordata', 'ncon', 'nefc', 'solver_niter', 'contact_geom')


class CMUWalker:
  """Index tables of the position-controlled CMU humanoid inside the compiled model (cmu_humanoid.py:296-356)."""

  def __init__(self, model, device):
    m = model
    bid = lambda n: m.name2id(n, 'body')
    self.root, self.head = bid('root'), bid('head')
    self.end_effectors = [bid(n) for n in ('rradius', 'lradius', 'rfoot', 'lfoot')]      # cmu_humanoid.py:330-335
    parent = np.asarray(m.body_parentid)
    def subtree(b):
      out, todo = [], [b]
      while todo:
        x = todo.pop(); out.append(x)
        todo.extend(int(c) for c in np.nonzero(parent == x)[0] if c != x)
      return out
    walker_bodies = set(subtree(self.root))
    foot_bodies = set(subtree(bid('lfoot'))) | set(subtree(bid('rfoot')))                 # ground_contact_geoms, :318-321
    gb = np.asarray(m.geom_bodyid)
    self.nonfoot_geom = torch.as_tensor(np.array([(int(b) in walker_bodies) and (int(b) not in foot_bodies) for b in gb]), device=device)
    self.ground_geom = m.name2id('ground_plane', 'geom')
    # observable joints = the joint of every actuator, in actuator (alphabetical) order (cmu_humanoid.py:337-340)
    trn = np.asarray(m.actuator_trnid)
    self.joint_qpos = torch.as_tensor(np.asarray(m.jnt_qposadr)[trn].astype(np.int64), device=device)
    self.joint_dof = torch.as_tensor(np.asarray(m.jnt_dofadr)[trn].astype(np.int64), device=device)
    names = m.ordered_names['sensor']
    adr, dim, typ = np.asarray(m.sensor_adr), np.asarray(m.sensor_dim), np.asarray(m.sensor_type)
    def cols(pred):
      idx = [a + k for n, a, d, t in zip(names, adr, dim, typ) if pred(n, int(t)) for k in range(int(d))]
      return torch.as_tensor(np.array(idx, dtype=np.int64), device=device)
    self.s_end_effectors = cols(lambda n, t: n.endswith('_end_effector'))
    self.s_gyro = cols(lambda n, t: t == 3)
    self.s_accel = cols(lambda n, t: t == 1)
    self.s_veloc = cols(lambda n, t: t == 2)
    self.s_touch = cols(lambda n, t: t == 0)
    self.s_torque = cols(lambda n, t: t == 5)
    self.appendages = torch.as_tensor(np.array(self.end_effectors + [self.head], dtype=np.int64), device=device)
    self.end_effector_ids = torch.as_tensor(np.array(self.end_effectors, dtype=np.int64), device=device)


class RunThroughCorridor(composer.Task):
  """Reward for running down the corridor at 3 m/s; ends when a non-foot geom touches the ground or an end effector
  drops below -0.5 m (tasks/corridors.py:33-158)."""

  def __init__(self, physics, seed=0, contact_termination=True, egocentric_camera=False):
    self._walker = CMUWalker(physics.model, physics.device)
    # walker.observables.egocentric_camera (legacy_base.py:276-279: the head camera, 64 x 64): ray-cast by the rendering
    # hand-off (dm_control_b200/render.py), every environment seeing its own walls
    self._camera = None
    if egocentric_camera:
      from .. import render
      self._camera = render.Camera(physics, height=64, width=64, camera_id='egocentric', sites=False)
    self._contact_termination = contact_termination
    self._gen = torch.Generator(device=physics.device).manual_seed(seed)
    m = physics.model
    self.wall_geoms = [m.name2id(f'wall_{k}', 'geom') for k in range(N_WALLS)]
    physics.set_variable_geoms(self.wall_geoms)
    self._failure = torch.zeros(physics.batch, dtype=torch.bool, device=physics.device)
    k = torch.arange(N_WALLS, dtype=torch.float64, device=physics.device)
    self._wall_x = _WALL_GAP - _X_PADDING + _WALL_GAP * k                  # arenas/corridors.py:407-440, no initial padding
    self._wall_sign = torch.where(k.long() % 2 == 0, 1.0, -1.0).to(torch.float64)   # swap_wall_side=True: sides alternate, first wall on +y

  @property
  def walker(self):
    return self._walker

  def initialize_episode_geoms(self, physics, env_mask):
    """`WallsCorridor.regenerate` per environment (arenas/corridors.py:394-440): wall widths ~ U(1, 7), alternating sides."""
    B, dev = physics.batch, physics.device
    w = _WALL_WIDTH_RANGE[0] + (_WALL_WIDTH_RANGE[1] - _WALL_WIDTH_RANGE[0]) * torch.rand(B, N_WALLS, generator=self._gen, device=dev, dtype=torch.float64)
    pos = torch.stack([self._wall_x.expand(B, -1), self._wall_sign * (_CORRIDOR_WIDTH - w) / 2, torch.full_like(w, _WALL_HEIGHT / 2)], dim=2)
    size = torch.stack([torch.full_like(w, _WALL_THICKNESS / 2), w / 2, torch.full_like(w, _WALL_HEIGHT / 2)], dim=2)
    d = physics.data
    if env_mask is None:
      d.var_geom_pos.copy_(pos); d.var_geom_size.copy_(size)
    else:
      d.var_geom_pos[env_mask] = pos[env_mask]; d.var_geom_size[env_mask] = size[env_mask]

  def initialize_episode(self, physics, env_mask):
    # UprightInitializer + shift_pose((0.5, 0, 0)) (walkers/initializers, tasks/corridors.py:98-111): the compiled model's
    # qpos0 IS that pose (upright root at x = 0.5, every joint at 0) and Physics.reset has just written it
    if env_mask is None:
      self._failure.zero_()
    else:
      self._failure[env_mask] = False

  def before_step(self, physics, action):
    physics.set_control(action)            # walker.apply_action (walkers/base.py:150-153)

  def after_step(self, physics):
    w, d = self._walker, physics.data
    fail = torch.zeros(physics.batch, dtype=torch.bool, device=physics.device)
    if self._contact_termination:
      cg = d.contact_geom.reshape(physics.batch, -1, 2).long()
      valid = torch.arange(cg.shape[1], device=physics.device)[None, :] < d.ncon[:, None]
      g1, g2 = cg[:, :, 0].clamp_min(0), cg[:, :, 1].clamp_min(0)
      bad = ((g1 == w.ground_geom) & w.nonfoot_geom[g2]) | ((g2 == w.ground_geom) & w.nonfoot_geom[g1])
      fail = (bad & valid).any(dim=1)
    z = d.xpos.reshape(physics.batch, -1, 3).index_select(1, w.end_effector_ids)[:, :, 2]
    self._failure = fail | (z < _TERMINATE_AT_HEIGHT).any(dim=1)

  def get_reward(self, physics):
    xvel = physics.data.subtree_linvel.reshape(physics.batch, -1, 3)[:, self._walker.root, 0]
    return rewards.tolerance(xvel, bounds=(_TARGET_VELOCITY, _TARGET_VELOCITY), margin=_TARGET_VELOCITY, sigmoid='linear',
                             value_at_margin=0.0)

  def should_terminate_episode(self, physics):
    return self._failure

  def get_discount(self, physics):
    return torch.where(self._failure, 0.0, 1.0).to(torch.float64)

  def get_observation(self, physics):
    w, d, B = self._walker, physics.data, physics.batch
    xpos = d.xpos.reshape(B, -1, 3); xmat = d.xmat.reshape(B, -1, 9)
    root_pos, root_mat = xpos[:, w.root], xmat[:, w.root].reshape(B, 3, 3)
    obs = collections.OrderedDict()
    obs['walker/joints_pos'] = d.qpos.index_select(1, w.joint_qpos)
    obs['walker/joints_vel'] = d.qvel.index_select(1, w.joint_dof)
    obs['walker/actuator_activation'] = d.act
    obs['walker/body_height'] = root_pos[:, 2]
    obs['walker/end_effectors_pos'] = d.sensordata.index_select(1, w.s_end_effectors)
    rel = xpos.index_select(1, w.appendages) - root_pos[:, None, :]
    obs['walker/appendages_pos'] = torch.bmm(rel, root_mat).reshape(B, -1)          # np.dot(end_effector - torso, xmat)
    obs['walker/world_zaxis'] = xmat[:, w.root, 6:]
    obs['walker/sensors_gyro'] = d.sensordata.index_select(1, w.s_gyro)
    obs['walker/sensors_accelerometer'] = d.sensordata.index_select(1, w.s_accel)
    obs['walker/sensors_velocimeter'] = d.sensordata.index_select(1, w.s_veloc)
    obs['walker/sensors_torque'] = torch.tanh(2 * d.sensordata.index_select(1, w.s_torque) / _TORQUE_THRESHOLD)
    obs['walker/sensors_touch'] = (d.sensordata.index_select(1, w.s_touch) > _TOUCH_THRESHOLD).to(torch.float64)
    if self._camera is not None:
      obs['walker/egocentric_camera'] = self._camera.render()
    return obs


def cmu_humanoid_run_walls(batch=1, seed=0, time_limit=_TIME_LIMIT, egocentric_camera=False, **physics_kw):
  physics_kw.setdefault('outputs', OUTPUTS + (('geom_xpos', 'geom_xmat') if egocentric_camera else ()))
  physics = BatchedPhysics(testing_models.load('cmu_corridor_walls'), batch=batch, **physics_kw)
  task = RunThroughCorridor(physics, seed=seed, egocentric_camera=egocentric_camera)
  return composer.BatchedComposerEnvironment(physics, task, time_limit=time_limit, physics_timestep=_PHYSICS_TIMESTEP,
                                             control_timestep=_CONTROL_TIMESTEP)
