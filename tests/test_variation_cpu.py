"""Bookkeeping of the batched PhysicsVariator (dm_control_b200/variation.py) on a stand-in physics: no engine, no GPU."""
import types

import numpy as np
import pytest
import torch

from dm_control_b200.variation import PhysicsVariator


class _FakeModel:
  def __init__(self):
    self.fields = {'body_mass': np.array([0., 1., 2.]), 'geom_friction': np.array([[1., .005, .0001], [.5, .005, .0001]])}
    self.names = {'body': {'world': 0, 'a': 1, 'b': 2}, 'geom': {'g0': 0, 'g1': 1}}

  def name2id(self, name, kind):
    return self.names[kind][name]


def _physics(B=4):
  p = types.SimpleNamespace(model=_FakeModel(), batch=B, device=torch.device('cpu'), env_model_fields=(), env_model=None, dirty=0)

  def set_env_model_fields(names):
    old = p.env_model
    p.env_model = types.SimpleNamespace()
    for n in names:
      keep = old is not None and hasattr(old, n)
      setattr(p.env_model, n, getattr(old, n).clone() if keep else
              torch.as_tensor(p.model.fields[n])[None].repeat((B,) + (1,) * p.model.fields[n].ndim))
    p.env_model_fields = tuple(names)

  def mark_as_dirty():
    p.dirty += 1
  p.set_env_model_fields, p.mark_as_dirty = set_env_model_fields, mark_as_dirty
  return p


def test_first_application_enables_fields_and_remembers_each_environments_value():
  p = _physics()
  seen = []

  def var(init, cur, gen, n):
    seen.append((init.clone(), cur.clone(), n))
    return cur * 2
  v = PhysicsVariator()
  v.bind_attributes('body', ['a', 'b'], mass=var)
  mask = torch.tensor([True, False, True, False])
  v.apply_variations(p, None, env_mask=mask)
  assert p.env_model_fields == ('body_mass',) and p.dirty == 1
  assert torch.equal(p.env_model.body_mass, torch.tensor([[0., 2., 4.], [0., 1., 2.], [0., 2., 4.], [0., 1., 2.]]))
  v.apply_variations(p, None, env_mask=mask)
  init, cur, n = seen[-1]
  assert n == 2 and torch.equal(init, torch.tensor([[1., 2.]] * 2, dtype=torch.float64))
  assert torch.equal(cur, torch.tensor([[2., 4.]] * 2, dtype=torch.float64))
  p.env_model.body_mass[1] = torch.tensor([0., 5., 6.], dtype=torch.float64)     # rows customised after the first application
  v.apply_variations(p, None, env_mask=torch.tensor([False, True, False, False]))
  assert torch.equal(seen[-1][0], torch.tensor([[1., 2.]], dtype=torch.float64))   # still the remembered value
  v.reset_initial_values()
  v.apply_variations(p, None, env_mask=torch.tensor([False, True, False, False]))
  assert torch.equal(seen[-1][0], torch.tensor([[10., 12.]], dtype=torch.float64))  # re-read: the row as it stands


def test_fixed_values_broadcast_and_unbinding():
  p = _physics()
  v = PhysicsVariator()
  v.bind_attributes('geom', 'g1', friction=torch.tensor([.3, .01, .001], dtype=torch.float64))
  v.bind_attributes('body', 'a', mass=7.0)
  v.apply_variations(p)
  assert torch.equal(p.env_model.geom_friction[:, 1], torch.tensor([[.3, .01, .001]] * 4, dtype=torch.float64))
  assert torch.equal(p.env_model.geom_friction[:, 0], torch.tensor([[1., .005, .0001]] * 4, dtype=torch.float64))
  assert torch.all(p.env_model.body_mass[:, 1] == 7.0)
  v.bind_attributes('body', 'a', mass=None)
  p.env_model.body_mass.zero_()
  v.apply_variations(p)
  assert torch.all(p.env_model.body_mass == 0)       # unbound: untouched
  v.clear()
  p.env_model.geom_friction.zero_()
  v.apply_variations(p)
  assert torch.all(p.env_model.geom_friction == 0)


def test_empty_mask_changes_nothing_and_unsupported_attributes_are_refused():
  p = _physics()
  v = PhysicsVariator()
  v.bind_attributes('body', 'a', mass=3.0)
  v.apply_variations(p, env_mask=torch.zeros(4, dtype=torch.bool))
  assert torch.equal(p.env_model.body_mass, torch.tensor([[0., 1., 2.]] * 4, dtype=torch.float64))
  with pytest.raises(ValueError, match='geom_size'):
    v.bind_attributes('geom', 'g0', size=1.0)
  with pytest.raises(ValueError, match='actuator_gear'):
    v.bind_attributes('actuator', 'm', gear=1.0)
