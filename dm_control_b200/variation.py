"""Batched `PhysicsVariator`: per-environment variations of model fields (composer/variation/__init__.py:90-136).

The reference's `PhysicsVariator` writes `physics.bind(element).<attr>` of one `Physics` per episode. Here one
`BatchedPhysics` holds B environments, each standing for one reference `Physics`, and a variation is drawn for the
environments of an `env_mask` only (a masked auto-reset must not touch the others). The values land in the
environments' rows of the per-environment model fields (`BatchedPhysics.set_env_model_fields`), which the first
`apply_variations` enables for the fields it touches, keeping fields already enabled and their values.

A variation is a fixed value or a callable `(initial_value, current_value, generator, n) -> [n, ...]`, where `...` is
the shape `bind` gives one environment (`[k]`, `[k, w]`, or without the `k` axis for a single name; a joint's
`damping` / `armature` keep one column per dof). As in the reference, the initial value is what each environment holds
when a variation is first applied (remembered for all B environments then); `initial_value` and `current_value` are
those of the n environments being varied, and `generator` is what `apply_variations` was given. No distributions are
provided: a task passes its own callable, e.g.
`lambda init, cur, g, n: init * (0.5 + torch.rand(init.shape, generator=g, dtype=init.dtype, device=init.device))`.
"""
from __future__ import annotations

import torch

from .binding import model_field, model_rows
from .physics import check_env_model_fields


class _VariationInfo:
  __slots__ = ('initial_value', 'variation')

  def __init__(self, variation):
    self.initial_value = None
    self.variation = variation


class PhysicsVariator:
  """Per-environment variations of the model fields a BatchedPhysics can hold per environment (ENV_MODEL_FIELDS)."""

  def __init__(self):
    self._variations = {}      # (kind, names) -> {attribute: _VariationInfo}

  def bind_attributes(self, kind, names, **kwargs):
    """Binds variations to attributes of the elements `names` of `kind` ('body', 'geom', 'joint', 'actuator'); the
    attribute names are `bind`'s (`mass`, `friction`, `damping`, `stiffness`, `gainprm`, ...). A variation of None
    unbinds."""
    key = (kind, names if isinstance(names, str) else tuple(names))
    check_env_model_fields([model_field(kind, a) for a in kwargs])
    attrs = self._variations.setdefault(key, {})
    for attr, variation in kwargs.items():
      if variation is None:
        attrs.pop(attr, None)
      else:
        attrs[attr] = _VariationInfo(variation)

  def apply_variations(self, physics, generator=None, env_mask=None):
    """Evaluates every bound variation once for the environments of `env_mask` ([B] bool; None: all) and writes the
    result into their rows only."""
    need = [model_field(kind, a) for (kind, _), attrs in self._variations.items() for a in attrs]
    missing = [f for f in dict.fromkeys(need) if f not in physics.env_model_fields]
    if missing:
      physics.set_env_model_fields(tuple(physics.env_model_fields) + tuple(missing))
    envs = (torch.arange(physics.batch, device=physics.device) if env_mask is None else
            torch.as_tensor(env_mask, device=physics.device).to(torch.bool).nonzero().reshape(-1))
    n = int(envs.numel())
    if n == 0:
      return
    m = physics.model
    for (kind, names), attrs in self._variations.items():
      single = isinstance(names, str)
      ids = [m.name2id(x, kind) for x in ([names] if single else names)]
      for attr, info in attrs.items():
        field, ragged, rows_idx = model_rows(m, kind, attr, ids)
        rows_idx = torch.as_tensor(rows_idx, dtype=torch.int64, device=physics.device)
        rows = getattr(physics.env_model, field)                # [B, nrows, *width]
        k_width = (len(rows_idx),) + rows.shape[2:]
        shape = k_width[1:] if single and not ragged else k_width     # bind's per-environment shape
        if info.initial_value is None:
          info.initial_value = rows[:, rows_idx].reshape((physics.batch,) + shape).clone()
        current = rows[envs][:, rows_idx].reshape((n,) + shape)
        v = info.variation
        value = v(info.initial_value[envs], current, generator, n) if callable(v) else v
        value = torch.as_tensor(value, dtype=rows.dtype, device=physics.device)
        rows[envs[:, None], rows_idx[None, :]] = value.expand((n,) + shape).reshape((n,) + k_width)
    physics.mark_as_dirty()

  def clear(self):
    """Clears all bound variations."""
    self._variations.clear()

  def reset_initial_values(self):
    """Forgets the remembered initial values: the next application takes the environments' values again."""
    for attrs in self._variations.values():
      for info in attrs.values():
        info.initial_value = None
