"""optax-shaped facade over the fused optimiser kernels (stx_clip_adam_step, stx_clip_radam_step).

`chain(clip_by_global_norm(m), adam(lr, eps=...))` mirrors the construction at
stoix/systems/ppo/anakin/ff_ppo.py:456-463.  The returned object's `.update` is what the reference
passes around as `update_fns`; `chain(clip_by_global_norm(m), radam(lr))` (ff_pqn.py:263-267) runs the RAdam rule; the learner reads its hyper-parameters and runs BOTH optimisers
(actor and critic) in a single fused launch over the flat arenas."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Callable, NamedTuple, Optional, Union


@dataclass
class _Clip:
    max_norm: float


@dataclass
class _Adam:
    learning_rate: Union[float, Callable]
    b1: float = 0.9
    b2: float = 0.999
    eps: float = 1e-8
    eps_root: float = 0.0


@dataclass
class _Radam(_Adam):
    threshold: float = 5.0


def clip_by_global_norm(max_norm: float) -> _Clip:
    return _Clip(float(max_norm))


def adam(learning_rate, b1: float = 0.9, b2: float = 0.999, eps: float = 1e-8, eps_root: float = 0.0) -> _Adam:
    if eps_root != 0.0:
        raise NotImplementedError("eps_root != 0 is not used by the reference PPO and is not built")
    return _Adam(learning_rate, b1, b2, eps, eps_root)


def radam(learning_rate, b1: float = 0.9, b2: float = 0.999, eps: float = 1e-8, eps_root: float = 0.0, threshold: float = 5.0) -> _Radam:
    """optax.radam (scale_by_radam without nesterov, then the learning rate), as ff_pqn.py:263-267 chains it after the clip."""
    return _Radam(learning_rate, b1, b2, eps, eps_root, threshold)


class OptState(NamedTuple):
    """(ScaleByAdamState{count, mu, nu}, ScaleByScheduleState{count}) as views into the flat state."""

    count: Any
    mu: Any
    nu: Any
    sched_count: Any


class GradientTransformation:
    """optax.GradientTransformation with `init` / `update` (stoix/systems/ppo/anakin/ff_ppo.py:449-463, 264-273).

    `update(updates, state, params=None) -> (updates, new_state)` is functional like optax: it runs the fused clip + Adam
    kernel (stx_clip_adam_step, ONE segment) on copies and returns the parameter DELTA, so
    `apply_updates(params, updates)` reproduces optax's two-step form.  The learner itself does not go through this
    face: it steps both optimisers in place in one launch over the shared arena and only reads the hyper-parameters."""

    def __init__(self, clip: Optional[_Clip], adam_: _Adam):
        self.clip, self.adam = clip, adam_

    @property
    def rule(self) -> str:
        """"radam" for an optax.radam stage, else "adam"."""
        return "radam" if isinstance(self.adam, _Radam) else "adam"

    def plan_kwargs(self) -> dict:
        """The AdamPlan arguments of this stage's update rule."""
        if self.rule == "radam":
            return {"rule": "radam", "eps_root": self.adam.eps_root, "threshold": self.adam.threshold}
        return {}

    @property
    def max_grad_norm(self) -> float:
        return self.clip.max_norm if self.clip is not None else float("inf")

    @property
    def init_lr(self) -> float:
        lr = self.adam.learning_rate
        return float(getattr(lr, "init_lr", lr))

    @property
    def schedule(self) -> Optional[Callable]:
        lr = self.adam.learning_rate
        return lr if callable(lr) else None

    @staticmethod
    def _flat(x):
        return x.flat if hasattr(x, "flat") and not hasattr(x, "numel") else x

    def init(self, params) -> OptState:
        """(ScaleByAdamState{count=0, mu=0, nu=0}, ScaleByScheduleState{count=0}) for a flat parameter tensor / ParamTree."""
        import torch

        p = self._flat(params)
        z = lambda: torch.zeros(1, dtype=torch.int32, device=p.device)
        return OptState(z(), torch.zeros_like(p), torch.zeros_like(p), z())

    def update(self, updates, state: OptState, params=None):
        import torch

        from . import ops

        g = self._flat(updates).contiguous()
        n = g.numel()
        pad = (-n) % 4  # the kernel wants 16-byte aligned arenas; a private copy is padded instead of asking the caller
        buf = lambda src: torch.cat([src.reshape(-1).float(), src.new_zeros(pad, dtype=torch.float32)]) if pad else src.reshape(-1).float().clone()
        p = torch.zeros(n + pad, dtype=torch.float32, device=g.device)
        mu, nu, gg = buf(state.mu), buf(state.nu), buf(g)
        sched = self.schedule
        plan = ops.AdamPlan([(0, n, self.init_lr, self.max_grad_norm if self.clip is not None else 3.0e38)], g.device,
                            b1=self.adam.b1, b2=self.adam.b2, eps=self.adam.eps, decay=sched is not None,
                            steps_per_update=getattr(sched, "steps_per_update", 1), num_updates=getattr(sched, "num_updates", 1),
                            **self.plan_kwargs())
        plan.counts[0:1].copy_(state.count.reshape(-1)[:1])
        plan.counts[1:2].copy_(state.sched_count.reshape(-1)[:1])
        ops.clip_adam_step(plan, p, gg, mu, nu)
        new_state = OptState(plan.counts[0:1].clone(), mu[:n].view_as(state.mu), nu[:n].view_as(state.nu), plan.counts[1:2].clone())
        return p[:n].view_as(g), new_state   # parameters started at zero: what is left is the update -lr * u


def apply_updates(params, updates):
    """optax.apply_updates: params + updates (functional)."""
    p = GradientTransformation._flat(params)
    return p + GradientTransformation._flat(updates)


def chain(*parts) -> GradientTransformation:
    clip = next((p for p in parts if isinstance(p, _Clip)), None)
    adam_ = next((p for p in parts if isinstance(p, _Adam)), None)
    if adam_ is None:
        raise ValueError("chain() needs an adam() or radam() stage")
    return GradientTransformation(clip, adam_)
