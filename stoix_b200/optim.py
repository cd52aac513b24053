"""optax-shaped facade over the fused optimiser kernels (stx_clip_adam_step, stx_clip_radam_step, stx_clip_rmsprop_step).

`chain(clip_by_global_norm(m), adam(lr, eps=...))` mirrors the construction at
stoix/systems/ppo/anakin/ff_ppo.py:456-463.  The returned object's `.update` is what the reference
passes around as `update_fns`; `chain(clip_by_global_norm(m), radam(lr))` (ff_pqn.py:263-267) runs the RAdam rule and
`chain(clip_by_global_norm(m), rmsprop(lr))` (ff_impala.py:754-766) the RMSProp rule; the learner reads its hyper-parameters and runs BOTH optimisers
(actor and critic) in a single fused launch over the flat arenas."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Callable, List, NamedTuple, Optional, Sequence, Tuple, Union


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


@dataclass
class _Rmsprop:
    learning_rate: Union[float, Callable]
    decay: float = 0.9
    eps: float = 1e-8


def clip_by_global_norm(max_norm: float) -> _Clip:
    return _Clip(float(max_norm))


def adam(learning_rate, b1: float = 0.9, b2: float = 0.999, eps: float = 1e-8, eps_root: float = 0.0) -> _Adam:
    if eps_root != 0.0:
        raise NotImplementedError("eps_root != 0 is not used by the reference PPO and is not built")
    return _Adam(learning_rate, b1, b2, eps, eps_root)


def radam(learning_rate, b1: float = 0.9, b2: float = 0.999, eps: float = 1e-8, eps_root: float = 0.0, threshold: float = 5.0) -> _Radam:
    """optax.radam (scale_by_radam without nesterov, then the learning rate), as ff_pqn.py:263-267 chains it after the clip."""
    return _Radam(learning_rate, b1, b2, eps, eps_root, threshold)


def rmsprop(learning_rate, decay: float = 0.9, eps: float = 1e-8, initial_scale: float = 0.0, eps_in_sqrt: bool = True, centered: bool = False,
            momentum: Optional[float] = None, nesterov: bool = False, bias_correction: bool = False) -> _Rmsprop:
    """optax.rmsprop: scale_by_rms (nu = (1 - decay) g^2 + decay nu, u = g / sqrt(nu + eps)), then the learning rate.  Only the defaults
    IMPALA uses (ff_impala.py:754-766) are built; the state is the nu arena alone."""
    if centered or momentum is not None or nesterov or bias_correction:
        raise NotImplementedError("rmsprop: centered, momentum, nesterov and bias_correction are not used by the reference IMPALA and are "
                                  "not built")
    if initial_scale != 0.0 or not eps_in_sqrt:
        raise NotImplementedError("rmsprop: only initial_scale=0 and eps_in_sqrt=True (optax's defaults) are built")
    return _Rmsprop(learning_rate, float(decay), float(eps))


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

    def __init__(self, clip: Optional[_Clip], adam_: Union[_Adam, _Rmsprop]):
        self.clip, self.adam = clip, adam_

    @property
    def rule(self) -> str:
        """"radam" for an optax.radam stage, "rmsprop" for an optax.rmsprop stage, else "adam"."""
        return "radam" if isinstance(self.adam, _Radam) else "rmsprop" if isinstance(self.adam, _Rmsprop) else "adam"

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
        counts = torch.cat([state.count.reshape(-1)[:1], state.sched_count.reshape(-1)[:1]]).to(device=g.device, dtype=torch.int32)
        plan = adam_plan([(0, n, self)], g.device, counts)
        ops.clip_adam_step(plan, p, gg, mu, nu)
        new_state = OptState(plan.counts[0:1].clone(), mu[:n].view_as(state.mu), nu[:n].view_as(state.nu), plan.counts[1:2].clone())
        return p[:n].view_as(g), new_state   # parameters started at zero: what is left is the update -lr * u


def apply_updates(params, updates):
    """optax.apply_updates: params + updates (functional)."""
    p = GradientTransformation._flat(params)
    return p + GradientTransformation._flat(updates)


def adam_plan(segments: Sequence[Tuple[int, int, GradientTransformation]], device, counts) -> "ops.AdamPlan":
    """The ops.AdamPlan of one fused optimiser launch over `segments` = (offset, count, transformation): each segment takes its
    learning rate and clip norm from its transformation; the update rule, b1 / b2 / eps and the learning-rate decay come from the
    first one's stage and schedule (make_learning_rate attaches steps_per_update and num_updates to a decaying schedule; without
    one the kernels read neither).  `counts` (int32, one {count, schedule count} pair per segment, usually a learner state's
    arena_counts) becomes the plan's counters, so the kernel steps it in place."""
    from . import ops

    opt = segments[0][2]
    sched = opt.schedule
    if opt.rule == "rmsprop":  # the kernel reads the RMSProp decay from b2
        rule = {"rule": "rmsprop", "b1": 0.0, "b2": opt.adam.decay}
    else:
        rule = {"rule": "radam", "eps_root": opt.adam.eps_root, "threshold": opt.adam.threshold} if opt.rule == "radam" else {}
        rule.update(b1=opt.adam.b1, b2=opt.adam.b2)
    plan = ops.AdamPlan([(off, n, o.init_lr, o.max_grad_norm if o.clip is not None else 3.0e38) for off, n, o in segments], device,
                        eps=opt.adam.eps, decay=sched is not None,
                        steps_per_update=getattr(sched, "steps_per_update", 1), num_updates=getattr(sched, "num_updates", 1), **rule)
    plan.counts = counts
    return plan


def arena_state(tree, arena, segments: Sequence[Tuple[int, int]]) -> List[OptState]:
    """The optimiser state of a flat parameter arena: mu / nu arenas shaped like it and one int32 {count, schedule count} pair per
    segment (offset, count).  Returns one OptState of views per segment, and attaches arena, arena_mu, arena_nu and arena_counts
    to `tree`: the fused kernels work on the whole arenas, and a checkpoint of the tree carries them."""
    import torch

    mu, nu = torch.zeros_like(arena), torch.zeros_like(arena)
    counts = torch.zeros(2 * len(segments), dtype=torch.int32, device=arena.device)
    tree.arena, tree.arena_mu, tree.arena_nu, tree.arena_counts = arena, mu, nu, counts
    return [OptState(counts[2 * i:2 * i + 1], mu[off:off + n], nu[off:off + n], counts[2 * i + 1:2 * i + 2])
            for i, (off, n) in enumerate(segments)]


def chain(*parts) -> GradientTransformation:
    clip = next((p for p in parts if isinstance(p, _Clip)), None)
    adam_ = next((p for p in parts if isinstance(p, (_Adam, _Rmsprop))), None)
    if adam_ is None:
        raise ValueError("chain() needs an adam(), radam() or rmsprop() stage")
    return GradientTransformation(clip, adam_)
