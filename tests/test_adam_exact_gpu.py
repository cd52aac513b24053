"""Every launch form of the clip + Adam step (K4), one optimiser step at a time, against the fp64 reference of
tests/adam_reference.py with its derived per-element bounds.

Each step is checked from the kernel's OWN pre-step state (copied to the host just before the launch), so nothing is chained
and nothing drifts.  Exact: the step counters, the bf16 shadow (== round-to-nearest-even of the new fp32 parameters), the
gradient arena (K4 must not write it) and every float outside the optimiser segments in the parameters, both moments and the
shadow.  Within the bounds: parameters, moments and the reported pre-clip global norm.

Forms: the local form (norm pass + grid barrier) on three segment layouts through a whole schedule; the prenorm form as the
bf16 learner chains it (the sum-of-squares partials come from K3's gradient reduction); both through the learner (the CUDA
graph on, as shipped).  The one-shot all-reduce form is checked the same way in
tests/test_distributed_gpu.py::test_fused_allreduce_kernel_on_one_device."""
import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from tests import adam_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _t(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype, device=DEV)


def _snap(p, mu, nu, counts, shadow=None, g=None, gnorm=None) -> dict:
    """Host copies (synchronising) of the optimiser state."""
    h = lambda t: None if t is None else t.detach().float().cpu().numpy().astype(np.float64 if t.dtype == torch.bfloat16 else np.float32)
    return dict(p=h(p), mu=h(mu), nu=h(nu), counts=counts.cpu().numpy().astype(np.int64), shadow=h(shadow), g=h(g), gnorm=h(gnorm))


# ---------------------------------------------------------------------------------------------------------------------------
# local form: segment layouts x a whole LR schedule
# ---------------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("decay,grad_scale", [(True, 1.0), (False, 0.25)])
@pytest.mark.parametrize("name", R.LAYOUTS)
def test_local_form_steps_through_the_schedule(name, decay, grad_scale):
    """steps_per_update 3, num_updates 4: all 12 steps up to the last step of the last update (lr = init_lr / 4, where
    1 - k / num_updates cancels most).  Every step has one segment clipped and one not; segment 0's gradient is all zero on odd
    steps; the padding of the gradient holds 1e3 (the kernel must not read it) and that of the other arenas sentinels."""
    from stoix_b200 import ops

    segs, total = R.layout(name)
    rng = np.random.default_rng(2 * R.LAYOUTS.index(name) + int(decay))
    p, mu, nu, counts = R.make_state(segs, total, rng)
    P, MU, NU = _t(p), _t(mu), _t(nu)
    SH = ops.cast_bf16(P)
    plan = ops.AdamPlan(segs, DEV, decay=decay, steps_per_update=3, num_updates=4)
    h = R.Hyper(grad_scale=grad_scale, decay=decay, steps_per_update=3, num_updates=4)
    for st in range(12):
        G = _t(R.make_grad(segs, total, rng, grad_scale, st))
        pre = _snap(P, MU, NU, plan.counts, SH, G)
        ops.clip_adam_step(plan, P, G, MU, NU, grad_scale=grad_scale, params_bf16=SH)
        got = _snap(P, MU, NU, plan.counts, SH, G, plan.gnorm)
        want = R.step(pre["p"], pre["mu"], pre["nu"], pre["counts"], pre["g"], segs, h)
        R.check(got, want, pre, label=f"{name} step {st}")
        assert want.clipped.any() and not want.clipped.all()


# ---------------------------------------------------------------------------------------------------------------------------
# prenorm (the benchmark's path)
# ---------------------------------------------------------------------------------------------------------------------------


def _net(rng, D, A, head_scale):
    p = O.init_mlp(rng, [D, 256, 256, A], head_scale)
    for i in range(3):
        p.b[i] = rng.standard_normal(p.b[i].shape) * 0.1
    p.W[-1] = rng.standard_normal(p.W[-1].shape) * 0.3
    return p


def _bf16_problem(D, A, mb, seed):
    from stoix_b200 import ops

    rng = np.random.default_rng(seed)
    B = 2 * mb
    actor, critic = _net(rng, D, A, 0.3), _net(rng, D, 1, 1.0)
    sa, sc = ops.MlpSpec((D, 256, 256, A)), ops.MlpSpec((D, 256, 256, 1))
    _, coff, total = ops.arena_offsets(sa, sc)
    segs = [(0, sa.param_count, 3e-3, 1e6), (coff, sc.param_count, 1e-3, 1e-6)]   # the actor never clips, the critic always
    p, mu, nu, _ = R.make_state(segs, total, rng)
    p[: sa.param_count] = actor.flat()
    p[coff: coff + sc.param_count] = critic.flat()
    batch = ops.PpoBatch(_t(rng.standard_normal((B, D))).to(torch.bfloat16), _t(rng.integers(0, A, B), torch.int32),
                         _t(-rng.random(B) - 1.0), _t(rng.standard_normal(B)), _t(rng.standard_normal(B) * 2), _t(rng.standard_normal(B)),
                         adv_stats=_t(np.array([0.1, 0.7])), perm=_t(rng.permutation(B), torch.int32))
    return sa, sc, segs, total, p, mu, nu, batch


SHAPES = [(D, A, mb) for D in (8, 64) for A in (1, 8, 16) for mb in (128, 4096, 32768)]   # mb 32768: the benchmark's minibatch


@pytest.mark.parametrize("form", ["prenorm"])
@pytest.mark.parametrize("D,A,mb", SHAPES)
def test_bf16_update_forms(D, A, mb, form):
    """prenorm: ppo_minibatch_grads(bf16, overwrite, adam_scratch) then clip_adam_step(prenorm) with nothing enqueued between
    them, so the programmatic-dependent-launch pairing is the one the learner ships.  The pre-state
    is copied before K3 (neither K3 nor the reduction writes it), the gradient and the post-state after the step; the reported
    norm must be the fp64 norm of the gradient arena K3 wrote.  Two steps: the adam count and the schedule (spu 2) advance."""
    from stoix_b200 import ops

    sa, sc, segs, total, p, mu, nu, batch = _bf16_problem(D, A, mb, D * 1000 + A * 10 + mb)
    P, MU, NU = _t(p), _t(mu), _t(nu)
    SH = ops.cast_bf16(P)
    G, metrics = torch.zeros(total, device=DEV), torch.zeros(8, device=DEV)
    ws = ops.ppo_workspace(sa, sc, mb, ops.STX_PREC_BF16, DEV)
    plan = ops.AdamPlan(segs, DEV, decay=True, steps_per_update=2, num_updates=4)
    h = R.Hyper(decay=True, steps_per_update=2, num_updates=4)
    for st in range(2):
        pre = _snap(P, MU, NU, plan.counts, SH)
        ops.ppo_minibatch_grads(sa, sc, P, batch, st * mb, mb, 0.2, 0.01, 0.5, True, G, metrics, ws, precision=ops.STX_PREC_BF16,
                                param_arena_bf16=SH, overwrite=True, adam_scratch=plan.scratch)
        ops.clip_adam_step(plan, P, G, MU, NU, params_bf16=SH, prenorm=True)
        got = _snap(P, MU, NU, plan.counts, SH, None, plan.gnorm)
        g = G.cpu().numpy()
        want = R.step(pre["p"], pre["mu"], pre["nu"], pre["counts"], g, segs, h, norm=R.NORM_DOUBLE)
        R.check(got, want, pre, label=f"{form} D={D} A={A} mb={mb} step {st}")
        assert want.clipped.tolist() == [False, True]
        assert (want.gnorm[1] > 0) and (A == 1 or want.gnorm[0] > 0)


# ---------------------------------------------------------------------------------------------------------------------------
# through the learner
# ---------------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("precision,fused", [("bf16", False), ("f32", False)])
def test_learner_optimiser_steps(precision, fused):
    """ff_ppo with one epoch of one minibatch: one optimiser step per update, two updates (the first eager, the second from the
    captured CUDA graph).  The reference takes b1, b2, eps, the learning rates, max_grad_norm and the schedule from the config's
    defaults (optax.adam's 0.9 / 0.999, eps 1e-5 at ff_ppo.py:571-572), not from the kernel's plan: the plumbing is under test
    too, and so are the counters living in the learner state's arena_counts."""
    from stoix_b200 import ops, random as srandom
    from stoix_b200.config import compose
    from stoix_b200.systems.ppo.anakin import ff_ppo
    from stoix_b200.utils import make_env
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    E, T = 256, 16
    cfg = compose("default_ff_ppo", ["env=synthetic/box", f"arch.total_num_envs={E}", f"system.rollout_length={T}", "system.epochs=1",
                                     "system.num_minibatches=1", f"arch.total_timesteps={E * T * 2}", "arch.num_evaluation=1",
                                     f"arch.precision={precision}", "logger.use_console=False"])
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, _ = make_env.make(cfg)
    keys = srandom.split(srandom.PRNGKey(11), 4)
    learn, _, state = ff_ppo.learner_setup(env, (keys[0], keys[2], keys[3]), cfg)
    cfg.arch.num_updates_per_eval = 1
    sa, sc = state.params.actor_params.spec, state.params.critic_params.spec
    _, coff, _ = ops.arena_offsets(sa, sc)
    sysc = cfg.system
    segs = [(0, sa.param_count, float(sysc.actor_lr), float(sysc.max_grad_norm)),
            (coff, sc.param_count, float(sysc.critic_lr), float(sysc.max_grad_norm))]
    h = R.Hyper(b1=0.9, b2=0.999, eps=1e-5, decay=bool(sysc.decay_learning_rates), steps_per_update=1,
                num_updates=int(cfg.arch.num_updates))
    assert h.decay and h.num_updates == 2
    for upd in range(2):
        a = state.params.actor_params
        pre = _snap(a.arena, a.arena_mu, a.arena_nu, a.arena_counts, a.arena_bf16)
        state = learn(state).learner_state
        a = state.params.actor_params
        got = _snap(a.arena, a.arena_mu, a.arena_nu, a.arena_counts, a.arena_bf16, None, learn.built["plan"].gnorm)
        g = learn.built["grads"].cpu().numpy()
        want = R.step(pre["p"], pre["mu"], pre["nu"], pre["counts"], g, segs, h,
                      norm=R.NORM_DOUBLE if precision == "bf16" else R.NORM_LOCAL)
        R.check(got, want, pre, label=f"{precision} fused={fused} update {upd}")
        assert got["counts"].tolist() == [upd + 1] * 4
        assert (learn.built["graph"] is not None) == (upd == 1)
