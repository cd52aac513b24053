"""bf16 tensor-core path (wgmma): fused MLP forward vs the oracle with bf16-rounded GEMM operands
(weights, inputs and hidden activations rounded to bf16, fp32 accumulate -- oracle.mlp_forward(
bf16_operands=True)).  Tolerance: the only differences left are fp32 accumulation order and rare
1-ulp bf16 rounding flips of a hidden activation: rtol 2e-3 / atol 2e-3 on outputs; vs the pure fp32
reference the bf16 path is reported at rtol 2e-2 (BASELINE.md section 4)."""
import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O

pytestmark = pytest.mark.gpu


def _t(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype, device="cuda:0")


def _net(rng, D, A, head_scale):
    p = O.init_mlp(rng, [D, 256, 256, A], head_scale)
    for i in range(3):
        p.b[i] = rng.standard_normal(p.b[i].shape) * 0.1
    p.W[-1] = rng.standard_normal(p.W[-1].shape) * 0.3
    return p


@pytest.mark.parametrize("M,D,A", [(128, 64, 8), (4096, 64, 8), (300, 64, 1), (128 * 150 + 5, 64, 8), (256, 32, 16), (64, 16, 2)])
def test_tc_forward_matches_bf16_oracle(M, D, A):
    from stoix_b200 import ops

    rng = np.random.default_rng(M + A)
    net = _net(rng, D, A, 1.0)
    x = rng.standard_normal((M, D)).astype(np.float32)
    spec = ops.MlpSpec((D, 256, 256, A))
    params = _t(net.flat())
    shadow = ops.cast_bf16(params)
    xb = _t(x).to(torch.bfloat16)
    out, h1, h2 = ops.tc_debug_forward(spec, params, shadow, xb)
    torch.cuda.synchronize()
    ref, acts = O.mlp_forward(net.astype(np.float32), x, bf16_operands=True)
    e1 = np.abs(h1.cpu().numpy() - acts[1]).max()
    e2 = np.abs(h2.cpu().numpy() - acts[2]).max()
    e3 = np.abs(out.cpu().numpy() - ref).max()
    print(f"M={M} D={D} A={A}: max|h1 err|={e1:.3e} max|h2 err|={e2:.3e} max|out err|={e3:.3e}")
    np.testing.assert_allclose(h1.cpu().numpy(), acts[1], rtol=1e-2, atol=1e-2)   # a bf16 ulp at |h|~2 is 1.6e-2 * 0.5
    np.testing.assert_allclose(h2.cpu().numpy(), acts[2], rtol=1e-2, atol=2e-2)
    # a hidden activation that sits on a bf16 rounding boundary may round the other way (fp32 accumulation
    # order differs from the oracle's): such 1-ulp flips move an output by ~|W2|*ulp; they are rare.
    err = np.abs(out.cpu().numpy() - ref)
    tight = err <= 2e-3 * np.abs(ref) + 5e-3
    assert tight.mean() > 0.999, f"only {tight.mean():.5f} of the outputs within rtol 2e-3 / atol 5e-3"
    assert err.max() < 3e-2
    # the public entry point (no debug outputs) gives the same numbers
    out2 = ops.mlp_forward(spec, params, xb, precision=ops.STX_PREC_BF16, params_bf16=shadow)
    assert torch.equal(out, out2)
    # and stays within the stated bf16-vs-fp32 band of the pure fp32 reference
    ref32, _ = O.mlp_forward(net, x.astype(np.float64))
    assert np.abs(out.cpu().numpy() - ref32).max() < 2e-2 * max(1.0, np.abs(ref32).max())


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)


_MINIBATCH_CASES = [
    (2048, 512, 1024, 64, 8, True),
    (512, 128, 256, 32, 5, False),
    (16384, 0, 16384, 64, 8, True),   # > 1 tile per CTA, every split-K CTA busy
    (384, 0, 128, 64, 16, True),      # a single tile: most CTAs idle
    # BASELINE config 2 (the shape bench.py runs): B = T*E = 524 288 rows, minibatch 32 768 = 256 tiles per
    # network (3.46 tiles per K3a CTA, every split-K CTA with >= 7 chunks), shuffle indices up to 2^19
    (524288, 5 * 32768, 32768, 64, 8, True),
]


@pytest.mark.parametrize("B,mb_off,mb,D,A,use_perm,saturated",
                         [pytest.param(*c, False, id="-".join(map(str, c))) for c in _MINIBATCH_CASES]
                         # K3a's actor head (__expf / __logf) at saturation: the final bias puts the other actions 30 to 110 below
                         # action 0, so the taken action's log-probability reaches ~ -110 and most probabilities underflow
                         + [pytest.param(2048, 512, 1024, 64, 8, True, True, id="saturated-2048-512-1024-64-8-True")])
def test_tc_ppo_minibatch_grads_vs_bf16_oracle(B, mb_off, mb, D, A, use_perm, saturated):
    """K3 on tensor cores vs the oracle with the same bf16 operand rounding (weights, activations, dY);
    what is left is fp32 summation order and rare relu/rounding flips -> norm-wise 5e-3 per tensor."""
    from stoix_b200 import ops

    rng = np.random.default_rng(B + mb + A)
    actor, critic = _net(rng, D, A, 0.3), _net(rng, D, 1, 1.0)
    if saturated:
        actor.b[-1] = -np.concatenate([[0.0], np.linspace(30.0, 110.0, A - 1)])
    sa, sc = ops.MlpSpec((D, 256, 256, A)), ops.MlpSpec((D, 256, 256, 1))
    _, coff, total = ops.arena_offsets(sa, sc)
    flat = np.zeros(total, np.float32)
    flat[: sa.param_count] = actor.flat()
    flat[coff : coff + sc.param_count] = critic.flat()
    arena = _t(flat)
    shadow = ops.cast_bf16(arena)
    obs = rng.standard_normal((B, D)).astype(np.float32)
    obs_b = _t(obs).to(torch.bfloat16)
    obs_r = obs_b.float().cpu().numpy().astype(np.float64)  # what the kernels actually see
    act = rng.integers(0, A, B).astype(np.int32)
    a32, c32 = actor.astype(np.float32), critic.astype(np.float32)
    logits, _ = O.mlp_forward(a32, obs_r, bf16_operands=True)
    lp_old = (O.categorical_log_prob(logits, act) + rng.standard_normal(B) * 0.3).astype(np.float32)
    v_old = rng.standard_normal(B).astype(np.float32)
    adv = (rng.standard_normal(B) * 2 + 0.3).astype(np.float32)
    tgt = rng.standard_normal(B).astype(np.float32)
    mean = adv.astype(np.float64).mean()
    rstd = 1.0 / np.sqrt((adv.astype(np.float64) ** 2).mean() - mean * mean + 1e-5)
    perm = rng.permutation(B).astype(np.int32) if use_perm else None
    idx = perm[mb_off : mb_off + mb] if use_perm else np.arange(mb_off, mb_off + mb)
    adv_n = (adv.astype(np.float64) - mean) * rstd
    lg, a_acts = O.mlp_forward(a32, obs_r[idx], bf16_operands=True)
    _, dlg, a_info = O.actor_loss_and_dlogits(lg.astype(np.float64), act[idx], lp_old[idx].astype(np.float64), adv_n[idx], 0.2, 0.01)
    ga = O.mlp_backward(a32, a_acts, dlg, bf16_operands=True)
    v, c_acts = O.mlp_forward(c32, obs_r[idx], bf16_operands=True)
    _, dv, c_info = O.critic_loss_and_dvalue(v[:, 0].astype(np.float64), v_old[idx].astype(np.float64), tgt[idx].astype(np.float64), 0.2, 0.5)
    gc = O.mlp_backward(c32, c_acts, dv[:, None], bf16_operands=True)

    batch = ops.PpoBatch(obs_b, _t(act, torch.int32), _t(lp_old), _t(v_old), _t(adv), _t(tgt),
                         adv_stats=_t(np.array([mean, rstd])), perm=_t(perm, torch.int32) if use_perm else None)
    grads = torch.zeros(total, device="cuda:0")
    metrics = torch.zeros(8, device="cuda:0")
    ws = ops.ppo_workspace(sa, sc, mb, ops.STX_PREC_BF16, "cuda:0")
    ops.ppo_minibatch_grads(sa, sc, arena, batch, mb_off, mb, 0.2, 0.01, 0.5, True, grads, metrics, ws,
                            precision=ops.STX_PREC_BF16, param_arena_bf16=shadow)
    torch.cuda.synchronize()
    g = grads.cpu().numpy().astype(np.float64)
    names = ["W0", "b0", "W1", "b1", "W2", "b2"]
    for label, spec, off, ref in (("actor", sa, 0, ga), ("critic", sc, coff, gc)):
        for i, (ws_, bs_) in enumerate(spec.layer_slices()):
            for nm, sl, r in ((names[2 * i], ws_, ref.W[i].ravel()), (names[2 * i + 1], bs_, ref.b[i].ravel())):
                got = g[off + sl.start : off + sl.stop]
                e = _rel(got, r)
                print(f"{label} d{nm}: rel err {e:.2e} (|ref|={np.linalg.norm(r):.3e})")
                assert e < 5e-3, f"{label} d{nm}: norm-wise relative error {e:.3e}"
    mt = metrics.cpu().numpy()
    np.testing.assert_allclose(mt[:3], [a_info["actor_loss"], a_info["entropy"], c_info["value_loss"]], rtol=2e-3, atol=1e-4)
    np.testing.assert_allclose(mt[3:6], [adv_n[idx].mean(), v[:, 0].mean(), tgt[idx].astype(np.float64).mean()], rtol=2e-3, atol=2e-4)
    # accumulation + determinism: a second call doubles the gradient exactly
    ops.ppo_minibatch_grads(sa, sc, arena, batch, mb_off, mb, 0.2, 0.01, 0.5, True, grads, metrics, ws,
                            precision=ops.STX_PREC_BF16, param_arena_bf16=shadow)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(grads.cpu().numpy(), (2 * g).astype(np.float32))
    # bf16 path vs the PURE fp32/fp64 oracle (no operand rounding anywhere): the stated tolerance of the tensor-core
    # path against the reference arithmetic.  bf16 operands carry 2^-9 relative rounding, and the surrogate's clip
    # indicator is discontinuous (a sample whose ratio sits at 1 +- eps flips in or out of the sum), so the bound is
    # norm-wise per network: relative error <= 0.15 (cosine >= 0.99).  Measured: actor 0.04-0.11 (0.063 at the BASELINE
    # shape), critic 0.003-0.014.
    obs64 = obs.astype(np.float64)[idx]
    lg32, acts32 = O.mlp_forward(actor, obs64)
    _, dlg32, _ = O.actor_loss_and_dlogits(lg32, act[idx], lp_old[idx].astype(np.float64), adv_n[idx], 0.2, 0.01)
    ga32 = O.mlp_backward(actor, acts32, dlg32).flat()
    v32, cacts32 = O.mlp_forward(critic, obs64)
    _, dv32, _ = O.critic_loss_and_dvalue(v32[:, 0], v_old[idx].astype(np.float64), tgt[idx].astype(np.float64), 0.2, 0.5)
    gc32 = O.mlp_backward(critic, cacts32, dv32[:, None]).flat()
    for label, got, ref32 in (("actor", g[: sa.param_count], ga32), ("critic", g[coff : coff + sc.param_count], gc32)):
        cos = float(got @ ref32 / (np.linalg.norm(got) * np.linalg.norm(ref32)))
        rel = _rel(got, ref32)
        print(f"bf16-path {label} gradient vs pure fp32 oracle: norm-wise rel {rel:.4f}, cosine {cos:.5f}")
        assert rel < 0.15 and cos > 0.99, f"{label}: bf16 path vs fp32 oracle rel {rel:.4f} cos {cos:.5f}"


@pytest.mark.parametrize("E,T,nmb", [
    (64, 8, 2),
    (4096, 128, 16),   # BASELINE config 2: the exact update step bench.py times (mb = 32 768, 64 optimiser steps)
])
def test_learner_bf16_update_tracks_bf16_oracle(E, T, nmb):
    """One whole Anakin update step with arch.precision=bf16 (tensor-core rollout, batched critic, K3 on tensor
    cores, bf16 weight shadows refreshed by the fused Adam) vs the oracle run with the same bf16 operand
    rounding, actions and permutations injected.

    Bounds.  This is the integration check of the whole graph-captured step: GAE targets tight (1e-4), loss metrics
    2e-2, optimiser counters exact, bf16 shadow == rounded master.  The END STATE of 4 x nmb chained Adam steps is
    compared loosely (first moments 0.3, second moments 0.1, parameter change 0.15 norm-wise; measured at the BASELINE
    shape: mu 0.06 / 0.18 (actor / critic), nu 0.011 / 0.042, parameter change 0.033 / 0.037): both sides' per-step gradients agree to ~1e-4 (scripts/diag_bf16_steps.py, and the per-step test below
    holds them to 5e-3), but Adam turns every entry's gradient into a step of ~lr whatever its size, so entries whose
    (tiny) gradient differs in the last bits move apart and the two parameter trajectories drift from each other."""
    from stoix_b200 import ops, random as srandom
    from stoix_b200.config import compose
    from stoix_b200.systems.ppo.anakin import ff_ppo
    from stoix_b200.utils import make_env
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    cfg = compose("default_ff_ppo", ["env=synthetic/box", f"arch.total_num_envs={E}", f"system.rollout_length={T}",
                                     f"system.num_minibatches={nmb}", f"arch.total_timesteps={E * T * 2}", "arch.num_evaluation=1",
                                     "arch.precision=bf16", "logger.use_console=False", "env.kwargs.p_term=0.05", "env.kwargs.p_trunc=0.05"])
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, _ = make_env.make(cfg)
    keys = srandom.split(srandom.PRNGKey(3), 4)
    learn, _, state = ff_ppo.learner_setup(env, (keys[0], keys[2], keys[3]), cfg)
    with torch.no_grad():
        g = torch.Generator(device="cuda").manual_seed(1)
        arena = state.params.actor_params.arena
        arena.add_(torch.randn(arena.shape, device="cuda", generator=g) * 0.05)
        ops.cast_bf16(arena, out=state.params.actor_params.arena_bf16)
    f64 = lambda t: t.detach().float().cpu().numpy().astype(np.float64)
    tree = lambda tr: O.MLPParams.from_flat(f64(tr.flat), list(tr.spec.sizes))
    actor, critic = tree(state.params.actor_params), tree(state.params.critic_params)
    p0a, p0c = actor.flat().copy(), critic.flat().copy()
    cfg.arch.num_updates_per_eval = 1
    out = learn(state)
    torch.cuda.synchronize()
    sh = learn.built["shards"][0]
    traj = O.Trajectory(obs=f64(sh.obs[:T]), action=sh.action.cpu().numpy(), reward=f64(sh.reward),
                        done=sh.done.cpu().numpy().astype(bool), truncated=sh.truncated.cpu().numpy().astype(bool), next_obs=f64(sh.next_obs))
    O.evaluate_rollout(actor, critic, traj, bf16=True)
    np.testing.assert_allclose(f64(sh.value), traj.value, rtol=2e-3, atol=2e-2)
    np.testing.assert_allclose(f64(sh.log_prob), traj.log_prob, rtol=2e-3, atol=2e-2)
    np.testing.assert_allclose(f64(sh.bootstrap_value), traj.bootstrap_value, rtol=2e-3, atol=2e-2)
    perms = np.stack([ops.make_permutation(T * E, state.key[1], ep, device="cuda").cpu().numpy() for ep in range(4)])
    for ep in range(4):  # the learner consumed exactly these shuffles, and each is a bijection of the flat index
        assert np.array_equal(perms[ep], sh.perms[ep].cpu().numpy())
        assert np.array_equal(np.sort(perms[ep]), np.arange(T * E))
    h = O.PPOHyper(num_minibatches=nmb, num_updates=int(cfg.arch.num_updates))
    # feed the oracle the kernel's own value / log_prob so both run the update from identical inputs
    traj.value, traj.bootstrap_value, traj.log_prob = f64(sh.value), f64(sh.bootstrap_value), f64(sh.log_prob)
    n_a, n_c = actor.flat().size, critic.flat().size
    a_st, c_st = O.AdamState(np.zeros(n_a), np.zeros(n_a)), O.AdamState(np.zeros(n_c), np.zeros(n_c))
    a2, c2, metrics, adv, tgt = O.ppo_update(actor, critic, a_st, c_st, traj, perms, h, bf16=True)
    np.testing.assert_allclose(f64(sh.targets), tgt, rtol=1e-4, atol=2e-5)
    a_tree = out.learner_state.params.actor_params
    _, coff, _ = ops.arena_offsets(a_tree.spec, out.learner_state.params.critic_params.spec)
    mu, nu = f64(a_tree.arena_mu), f64(a_tree.arena_nu)
    errs = {
        "actor mu": _rel(mu[:n_a], a_st.mu), "actor nu": _rel(nu[:n_a], a_st.nu),
        "critic mu": _rel(mu[coff:coff + n_c], c_st.mu), "critic nu": _rel(nu[coff:coff + n_c], c_st.nu),
    }
    da, dc = f64(a_tree.flat) - p0a, f64(out.learner_state.params.critic_params.flat) - p0c
    ra, rc = _rel(da, a2.flat() - p0a), _rel(dc, c2.flat() - p0c)
    print(f"E={E} T={T}: after {4 * nmb} Adam steps, bf16 kernels vs bf16 oracle: " + ", ".join(f"{k} rel {v:.2e}" for k, v in errs.items())
          + f"; parameter change actor rel {ra:.3e}, critic rel {rc:.3e}")
    # end state of a whole update: trajectory divergence under Adam's per-entry normalisation dominates (see the docstring;
    # the per-step gradients are held to 5e-3 by test_learner_bf16_per_step_gradients_match_oracle)
    for k, v in errs.items():
        assert v < (0.3 if k.endswith("mu") else 0.1), f"{k}: norm-wise relative error {v:.3e} of the Adam moment after {4 * nmb} steps"
    assert ra < 0.15 and rc < 0.15, (ra, rc)
    assert a_tree.arena_counts.cpu().tolist() == [4 * nmb] * 4
    shadow = a_tree.arena_bf16
    assert torch.equal(shadow, a_tree.arena.to(torch.bfloat16))
    for name in ("actor_loss", "entropy", "value_loss"):
        np.testing.assert_allclose(f64(out.train_metrics[name][0]), metrics[name], rtol=2e-2, atol=2e-3)


def _per_step_gradient_errors(E, T, nmb, check_steps, perturb=0.05):
    """Runs the bf16 learner's rollout + GAE, then the update's epochs x minibatches by hand through the C ABI
    (stx_ppo_minibatch_grads + stx_clip_adam_step, the calls the learner makes); at every step in `check_steps` the
    oracle evaluates the gradient FROM THE KERNELS' CURRENT PARAMETERS with the same bf16 operand rounding, so each
    optimiser step is compared on its own (no trajectory drift).  Returns {step: (actor rel err, critic rel err)}."""
    from stoix_b200 import ops, random as srandom
    from stoix_b200.config import compose
    from stoix_b200.systems.ppo.anakin import ff_ppo
    from stoix_b200.utils import make_env
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    cfg = compose("default_ff_ppo", ["env=synthetic/box", f"arch.total_num_envs={E}", f"system.rollout_length={T}",
                                     f"system.num_minibatches={nmb}", f"arch.total_timesteps={E * T * 2}", "arch.num_evaluation=1",
                                     "arch.precision=bf16", "logger.use_console=False", "arch.cuda_graph=False"])
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, _ = make_env.make(cfg)
    keys = srandom.split(srandom.PRNGKey(0), 4)
    learn, _, state = ff_ppo.learner_setup(env, (keys[0], keys[2], keys[3]), cfg)
    a_tree, c_tree = state.params.actor_params, state.params.critic_params
    with torch.no_grad():
        g = torch.Generator(device="cuda").manual_seed(1)
        a_tree.arena.add_(torch.randn(a_tree.arena.shape, device="cuda", generator=g) * perturb)
        ops.cast_bf16(a_tree.arena, out=a_tree.arena_bf16)
    learn.ensure_built(state)
    b = learn.built
    learn.phases["rollout"](state)
    learn.phases["gae"](state)
    torch.cuda.synchronize()
    sh, sa, sc = b["shards"][0], b["sa"], b["sc"]
    _, coff, total = ops.arena_offsets(sa, sc)
    D, B = sa.sizes[0], T * E
    mb = B // nmb
    f64 = lambda t: t.detach().float().cpu().numpy().astype(np.float64)
    obs, act = f64(sh.obs[:T]).reshape(B, D), sh.action.cpu().numpy().reshape(B)
    lp_old, v_old, tgt = f64(sh.log_prob).reshape(B), f64(sh.value).reshape(B), f64(sh.targets).reshape(B)
    adv = O.standardize(f64(sh.advantages)).reshape(B)
    batch = ops.PpoBatch(sh.obs[:T].view(B, D), sh.action.view(B), sh.log_prob.view(B), sh.value.view(B), sh.advantages.view(B),
                         sh.targets.view(B), sh.adv_stats, None)
    grads, metrics = torch.zeros(total, device="cuda"), torch.zeros(8, device="cuda")
    rng = np.random.default_rng(0)
    out, step = {}, 0
    for ep in range(4):
        perm = rng.permutation(B).astype(np.int32)
        batch.perm = torch.as_tensor(perm, device="cuda")
        for i in range(nmb):
            if step in check_steps:
                actor = O.MLPParams.from_flat(f64(a_tree.flat), list(sa.sizes)).astype(np.float32)
                critic = O.MLPParams.from_flat(f64(c_tree.flat), list(sc.sizes)).astype(np.float32)
            ops.ppo_minibatch_grads(sa, sc, b["arena"], batch, i * mb, mb, 0.2, 0.01, 0.5, True, grads, metrics, b["ws"],
                                    ops.STX_PREC_BF16, 1.0, b["arena_bf16"], overwrite=True)
            if step in check_steps:
                idx = perm[i * mb:(i + 1) * mb]
                gk = f64(grads)
                lg, a_acts = O.mlp_forward(actor, obs[idx], bf16_operands=True)
                _, dlg, _ = O.actor_loss_and_dlogits(lg.astype(np.float64), act[idx], lp_old[idx], adv[idx], 0.2, 0.01)
                ga = O.mlp_backward(actor, a_acts, dlg, bf16_operands=True).flat()
                v, c_acts = O.mlp_forward(critic, obs[idx], bf16_operands=True)
                _, dv, _ = O.critic_loss_and_dvalue(v[:, 0].astype(np.float64), v_old[idx], tgt[idx], 0.2, 0.5)
                gc = O.mlp_backward(critic, c_acts, dv[:, None], bf16_operands=True).flat()
                out[step] = (_rel(gk[:sa.param_count], ga), _rel(gk[coff:coff + sc.param_count], gc))
            ops.clip_adam_step(b["plan"], b["arena"], grads, a_tree.arena_mu, a_tree.arena_nu, params_bf16=b["arena_bf16"])
            step += 1
    torch.cuda.synchronize()
    assert a_tree.arena_counts.cpu().tolist() == [4 * nmb] * 4
    return out


@pytest.mark.parametrize("E,T,nmb,check_steps", [
    (128, 16, 4, tuple(range(16))),
    (4096, 128, 16, (0, 1, 15, 16, 31, 47, 63)),   # BASELINE config 2; the oracle costs ~1 s per checked step
])
def test_learner_bf16_per_step_gradients_match_oracle(E, T, nmb, check_steps):
    """Every checked optimiser step of a real update (real rollout values, GAE targets, standardised advantages, the
    parameters Adam has produced so far): gradient of both losses vs the bf16-rounding oracle, norm-wise 5e-3 per
    network (measured ~1e-4; the layer-0 bias gradient alone sits at ~1.5e-3: it is summed from bf16-rounded dh1)."""
    errs = _per_step_gradient_errors(E, T, nmb, set(check_steps))
    for st in sorted(errs):
        print(f"E={E} T={T} step {st:2d}: actor rel {errs[st][0]:.2e}  critic rel {errs[st][1]:.2e}")
    assert sorted(errs) == sorted(check_steps)
    for st, (ra, rc) in errs.items():
        assert ra < 5e-3 and rc < 5e-3, f"step {st}: actor {ra:.3e} critic {rc:.3e}"


def test_fused_rollout_is_bit_identical_to_per_step_path():
    """stx_tc_rollout_synth (one persistent launch for the T-step scan) must reproduce the per-step path
    (forward kernel + stx_categorical + stx_synth_env_step per step) exactly: same Philox streams, same GEMMs."""
    _fused_vs_per_step_rollout(256, 12, 64, 8, 2)


@pytest.mark.parametrize("E,T,D,A,nmb", [
    (128, 13, 8, 16, 1),    # T prime: the rollout runs in one chunk; D = 8 and a 16-column head
    (8704, 4, 24, 9, 2),    # 136 rollout CTAs (> 132 SMs); the critic's forward CTA budget 132 - 136 is negative
])
def test_fused_rollout_is_bit_identical_at_edge_shapes(E, T, D, A, nmb):
    """The same comparison at shapes where the rollout's chunking, tile count or head width differ from the default."""
    _fused_vs_per_step_rollout(E, T, D, A, nmb)


def _fused_vs_per_step_rollout(E, T, D, A, nmb):
    """Two update steps with the fused rollout and two with the per-step path: every trajectory field and the updated
    actor arena must be bit-identical."""
    from stoix_b200 import random as srandom
    from stoix_b200.config import compose
    from stoix_b200.systems.ppo.anakin import ff_ppo
    from stoix_b200.utils import make_env
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    def run(fused):
        cfg = compose("default_ff_ppo", ["env=synthetic/box", f"arch.total_num_envs={E}", f"system.rollout_length={T}",
                                         f"system.num_minibatches={nmb}", f"arch.total_timesteps={E * T * 2}", "arch.num_evaluation=1",
                                         "arch.precision=bf16", f"arch.fused_rollout={fused}", "logger.use_console=False",
                                         "env.kwargs.p_term=0.05", "env.kwargs.p_trunc=0.05", f"env.kwargs.obs_dim={D}",
                                         f"env.kwargs.num_actions={A}"])
        cfg.num_devices, cfg.rank = 1, 0
        cfg = check_total_timesteps(cfg, quiet=True)
        env, _ = make_env.make(cfg)
        keys = srandom.split(srandom.PRNGKey(5), 4)
        learn, _, state = ff_ppo.learner_setup(env, (keys[0], keys[2], keys[3]), cfg)
        cfg.arch.num_updates_per_eval = 1
        outs = []
        for _ in range(2):
            out = learn(state)
            state = out.learner_state
            torch.cuda.synchronize()
            sh = learn.built["shards"][0]
            outs.append({k: getattr(sh, k).clone() for k in ("obs", "next_obs", "action", "log_prob", "reward", "done", "truncated",
                                                             "episode_return", "episode_length", "is_terminal_step", "value", "advantages")})
        return outs, state.params.actor_params.arena.clone()

    a, pa = run(True)
    b, pb = run(False)
    for upd in range(2):
        for k in a[upd]:
            assert torch.equal(a[upd][k], b[upd][k]), f"update {upd}: trajectory field {k} differs between fused and per-step rollout"
    assert torch.equal(pa, pb)
