"""Per-optimiser-step diagnosis of the bf16 (wgmma) update against the bf16-rounding oracle in the LEARNER setting
(real rollout values / GAE targets instead of independent random inputs).  For every minibatch step the gradient is
taken from the kernels' CURRENT parameters on both sides, so trajectory divergence cannot hide (or fake) an error:

    python scripts/diag_bf16_steps.py [E T nmb]

prints, per step, the norm-wise relative error of the actor / critic gradient (per tensor for the worst step)."""
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from oracle import ppo_oracle as O  # noqa: E402
from stoix_b200 import ops, random as srandom  # noqa: E402
from stoix_b200.config import compose  # noqa: E402
from stoix_b200.systems.ppo.anakin import ff_ppo  # noqa: E402
from stoix_b200.utils import make_env  # noqa: E402
from stoix_b200.utils.total_timestep_checker import check_total_timesteps  # noqa: E402


def main():
    E, T, nmb = (int(x) for x in (sys.argv[1:4] if len(sys.argv) >= 4 else (128, 16, 4)))
    perturb = float(sys.argv[4]) if len(sys.argv) > 4 else 0.0
    precision = sys.argv[5] if len(sys.argv) > 5 else "bf16"     # "f32": the CUDA-core path against the plain fp64 oracle
    bf16 = precision == "bf16"
    extra = sys.argv[6:]
    cfg = compose("default_ff_ppo", ["env=synthetic/box", f"arch.total_num_envs={E}", f"system.rollout_length={T}",
                                     f"system.num_minibatches={nmb}", f"arch.total_timesteps={E * T * 2}", "arch.num_evaluation=1",
                                     f"arch.precision={precision}", "logger.use_console=False", "arch.cuda_graph=False"] + extra)
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, _ = make_env.make(cfg)
    keys = srandom.split(srandom.PRNGKey(0), 4)
    learn, _, state = ff_ppo.learner_setup(env, (keys[0], keys[2], keys[3]), cfg)
    a_tree, c_tree = state.params.actor_params, state.params.critic_params
    if perturb > 0:
        with torch.no_grad():
            g = torch.Generator(device="cuda").manual_seed(1)
            a_tree.arena.add_(torch.randn(a_tree.arena.shape, device="cuda", generator=g) * perturb)
            if bf16:
                ops.cast_bf16(a_tree.arena, out=a_tree.arena_bf16)
    learn.ensure_built(state)
    b = learn.built
    learn.phases["rollout"](state)
    learn.phases["gae"](state)
    torch.cuda.synchronize()
    sh = b["shards"][0]
    sa, sc = b["sa"], b["sc"]
    _, coff, total = ops.arena_offsets(sa, sc)
    D = sa.sizes[0]
    B = T * E
    mb = B // nmb
    f64 = lambda t: t.detach().float().cpu().numpy().astype(np.float64)
    obs = f64(sh.obs[:T]).reshape(B, D)
    act = sh.action.cpu().numpy().reshape(B)
    lp_old, v_old = f64(sh.log_prob).reshape(B), f64(sh.value).reshape(B)
    adv_raw, tgt = f64(sh.advantages).reshape(B), f64(sh.targets).reshape(B)
    adv = O.standardize(adv_raw.reshape(T, E)).reshape(B)
    print(f"E={E} T={T} mb={mb}: |v_old| rms {np.sqrt((v_old**2).mean()):.3f}, |tgt| rms {np.sqrt((tgt**2).mean()):.3f}, "
          f"|v_old-tgt| rms {np.sqrt(((v_old-tgt)**2).mean()):.3f}")
    batch = ops.PpoBatch(sh.obs[:T].view(B, D), sh.action.view(B), sh.log_prob.view(B), sh.value.view(B), sh.advantages.view(B),
                         sh.targets.view(B), sh.adv_stats, None)
    grads = torch.zeros(total, device="cuda")
    metrics = torch.zeros(8, device="cuda")
    rel = lambda a, r: float(np.linalg.norm(a - r) / max(np.linalg.norm(r), 1e-30))
    names = ["W0", "b0", "W1", "b1", "W2", "b2"]
    rng = np.random.default_rng(0)
    step = 0
    for ep in range(4):
        perm = rng.permutation(B).astype(np.int32)
        batch.perm = torch.as_tensor(perm, device="cuda")
        for i in range(nmb):
            idx = perm[i * mb:(i + 1) * mb]
            actor = O.MLPParams.from_flat(f64(a_tree.flat), list(sa.sizes))
            critic = O.MLPParams.from_flat(f64(c_tree.flat), list(sc.sizes))
            if bf16:
                actor, critic = actor.astype(np.float32), critic.astype(np.float32)
            ops.ppo_minibatch_grads(sa, sc, b["arena"], batch, i * mb, mb, 0.2, 0.01, 0.5, True, grads, metrics, b["ws"],
                                    ops.STX_PREC_BF16 if bf16 else ops.STX_PREC_F32, 1.0, b["arena_bf16"], overwrite=True)
            torch.cuda.synchronize()
            g = f64(grads)
            lg, a_acts = O.mlp_forward(actor, obs[idx], bf16_operands=bf16)
            _, dlg, _ = O.actor_loss_and_dlogits(lg.astype(np.float64), act[idx], lp_old[idx], adv[idx], 0.2, 0.01)
            ga = O.mlp_backward(actor, a_acts, dlg, bf16_operands=bf16)
            v, c_acts = O.mlp_forward(critic, obs[idx], bf16_operands=bf16)
            _, dv, _ = O.critic_loss_and_dvalue(v[:, 0].astype(np.float64), v_old[idx], tgt[idx], 0.2, 0.5)
            gc = O.mlp_backward(critic, c_acts, dv[:, None], bf16_operands=bf16)
            ra, rc = rel(g[:sa.param_count], ga.flat()), rel(g[coff:coff + sc.param_count], gc.flat())
            per = []
            for label, spec, off, ref in (("a", sa, 0, ga), ("c", sc, coff, gc)):
                for li, (ws_, bs_) in enumerate(spec.layer_slices()):
                    per.append(f"{label}{names[2*li]} {rel(g[off+ws_.start:off+ws_.stop], ref.W[li].ravel()):.1e}")
                    per.append(f"{label}{names[2*li+1]} {rel(g[off+bs_.start:off+bs_.stop], ref.b[li].ravel()):.1e}")
            print(f"step {step:2d} (ep {ep} mb {i}): actor rel {ra:.2e} |g| {np.linalg.norm(ga.flat()):.3e}   critic rel {rc:.2e} "
                  f"|g| {np.linalg.norm(gc.flat()):.3e}   " + " ".join(per))
            ops.clip_adam_step(b["plan"], b["arena"], grads, a_tree.arena_mu, a_tree.arena_nu, params_bf16=b["arena_bf16"])
            if not bf16:   # end-state sensitivity: the same step from the same state on the oracle side
                pass
            step += 1


if __name__ == "__main__":
    main()
