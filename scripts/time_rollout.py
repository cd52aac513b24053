#!/usr/bin/env python
"""Where the rollout phase of the benchmark step goes (bf16, one H100, bench.py's shape: E=4096, T=128, obs_dim 64).

  python scripts/time_rollout.py [--reps 20] [--profile DIR]

Each item is captured into a CUDA graph and timed with CUDA events around single replays after a warm-up; the median is
reported in ms:
  (a) phase          the rollout phase as the learner runs it
  (b) trajectory     the synthetic env's whole-trajectory kernel alone (whole GPU), with its achieved bytes/s against the
                     3.35 TB/s data-sheet HBM3 bandwidth
  (c) policy         the rollout's policy alone (stx_tc_rollout_policy) on the CTAs the learner gives it and on every SM
  (d) critic_once    the critic, once per observation plus the ended rows (stx_tc_rollout_values), at the CTA budget the learner
                     gives it beside the policy (132 - POLICY_CTAS) and on the full GPU; critic_two: the two full passes it
                     replaces, at the same budgets
  (e) phase_split_N  the phase with N policy CTAs and the critic on the other SMs (--splits), to tune ff_ppo.POLICY_CTAS
--profile DIR also writes one torch.profiler table of the phase's kernels (a run of its own).  The card's name, power limit and SM clock are printed with
the numbers.  Prints one JSON line."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

E, T, D, A = 4096, 128, 64, 8


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = (x.strip() for x in q.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:  # the numbers stay usable; the card is then unknown
        return {"error": f"{type(e).__name__}: {e}"}


def time_graph(fn, reps):
    import torch

    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def trajectory_bytes(T, E, D):
    """What the trajectory kernel must move: obs rows 1..T and next_obs (bf16), the (T, E) scalars (reward, ep_return f32,
    ep_length i32, done, truncated, is_terminal u8) and the carried return / length read and written."""
    return 2 * T * E * D * 2 + T * E * (4 + 4 + 4 + 1 + 1 + 1) + 2 * E * (4 + 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--splits", default="70,76,82,88", help="policy CTA counts for (e)")
    ap.add_argument("--profile", default=None, help="directory for one torch.profiler table of the rollout phase's kernels")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise RuntimeError("time_rollout.py needs a CUDA device")
    from stoix_b200 import ops, random as srandom
    from stoix_b200.config import compose
    from stoix_b200.systems.ppo.anakin import ff_ppo
    from stoix_b200.utils import make_env
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    cfg = compose("default_ff_ppo", [
        "env=synthetic/box", f"env.kwargs.obs_dim={D}", f"env.kwargs.num_actions={A}", f"arch.total_num_envs={E}",
        f"system.rollout_length={T}", "system.epochs=4", "system.num_minibatches=16", f"arch.total_timesteps={E * T * 20}",
        "arch.num_evaluation=1", "arch.precision=bf16", "logger.use_console=False",
    ])
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, _ = make_env.make(cfg)
    keys = srandom.split(srandom.PRNGKey(cfg.arch.seed), 4)
    learn, _, state = ff_ppo.learner_setup(env, (keys[0], keys[2], keys[3]), cfg)
    cfg.arch.num_updates_per_eval = 1
    for _ in range(3):  # eager update, graph capture, one replay: trajectory buffers and parameters are as the benchmark has them
        state = learn(state).learner_state
    torch.cuda.synchronize()

    b = learn.built
    sh = b["shards"][0]
    sa, sc = b["sa"], b["sc"]
    a_tree, c_tree = state.params.actor_params, state.params.critic_params
    res = {"card": card(), "shape": {"E": E, "T": T, "D": D}, "ms": {}}
    ms = res["ms"]
    env_state = state.env_state[0]
    # the timed items below write the shard's buffers and the env's carried episode state: keep a copy to restore
    saved = {k: env_state[k].clone() for k in ("run_return", "run_length")}

    ms["a_phase"] = time_graph(lambda: learn.phases["rollout"](state), args.reps)
    ms["b_trajectory"] = time_graph(lambda: env.fused_trajectory(env_state, sh, T), args.reps)
    nbytes = trajectory_bytes(T, E, D)
    res["trajectory_bytes"] = nbytes
    res["trajectory_TBps"] = nbytes / (ms["b_trajectory"] * 1e-3) / 1e12
    res["trajectory_share_of_hbm_peak"] = res["trajectory_TBps"] / 3.35
    def policy(ctas):
        return lambda: ops.tc_rollout_policy(sa, a_tree.flat, a_tree.flat_bf16, sh.obs[:T], sh.action, sh.log_prob, state.key[0], 0,
                                             b["roll_ctr"], max_ctas=ctas)
    beside = ops.NUM_SMS - ff_ppo.POLICY_CTAS
    res["policy_ctas"] = ff_ppo.POLICY_CTAS
    ms["c_policy"] = time_graph(policy(ff_ppo.POLICY_CTAS), args.reps)
    ms["c_policy_full"] = time_graph(policy(0), args.reps)

    def critic_once(budget):
        def run():
            ops.set_forward_cta_budget(budget)
            ops.tc_rollout_values(sc, c_tree.flat, c_tree.flat_bf16, sh.obs, sh.next_obs, sh.is_terminal_step, sh.value, sh.bootstrap_value,
                                  ws_key="learner-rollout-values")
            ops.set_forward_cta_budget(0)
        return run

    def critic_two(budget):
        def run():
            ops.set_forward_cta_budget(budget)
            n = T * E
            ops.mlp_forward(sc, c_tree.flat, sh.obs[:T].view(n, D), precision=ops.STX_PREC_BF16, params_bf16=c_tree.flat_bf16,
                            out=sh.value.view(n, 1), ws_key="learner-critic")
            ops.mlp_forward(sc, c_tree.flat, sh.next_obs.view(n, D), precision=ops.STX_PREC_BF16, params_bf16=c_tree.flat_bf16,
                            out=sh.bootstrap_value.view(n, 1), ws_key="learner-critic")
            ops.set_forward_cta_budget(0)
        return run
    ms["d_critic_once_beside"] = time_graph(critic_once(beside), args.reps)
    ms["d_critic_once_full"] = time_graph(critic_once(0), args.reps)
    ms["d_critic_two_beside"] = time_graph(critic_two(beside), args.reps)
    ms["d_critic_two_full"] = time_graph(critic_two(0), args.reps)
    res["ended_rows"] = int(sh.is_terminal_step.sum())
    shipped = ff_ppo.POLICY_CTAS
    for n in (int(x) for x in args.splits.split(",") if x):
        ff_ppo.POLICY_CTAS = n
        ms[f"e_phase_split_{n}"] = time_graph(lambda: learn.phases["rollout"](state), args.reps)
    ff_ppo.POLICY_CTAS = shipped

    if args.profile:
        from torch.profiler import ProfilerActivity, profile

        os.makedirs(args.profile, exist_ok=True)
        learn.phases["rollout"](state)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            learn.phases["rollout"](state)
            torch.cuda.synchronize()
        table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=20)
        with open(os.path.join(args.profile, "rollout_phase_kernels.txt"), "w") as f:
            f.write(table)
        print(table, flush=True)
    for k, v in saved.items():
        env_state[k].copy_(v)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
