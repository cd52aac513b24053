#!/usr/bin/env python
"""Where the rollout phase of the benchmark step goes (bf16, one H100, bench.py's shape: E=4096, T=128, obs_dim 64).

  python scripts/time_rollout.py [--reps 20] [--chunks 8]

Each item is captured into a CUDA graph and timed with CUDA events around single replays after a warm-up; the median is
reported in ms:
  (a) phase          the rollout phase as the learner runs it
  (b) actor_chunks   only the rollout kernel's chunks (arch.rollout_chunks, default 8), no critic
  (c) critic_two     the two critic evaluations of every chunk (2 x Tc E rows each), at the CTA budget the learner gives them
                     beside the rollout (132 - E/64 CTAs) and on the full GPU
If (b) is close to (a), the actor chain bounds the phase and the critic runs in its shadow.  The card's name and power limit are printed with the numbers.  Prints one JSON line."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--chunks", type=int, default=8)
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
        "arch.num_evaluation=1", "arch.precision=bf16", "logger.use_console=False", f"arch.rollout_chunks={args.chunks}",
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
    chunks = args.chunks
    while T % chunks:
        chunks -= 1
    Tc = T // chunks
    beside = ops.NUM_SMS - E // 64
    res = {"card": card(), "shape": {"E": E, "T": T, "D": D, "chunks": chunks}, "ms": {}}
    ms = res["ms"]

    ms["a_phase"] = time_graph(lambda: learn.phases["rollout"](state), args.reps)

    def actor_chunks():
        for c in range(chunks):
            env.fused_rollout(state.env_state[0], sa, a_tree.flat, a_tree.flat_bf16, sh, T, state.key[0], b["roll_ctr"], t0=c * Tc, steps=Tc)
    ms["b_actor_chunks"] = time_graph(actor_chunks, args.reps)

    def critic_two(budget):
        def run():
            ops.set_forward_cta_budget(budget)
            for c in range(chunks):
                n = Tc * E
                lo = c * Tc
                ops.mlp_forward(sc, c_tree.flat, sh.obs[lo:lo + Tc].view(n, D), precision=ops.STX_PREC_BF16, params_bf16=c_tree.flat_bf16,
                                out=sh.value[lo:lo + Tc].view(n, 1), ws_key="learner-critic")
                ops.mlp_forward(sc, c_tree.flat, sh.next_obs[lo:lo + Tc].view(n, D), precision=ops.STX_PREC_BF16,
                                params_bf16=c_tree.flat_bf16, out=sh.bootstrap_value[lo:lo + Tc].view(n, 1), ws_key="learner-critic")
            ops.set_forward_cta_budget(0)
        return run
    ms["c_critic_two_beside"] = time_graph(critic_two(beside), args.reps)
    ms["c_critic_two_full"] = time_graph(critic_two(0), args.reps)

    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
