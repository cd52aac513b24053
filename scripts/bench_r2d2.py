"""rec_r2d2 on one GPU, with rec_ppo at the same env count alternated in the same run: env-steps/s, ms per captured update, ms per
eager epoch, kernel launches per update, and the share of the update spent in the recurrence.  Reads the GPU name and power limit
in the same run.

  python scripts/bench_r2d2.py [--updates 10] [--rounds 2]

Workloads: rec_r2d2 at the reference default (1024 envs, GRU 256, 32 sequences of 80 rows), a wider batch (4096 envs, 128 sequences),
and rec_ppo at each env count.  At H = 256 W_h is 768 KB, more than the GRU's cluster and persistent forms take, so every step of
the recurrence runs as one SIMT GEMM (h @ W_h) and one gate kernel, and the backward adds a DX GEMM per step and one d W_h GEMM.
Those GEMMs are the same kernels the MLPs run, so kernel names cannot split R2D2's time.  Instead the script captures the GRU calls of
one update alone -- the rollout's T one-step forwards and, per epoch, the target's S-row forward, the online burn-in, the learn-window
forward and its backward, on the learner's own buffers and shapes -- into a CUDA graph and times its replays: `gru_ms_per_update`,
and its ratio to the captured update, `gru_share`.  rec_ppo at H = 128 runs the persistent / cluster gru_* kernels, so its share is
taken from kernel names in a profile of one captured update (its d W_h GEMM counts as an MLP GEMM there)."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

WORKLOADS = {
    "rec_r2d2 default": ("q_learning.rec_r2d2", "default_rec_r2d2", []),
    "rec_ppo 1024 envs": ("ppo.anakin.rec_ppo", "default_rec_ppo", ["arch.total_num_envs=1024"]),
    "rec_r2d2 wide": ("q_learning.rec_r2d2", "default_rec_r2d2", ["arch.total_num_envs=4096", "system.total_batch_size=128",
                                                                  "system.total_buffer_size=400000"]),
    "rec_ppo 4096 envs": ("ppo.anakin.rec_ppo", "default_rec_ppo", ["arch.total_num_envs=4096"]),
}


def _learner(module, config, overrides):
    from stoix_b200 import random as srandom
    from stoix_b200.config import compose
    from stoix_b200.utils import make_env
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps
    cfg = compose(config, ["arch.total_timesteps=~", "arch.num_updates=100", "logger.use_console=False", *overrides], config_dir="default/anakin")
    cfg.num_devices = 1
    cfg = check_total_timesteps(cfg, quiet=True)
    env, _ = make_env.make(cfg)
    mod = importlib.import_module(f"stoix_b200.systems.{module}")
    n_keys = 2 if "r2d2" in module else 3
    keys = srandom.split(srandom.PRNGKey(0), num=n_keys)
    learn, _, state = mod.learner_setup(env, tuple(keys), cfg)
    return cfg, learn, state


def _time_graph(fn, reps: int) -> float:
    """ms per replay of a CUDA graph of fn()."""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        g.replay()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


def _r2d2_gru_ms(cfg, learn, state) -> float:
    """ms of the GRU calls of one rec_r2d2 update (U shards), timed alone as a graph on the learner's buffers."""
    from stoix_b200 import ops
    b, sysc = learn.built, cfg.system
    lay, w = b["layout"], b["work"]
    if lay.cell_type != "gru":
        raise ValueError("the GRU timing covers the gru cell")
    T, E, bi = int(sysc.rollout_length), int(cfg.arch.num_envs), int(sysc.burn_in_length)
    _, w_h, b_hn, _ = lay.blocks(state.params.online.flat)
    _, g_wh, g_bhn, _ = lay.blocks(b["grads"].clone())
    z = lambda *sh, dt=torch.float32: torch.zeros(*sh, dtype=dt, device=b["dev"])
    gi1, h1, reset1, ws1, h0 = z(1, E, 3 * lay.H), z(1, E, lay.H), z(1, E, dt=torch.uint8), ops.gru_workspace(1, E, lay.H, b["dev"]), z(E, lay.H)
    bt = b["batches"][0]

    def rollout():
        for _ in range(T):
            ops.gru_sequence_forward(gi1, reset1, h0, w_h, b_hn, ws1, out=h1)

    def epoch():
        ops.gru_sequence_forward(w.gi_all, bt.reset, bt.carry0, w_h, b_hn, w.ws_all, out=w.h_all)
        if bi > 0:
            ops.gru_sequence_forward(w.gi_burn, bt.reset[:bi], bt.carry0, w_h, b_hn, w.ws_burn, out=w.h_burn)
        ops.gru_sequence_forward(w.gi, bt.reset[bi:], w.carry_on, w_h, b_hn, w.ws_seq, out=w.h_seq)
        ops.gru_sequence_backward(w.d_h, bt.reset[bi:], w_h, w.ws_seq, w.d_gi, d_w_h=g_wh, d_b_hn=g_bhn)

    U = int(cfg.arch.update_batch_size)
    return U * (_time_graph(rollout, 20) + int(sysc.epochs) * _time_graph(epoch, 20))


def _name_share(learn, state, buffers, items):
    """Kernel-name split of one captured update: gru_* / lstm_* kernels against all kernels, and the kernel count."""
    from stoix_b200.systems import anakin
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        anakin.update_once(learn.built, True, learn.update_step, state, buffers, items)
        torch.cuda.synchronize()
    rec = tot = 0.0
    n = 0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", 0.0)
        if t <= 0:
            continue
        n += ev.count
        tot += t
        if "gru" in ev.key.lower() or "lstm" in ev.key.lower():
            rec += t
    return rec / max(tot, 1e-9), n


def _measure(label, module, config, over, updates):
    from stoix_b200.systems import anakin
    cfg, learn, state = _learner(module, config, over)
    learn.ensure_built(state)
    b = learn.built
    items = int(cfg.system.rollout_length) * int(cfg.arch.num_envs)
    buffers = getattr(state, "buffer_state", ())
    step = lambda: anakin.update_once(b, True, learn.update_step, state, buffers, items)
    for _ in range(3):   # eager, capture, one replay
        step()
    torch.cuda.synchronize()
    t0 = time.time()
    for _ in range(updates):
        step()
    torch.cuda.synchronize()
    ms = (time.time() - t0) * 1e3 / updates
    out = {"workload": label, "env_steps_per_s": items / (ms / 1e3), "ms_per_update": ms}
    if hasattr(learn, "update_epoch"):
        learn.update_epoch(state, 0)
        torch.cuda.synchronize()
        t0 = time.time()
        for _ in range(10):
            learn.update_epoch(state, 0)
        torch.cuda.synchronize()
        out["ms_per_eager_epoch"] = (time.time() - t0) * 1e3 / 10
    share, n = _name_share(learn, state, buffers, items)
    out["kernels_per_update"] = n
    if "r2d2" in module:
        out["gru_ms_per_update"] = _r2d2_gru_ms(cfg, learn, state)
        out["gru_share"] = out["gru_ms_per_update"] / ms
    else:
        out["gru_share_by_kernel_name"] = share
    del learn, state, b
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    for rnd in range(args.rounds):
        for label, (module, config, over) in WORKLOADS.items():
            out = _measure(label, module, config, over, args.updates)
            out["round"] = rnd
            print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
