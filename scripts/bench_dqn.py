"""DQN-family update-step timing: env steps/s and optimiser steps/s of the captured update step of ff_dqn, ff_ddqn, ff_mdqn and
ff_dqn_reg at two shapes, the systems alternated within each of three rounds, min-max over the rounds; plus the kernels of one
eager update: stx_launch_count (the project's launches that go through STX_LAUNCH_OK, which leaves out the SIMT GEMMs of the MLP
forward and backward) and every kernel the profiler records, GEMMs counted apart.  The card name and power limit are read in the same call.

    python scripts/bench_dqn.py [--updates 50] [--rounds 3]

Shapes (all four systems run the same schedule, so that they differ only in the loss):
  "default" = the reference's ff_dqn default: CartPole, 1024 envs, T = 2, 16 epochs of batch 512, silu MLP 2 x 256;
  "wide"    = the synthetic Box, obs 64, A = 8, 1024 envs, T = 2, 16 epochs of batch 4096, same network.
Prints one JSON line per (round, shape, system), then one summary line per (shape, system)."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

SYSTEMS = ("ff_dqn", "ff_ddqn", "ff_mdqn", "ff_dqn_reg")
COMMON = ["arch.total_num_envs=1024", "system.rollout_length=2", "system.epochs=16", "system.total_buffer_size=1000000", "system.warmup_steps=16",
          "logger.use_console=False", "arch.num_evaluation=1"]
SHAPES = {
    "default": ["env=gymnax/cartpole", "system.total_batch_size=512"],
    "wide": ["env=synthetic/box", "env.kwargs.obs_dim=64", "env.kwargs.num_actions=8", "system.total_batch_size=4096"],
}


def _card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=20).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as e:  # the timing stands without it, but says so
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"not read ({type(e).__name__})"}


def _setup(system: str, shape: str, updates: int):
    import importlib

    from stoix_b200 import random as srandom
    from stoix_b200.config import compose
    from stoix_b200.utils import make_env as environments
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    mod = importlib.import_module(f"stoix_b200.systems.q_learning.{system}")
    cfg = compose(f"default_{system}", COMMON + SHAPES[shape] + [f"arch.total_timesteps={1024 * 2 * (updates + 8)}"], config_dir="default/anakin")
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, _ = environments.make(cfg)
    learn, _, state = mod.learner_setup(env, tuple(srandom.split(srandom.PRNGKey(0), 2)), cfg)
    return cfg, learn, state


def _kernels(fn) -> dict:
    """Every kernel fn() launches eagerly, as the profiler records them: all of them, and those named like the SIMT GEMMs of the MLP
    forward / backward (which stx_launch_count does not count: it counts the launches that go through STX_LAUNCH_OK)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset"))]
    short = [n.split("<")[0].split("(")[0].replace("void ", "").strip() for n in names]
    return {"all": len(names), "gemm": sum("gemm" in n.lower() for n in names), "names": {k: short.count(k) for k in sorted(set(short))}}


def run(system: str, shape: str, updates: int) -> dict:
    from stoix_b200 import _lib

    cfg, learn, state = _setup(system, shape, updates)
    lib = _lib.load()
    cfg.arch.num_updates_per_eval = 1
    learn.ensure_built(state)
    torch.cuda.synchronize()
    n0 = lib.stx_launch_count()
    learn.update_step(state)                      # one eager update: the launches the graph captures
    torch.cuda.synchronize()
    launches = lib.stx_launch_count() - n0
    kernels = _kernels(lambda: learn.update_step(state))
    step = _kernels(lambda: learn.update_epoch(state, 0))   # one optimiser step: sample, forwards, loss, backward, clip + Adam, Polyak
    learn.built["eager_done"] = True
    cfg.arch.num_updates_per_eval = 2
    state = learn(state).learner_state            # capture + two replays
    torch.cuda.synchronize()
    cfg.arch.num_updates_per_eval = updates
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    state = learn(state).learner_state
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / updates
    T, E, epochs = int(cfg.system.rollout_length), int(cfg.arch.num_envs), int(cfg.system.epochs)
    return {"shape": shape, "system": system, "num_envs": E, "rollout_length": T, "epochs": epochs, "batch_size": int(cfg.system.batch_size),
            "update_ms": round(ms, 4), "env_steps_per_s": round(T * E / (ms / 1e3)), "opt_steps_per_s": round(epochs / (ms / 1e3)),
            "stx_launches_per_update": int(launches), "kernels_per_update": kernels["all"], "gemm_kernels_per_update": kernels["gemm"],
            "kernels_per_opt_step": step["all"], "gemm_kernels_per_opt_step": step["gemm"],
            "opt_step_kernels": step["names"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="default,wide")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    card = _card()
    seen = {}
    for r in range(a.rounds):
        for shape in a.shapes.split(","):
            for system in SYSTEMS:          # alternate the systems within each round
                res = run(system, shape, a.updates)
                seen.setdefault((shape, system), []).append(res)
                print(json.dumps({"round": r, **res, **card}), flush=True)
                torch.cuda.empty_cache()
    for (shape, system), rs in seen.items():
        sps = [x["env_steps_per_s"] for x in rs]
        ops_ = [x["opt_steps_per_s"] for x in rs]
        print(json.dumps({"summary": True, "shape": shape, "system": system, "env_steps_per_s_min_max": [min(sps), max(sps)],
                          "opt_steps_per_s_min_max": [min(ops_), max(ops_)], "stx_launches_per_update": rs[0]["stx_launches_per_update"],
                          "kernels_per_update": rs[0]["kernels_per_update"], "gemm_kernels_per_update": rs[0]["gemm_kernels_per_update"],
                          "kernels_per_opt_step": rs[0]["kernels_per_opt_step"], "gemm_kernels_per_opt_step": rs[0]["gemm_kernels_per_opt_step"],
                          **card}), flush=True)


if __name__ == "__main__":
    main()
