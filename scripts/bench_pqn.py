"""ff_pqn update-step timing: env steps/s of the captured update step and the phase split (rollout, targets, update) measured
eagerly on the same state, at two shapes, three alternated runs each, with the card name and power limit read in the same call.

    python scripts/bench_pqn.py [--updates 20] [--runs 3]

Shapes: "default" = the reference default (CartPole, 1024 envs, T = 8, 4 epochs x 16 minibatches, silu MLP 2 x 256, LayerNorm on);
"wide" = the synthetic Box at 16384 envs, obs 64, A = 8, same network and schedule.  Prints one JSON line per (shape, run)."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

SHAPES = {
    "default": ["env=gymnax/cartpole", "arch.total_num_envs=1024"],
    "wide": ["env=synthetic/box", "arch.total_num_envs=16384", "env.kwargs.obs_dim=64", "env.kwargs.num_actions=8"],
}


def _card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=20).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as e:  # the timing stands without it, but says so
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"not read ({type(e).__name__})"}


def _setup(shape: str, updates: int):
    from stoix_b200 import random as srandom
    from stoix_b200.config import compose
    from stoix_b200.systems.q_learning import ff_pqn
    from stoix_b200.utils import make_env as environments
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    ov = SHAPES[shape] + ["network.actor_network.pre_torso.use_layer_norm=True", "logger.use_console=False", "arch.num_evaluation=1"]
    E = int(ov[1].split("=")[1])
    ov.append(f"arch.total_timesteps={E * 8 * updates}")
    cfg = compose("default_ff_pqn", ov, config_dir="default/anakin")
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, _ = environments.make(cfg)
    learn, _, state = ff_pqn.learner_setup(env, tuple(srandom.split(srandom.PRNGKey(0), 2)), cfg)
    return cfg, learn, state


def _time(fn, n: int) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def run(shape: str, updates: int) -> dict:
    cfg, learn, state = _setup(shape, updates)
    cfg.arch.num_updates_per_eval = 2
    state = learn(state).learner_state          # eager update + capture + one replay
    torch.cuda.synchronize()
    cfg.arch.num_updates_per_eval = updates
    box = [state]

    def step():
        box[0] = learn(box[0]).learner_state

    ms = _time(step, 1) / updates
    T, E = int(cfg.system.rollout_length), int(cfg.arch.num_envs)
    st = box[0]
    ph = {name: _time(lambda: learn.phases[name](st), 10) for name in ("rollout", "targets")}
    learn.phases["shuffle"](st)
    ph["update"] = _time(lambda: learn.phases["update"](st, shuffled=True), 5)
    return {"shape": shape, "num_envs": E, "rollout_length": T, "epochs": int(cfg.system.epochs), "num_minibatches": int(cfg.system.num_minibatches),
            "update_ms": round(ms, 4), "env_steps_per_s": round(T * E / (ms / 1e3)),
            "eager_phase_ms": {k: round(v, 4) for k, v in ph.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--shapes", default="default,wide")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    card = _card()
    for r in range(a.runs):          # alternate the shapes run by run
        for shape in a.shapes.split(","):
            print(json.dumps({"run": r, **run(shape, a.updates), **card}), flush=True)


if __name__ == "__main__":
    main()
