"""The PPO variants next to their clip counterparts at the same shape (fp32 SIMT kernels): env steps/s and ms per captured update
step, and the eager update-phase time, of
  discrete    ff_ppo             vs ff_ppo_penalty                          (synthetic Box, the default MLP)
  continuous  ff_ppo_continuous  vs ff_ppo_penalty_continuous, ff_dpo_continuous   (default_ff_ppo_continuous's shape)
Every learner is built first; then `--rounds` rounds each time every system once, in turn, so that drift on a shared host spreads
over all of them.  The GPU's name and power limit are read in the same run.

    python scripts/bench_ppo_variants.py [--envs N] [--rollout T] [--updates K] [--rounds R]
Prints one JSON line per system (min / median / max over the rounds)."""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

# system -> (entry config, extra overrides); the continuous variants take ff_ppo_continuous's epochs / minibatches / rollout
SYSTEMS = {
    "ff_ppo": ("default_ff_ppo", ["env=synthetic/box"]),
    "ff_ppo_penalty": ("default_ff_ppo", ["env=synthetic/box"]),
    "ff_ppo_continuous": ("default_ff_ppo_continuous", []),
    "ff_ppo_penalty_continuous": ("default_ff_ppo_continuous", []),
    "ff_dpo_continuous": ("default_ff_dpo_continuous", ["system.epochs=4", "system.num_minibatches=16"]),
}


def _power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", f"--id={torch.cuda.current_device()}"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:  # no nvidia-smi: report the number without it
        return None


def _learner(system, envs, rollout, updates):
    from stoix_b200 import random as srandom
    from stoix_b200.config import compose
    from stoix_b200.utils import make_env as environments
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    name, extra = SYSTEMS[system]
    cfg = compose(name, ["logger.use_console=False", "arch.precision=f32", f"arch.total_num_envs={envs}", f"system.rollout_length={rollout}"]
                  + extra, config_dir="default/anakin")
    cfg.arch.total_timesteps = envs * rollout * updates * 2
    cfg.arch.num_evaluation = 2
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, _ = environments.make(cfg)
    mod = importlib.import_module(f"stoix_b200.systems.ppo.anakin.{system}")
    learn, _, state = mod.learner_setup(env, tuple(srandom.split(srandom.PRNGKey(0), 3)), cfg)
    out = learn(state)  # eager update + capture + replays (warm-up)
    torch.cuda.synchronize()
    return cfg, learn, out.learner_state


def _time(learn, state, n_upd):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = learn(state)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n_upd
    fn = learn.phases["update"]
    fn(out.learner_state)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(3):
        fn(out.learner_state)
    e1.record()
    torch.cuda.synchronize()
    return out.learner_state, ms, e0.elapsed_time(e1) / 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=1024)
    ap.add_argument("--rollout", type=int, default=128)
    ap.add_argument("--updates", type=int, default=5, help="captured update steps per timed window")
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    runs = {s: _learner(s, a.envs, a.rollout, a.updates) for s in SYSTEMS}
    res = {s: ([], []) for s in SYSTEMS}
    for _ in range(a.rounds):
        for s, (cfg, learn, state) in runs.items():
            state, ms, upd_ms = _time(learn, state, int(cfg.arch.num_updates_per_eval))
            runs[s] = (cfg, learn, state)
            res[s][0].append(ms)
            res[s][1].append(upd_ms)
    gpu, power = torch.cuda.get_device_name(), _power_limit_w()
    for s, (ms, upd) in res.items():
        cfg = runs[s][0]
        steps = a.envs * a.rollout
        rng = lambda xs: [min(xs), statistics.median(xs), max(xs)]
        print(json.dumps({"system": s, "env_steps_per_s": [steps / x * 1e3 for x in rng(ms)][::-1], "ms_per_update": rng(ms),
                          "update_phase_eager_ms": rng(upd), "rounds": a.rounds, "gpu": gpu, "power_limit_w": power,
                          "config": {"envs": a.envs, "rollout": a.rollout, "epochs": int(cfg.system.epochs),
                                     "minibatches": int(cfg.system.num_minibatches), "env": str(cfg.env.env_name), "dtype": "f32"}}))


if __name__ == "__main__":
    main()
