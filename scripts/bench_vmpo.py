"""V-MPO next to fp32 PPO at the same shape: env steps/s and ms per captured update step, and an eager split of the update step into
rollout, targets (one epoch's critic evaluation + GAE, which the update repeats every epoch) and update phase, of
  cartpole    ff_vmpo            vs ff_ppo             (the reference's ff_vmpo default: CartPole, 1024 envs, T = 32, 16 epochs, MLP 2 x 256)
  wide        ff_vmpo            vs ff_ppo             (synthetic Box, --wide-envs envs, T = 32)
  continuous  ff_vmpo_continuous vs ff_ppo_continuous  (default_ff_ppo_continuous's shape: synthetic continuous, 1024 envs, T = 128)
Every learner is built first; then `--rounds` rounds time every system once, in turn, so that drift on a shared host spreads over all
of them.  A last eager V-MPO update phase of each workload runs under torch.profiler, which gives the top-k and loss kernels' share of
the device time.  The GPU's name and power limit are read in the same run.

    python scripts/bench_vmpo.py [--updates K] [--rounds R] [--wide-envs E]
Prints one JSON line per (workload, system): min / median / max over the rounds."""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

MODULES = {"ff_vmpo": "stoix_b200.systems.mpo.ff_vmpo", "ff_vmpo_continuous": "stoix_b200.systems.mpo.ff_vmpo_continuous",
           "ff_ppo": "stoix_b200.systems.ppo.anakin.ff_ppo", "ff_ppo_continuous": "stoix_b200.systems.ppo.anakin.ff_ppo_continuous"}


def workloads(wide_envs):
    """(workload, system, entry config, overrides, envs, rollout)"""
    return [
        ("cartpole", "ff_vmpo", "default_ff_vmpo", [], 1024, 32),
        ("cartpole", "ff_ppo", "default_ff_ppo", ["env=gymnax/cartpole"], 1024, 32),
        ("wide", "ff_vmpo", "default_ff_vmpo", ["env=synthetic/box"], wide_envs, 32),
        ("wide", "ff_ppo", "default_ff_ppo", ["env=synthetic/box"], wide_envs, 32),
        ("continuous", "ff_vmpo_continuous", "default_ff_vmpo_continuous", [], 1024, 128),
        ("continuous", "ff_ppo_continuous", "default_ff_ppo_continuous", [], 1024, 128),
    ]


def _power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", f"--id={torch.cuda.current_device()}"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:  # no nvidia-smi: report the number without it
        return None


def _learner(system, name, extra, envs, rollout, updates):
    from stoix_b200 import random as srandom
    from stoix_b200.config import compose
    from stoix_b200.utils import make_env as environments
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    cfg = compose(name, ["logger.use_console=False", "arch.precision=f32", f"arch.total_num_envs={envs}", f"system.rollout_length={rollout}"] + extra,
                  config_dir="default/anakin")
    cfg.arch.total_timesteps = envs * rollout * updates * 2
    cfg.arch.num_evaluation = 2
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, _ = environments.make(cfg)
    mod = importlib.import_module(MODULES[system])
    learn, _, state = mod.learner_setup(env, tuple(srandom.split(srandom.PRNGKey(0), 3)), cfg)
    out = learn(state)  # eager update + capture + replays (warm-up)
    torch.cuda.synchronize()
    return cfg, learn, out.learner_state


def _events(fn, reps=1):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _time(learn, state, n_upd):
    """(state, ms per captured update, eager rollout ms, eager targets ms (one epoch's, or the PPO GAE), eager update-phase ms)"""
    out = None

    def run():
        nonlocal out
        out = learn(state)

    ms = _events(run) / n_upd
    st = out.learner_state
    ph = learn.phases
    roll = _events(lambda: ph["rollout"](st))
    tgt = _events(lambda: ph["targets"](st) if "targets" in ph else ph["gae"](st))
    upd = _events(lambda: ph["update"](st))
    return st, ms, roll, tgt, upd


def _kernel_share(learn, state):
    """Device time of one eager update phase by kernel, from torch.profiler: the top-k and loss kernels against the total."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        learn.phases["update"](state)
        torch.cuda.synchronize()
    tot, topk, loss = 0.0, 0.0, 0.0
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        tot += t
        if "topk_" in e.key:
            topk += t
        elif "vmpo_stats" in e.key or "vmpo_grads" in e.key:
            loss += t
    return {"update_device_ms": tot / 1e3, "topk_ms": topk / 1e3, "loss_ms": loss / 1e3, "topk_share": topk / tot if tot else None,
            "loss_share": loss / tot if tot else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=4, help="captured update steps per timed window")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--wide-envs", type=int, default=8192)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    wl = workloads(a.wide_envs)
    runs = {(w, s): (_learner(s, n, ex, E, T, a.updates), E, T) for w, s, n, ex, E, T in wl}
    res = {k: ([], [], [], [], []) for k in runs}
    for _ in range(a.rounds):
        for k, ((cfg, learn, state), E, T) in runs.items():
            state, *times = _time(learn, state, int(cfg.arch.num_updates_per_eval))
            runs[k] = ((cfg, learn, state), E, T)
            for lst, x in zip(res[k], times):
                lst.append(x)
    gpu, power = torch.cuda.get_device_name(), _power_limit_w()
    rng = lambda xs: [min(xs), statistics.median(xs), max(xs)]
    for (w, s), (ms, roll, tgt, upd, _) in ((k, v) for k, v in res.items()):
        (cfg, learn, state), E, T = runs[(w, s)]
        line = {"workload": w, "system": s, "env_steps_per_s": [E * T / x * 1e3 for x in rng(ms)][::-1], "ms_per_update": rng(ms),
                "eager_rollout_ms": rng(roll), "eager_targets_ms": rng(tgt), "eager_update_phase_ms": rng(upd), "rounds": a.rounds, "gpu": gpu,
                "power_limit_w": power, "config": {"envs": E, "rollout": T, "epochs": int(cfg.system.epochs),
                                                    "minibatches": int(cfg.system.get("num_minibatches", 1)), "env": str(cfg.env.env_name), "dtype": "f32"}}
        if s.startswith("ff_vmpo"):
            line["kernels"] = _kernel_share(learn, state)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
