"""ff_mpo and ff_mpo_continuous on one GPU: env-steps/s and ms per captured update at three workloads, and a torch.profiler share of
the update's device time in the ring sample (seq_*), the target-Q input rows and loss kernels (mpo_*, retrace, q_grad) and every other
kernel (the MLP forwards and backwards, the sampled target-Q forward among them).  Reads the GPU name and power limit in the same run.

  python scripts/bench_mpo.py [--updates 5]

The workloads: ff_mpo at the reference CartPole default, ff_mpo_continuous at its default on synthetic continuous (M = 4096 states,
2 x 128 sampled actions per state), and a smaller continuous shape (32 samples, 64 sequences).  ff_dqn / ff_sac rates at their shapes
come from scripts/bench_dqn.py / bench_sac.py."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

WORKLOADS = {
    "ff_mpo cartpole default": ("ff_mpo", []),
    "ff_mpo_continuous default": ("ff_mpo_continuous", []),
    "ff_mpo_continuous small": ("ff_mpo_continuous", ["system.num_samples=32", "system.total_batch_size=64", "system.epochs=16"]),
}


def _learner(system, overrides):
    import importlib

    from stoix_b200 import random as srandom
    from stoix_b200.config import compose
    from stoix_b200.utils import make_env
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps
    cfg = compose(f"default_{system}", ["arch.total_timesteps=~", "arch.num_updates=100", "logger.use_console=False", *overrides],
                  config_dir="default/anakin")
    cfg.num_devices = 1
    cfg = check_total_timesteps(cfg, quiet=True)
    env, _ = make_env.make(cfg)
    key, _, a_key, q_key = srandom.split(srandom.PRNGKey(0), num=4)
    learn, _, state = importlib.import_module(f"stoix_b200.systems.mpo.{system}").learner_setup(env, (key, a_key, q_key), cfg)
    return cfg, learn, state


def _group(name):
    if name.startswith("seq_") or "seq_sample" in name or "seq_write" in name:
        return "ring"
    if any(k in name for k in ("mpo_", "retrace", "q_grad")):
        return "mpo_kernels"
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=5)
    args = ap.parse_args()
    from stoix_b200.systems import anakin
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    for label, (system, over) in WORKLOADS.items():
        cfg, learn, state = _learner(system, over)
        learn.ensure_built(state)
        b = learn.built
        items = int(cfg.system.rollout_length) * int(cfg.arch.num_envs)
        step = lambda: anakin.update_once(b, True, learn.update_step, state, state.buffer_state, items)
        for _ in range(3):   # eager, capture, one replay
            step()
        torch.cuda.synchronize()
        t0 = time.time()
        for _ in range(args.updates):
            step()
        torch.cuda.synchronize()
        ms = (time.time() - t0) * 1e3 / args.updates
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        share = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0))
            share[_group(ev.key)] = share.get(_group(ev.key), 0.0) + t
        tot = sum(share.values()) or 1.0
        print(json.dumps({"workload": label, "gpu": gpu, "env_steps_per_s": items / (ms / 1e3), "ms_per_update": ms,
                          "device_time_share": {k: v / tot for k, v in sorted(share.items())}}), flush=True)
        del learn, state, b


if __name__ == "__main__":
    main()
