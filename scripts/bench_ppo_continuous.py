"""ff_ppo_continuous update-step timing at the default continuous config (configs/default/anakin/default_ff_ppo_continuous.yaml:
synthetic continuous Box obs_dim=17 act_dim=6, actor and critic MLP 4x256 silu, tanh-Normal head, fp32 SIMT kernels): env steps/s
and ms per update of the captured update step, the rollout / update split measured eagerly on the same state, the model FLOPs
per env step computed from the layer shapes, and the GPU's name and power limit read in the same run.

    python scripts/bench_ppo_continuous.py [--envs N] [--rollout T] [--updates K]
Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch


def _power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", f"--id={torch.cuda.current_device()}"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:  # no nvidia-smi: report the number without it
        return None


def _macs(sizes):
    return sum(sizes[i] * sizes[i + 1] for i in range(len(sizes) - 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=None, help="arch.total_num_envs (default: the config's)")
    ap.add_argument("--rollout", type=int, default=None, help="system.rollout_length (default: the config's)")
    ap.add_argument("--updates", type=int, default=10, help="timed update steps (graph replays)")
    a = ap.parse_args()
    from stoix_b200 import random as srandom
    from stoix_b200.config import compose
    from stoix_b200.systems.ppo.anakin import ff_ppo_continuous
    from stoix_b200.utils import make_env as environments
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    torch.cuda.set_device(0)
    cfg = compose("default_ff_ppo_continuous", ["logger.use_console=False"], config_dir="default/anakin")
    if a.envs is not None:
        cfg.arch.total_num_envs = a.envs
    if a.rollout is not None:
        cfg.system.rollout_length = a.rollout
    E, T = int(cfg.arch.total_num_envs), int(cfg.system.rollout_length)
    cfg.arch.total_timesteps = E * T * a.updates * 2
    cfg.arch.num_evaluation = 2
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, _ = environments.make(cfg)
    learn, _, state = ff_ppo_continuous.learner_setup(env, tuple(srandom.split(srandom.PRNGKey(0), 3)), cfg)
    out = learn(state)                       # eager update + capture + replays (warm-up)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = learn(out.learner_state)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / cfg.arch.num_updates_per_eval
    ph = {}
    st = out.learner_state
    for name in ("rollout", "update"):
        fn = learn.phases[name]
        for _ in range(2):
            fn(st)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(5):
            fn(st)
        e1.record()
        torch.cuda.synchronize()
        ph[name + "_eager_ms"] = e0.elapsed_time(e1) / 5
    sa, sc = learn.built["sa"], learn.built["sc"]
    epochs = int(cfg.system.epochs)
    # 2 FLOPs per multiply-add; rollout: actor + two critic evaluations per step; update: forward + backward (3x forward) of both
    # networks per sample and epoch
    fwd_a, fwd_c = 2 * _macs(sa.sizes), 2 * _macs(sc.sizes)
    flops = fwd_a + 2 * fwd_c + epochs * 3 * (fwd_a + fwd_c)
    steps = E * T
    print(json.dumps({"metric": "env steps/sec ff_ppo_continuous Anakin (synthetic continuous Box)", "value": steps / ms * 1e3,
                      "unit": "env_steps/s", "ms_per_update": ms, "model_flops_per_env_step": flops,
                      "model_tflops_per_s": flops * steps / ms * 1e3 / 1e12, "n_gpus": 1,
                      "gpu": torch.cuda.get_device_name(), "power_limit_w": _power_limit_w(),
                      "config": {"workload": f"ff_ppo_continuous, obs_dim={sa.sizes[0]} act_dim={sa.sizes[-1] // 2}, envs={E}, rollout={T}, "
                                             f"epochs={epochs}, minibatches={int(cfg.system.num_minibatches)}, actor/critic MLP[256x4] silu",
                                 "dtype": "f32", "cuda_graph": bool(cfg.arch.get("cuda_graph", True))}, **ph}))


if __name__ == "__main__":
    main()
