"""Sebulba ff_impala throughput next to Sebulba ff_ppo at the same shape, MLP torso on the synthetic Box CPU environment.

    python scripts/bench_impala.py [--threads 2] [--envs-per-thread 256] [--rollout-length 128] [--updates 24] [--minibatches 4]

One process per system: `threads` actor threads on cuda:0 (each: CPU envs -> pinned H2D -> forward + sampling kernels -> pinned D2H),
one learner thread on cuda:0.  Then, on the IMPALA learner's buffers as the run left them, one minibatch timed stage by stage with
CUDA events (forwards, V-trace, backwards, clip + RMSProp; median of 50) and the kernel launches of one learner step counted with
torch.profiler.  Prints ONE JSON line."""
import argparse
import json
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
from stoix_b200 import ops  # noqa: E402
from stoix_b200 import random as srandom  # noqa: E402
from stoix_b200.config import compose  # noqa: E402
from stoix_b200.envs import cpu as cpu_envs  # noqa: E402
from stoix_b200.systems.impala.sebulba import ff_impala  # noqa: E402
from stoix_b200.systems.ppo.sebulba import ff_ppo as seb  # noqa: E402
from stoix_b200.utils.logger import StoixLogger  # noqa: E402
from stoix_b200.utils.sebulba_utils import OnPolicyPipeline, ParameterServer, ThreadLifetime  # noqa: E402
from stoix_b200.utils.total_timestep_checker import check_total_timesteps  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--threads", type=int, default=2)
ap.add_argument("--envs-per-thread", type=int, default=256)
ap.add_argument("--rollout-length", type=int, default=128)
ap.add_argument("--updates", type=int, default=24)
ap.add_argument("--minibatches", type=int, default=4)
a = ap.parse_args()
E, T = a.threads * a.envs_per_thread, a.rollout_length
dev = torch.device("cuda", 0)


def run(system: str):
    mod = ff_impala if system == "ff_impala" else seb
    cfg = compose(f"default_{system}", [f"arch.total_num_envs={E}", f"system.rollout_length={T}", f"system.num_minibatches={a.minibatches}",
                                        f"arch.total_timesteps={E * T * a.updates}", f"arch.actor.actor_per_device={a.threads}",
                                        "arch.num_evaluation=1", "logger.use_console=False", "arch.precision=f32"], config_dir="default/sebulba")
    cfg.num_learner_devices, cfg.num_actor_devices, cfg.arch.world_size = 1, 1, 1
    cfg.arch.total_num_actor_threads = a.threads
    cfg = check_total_timesteps(cfg, quiet=True)
    factory = cpu_envs.make_factory(cfg)
    keys = srandom.split(srandom.PRNGKey(cfg.arch.seed), 4)
    torch.cuda.set_device(dev)
    learn_step, apply_fns, state = mod.learner_setup(factory, (keys[0], keys[2], keys[3]), [dev], cfg)
    logger = StoixLogger(cfg)
    ps = ParameterServer(a.threads, [dev], a.threads, queue_maxsize=1)
    pipe = OnPolicyPipeline(a.threads, queue_maxsize=1)
    ps.distribute_params(state.params)
    np_rng = np.random.default_rng(0)
    threads, lifetimes = [], []
    tkeys = srandom.split(keys[0], a.threads)
    for i in range(a.threads):
        lt = ThreadLifetime(f"Actor-{i}", i)
        th = mod.get_actor_thread(factory, dev, ps, pipe, apply_fns, tkeys[i], cfg, np_rng.integers(2 ** 31 - 1, size=a.envs_per_thread).tolist(),
                                  logger, [dev], lt)
        th.start()
        threads.append(th)
        lifetimes.append(lt)
    learner = seb.get_learner_thread(cfg, learn_step, state, ps, pipe, logger, None, keys[1])
    t0 = time.perf_counter()
    learner.start()
    learner.join()
    wall = time.perf_counter() - t0
    seb.stop_all_actor_threads(lifetimes, ps, pipe, threads)
    ls = learner.learner_rollout.stats
    steps = int(cfg.arch.num_updates) * E * T
    return {"env_steps_per_s": steps / wall, "learner_step_ms": 1e3 * ls.get("learn_step_time", 0.0), "updates": int(ls["updates"])}, \
        learn_step, learner.learner_rollout.final_state


impala, learn, state = run("ff_impala")
ppo, _, _ = run("ff_ppo")

# stage times of one IMPALA minibatch on the buffers the run left behind
b = learn.built
T_, Em = T, E // a.minibatches
idx = b["row_idx"][0]
x = b["obs"].view((T_ + 1) * E, b["D"])
a_tree = state.params.actor_params
sysc = dict(gamma=0.99, lambda_=1.0, clip_rho=1.0, clip_pg_rho=1.0, ent_coef=0.01, vf_coef=0.5)
stages = {
    "forwards": lambda: (ops.mlp_forward_train(b["sa"], b["arena"], x, b["ws_a"], out=b["logits"], row_idx=idx[: T_ * Em]),
                         ops.mlp_forward_train(b["sc"], b["arena"][b["coff"]:], x, b["ws_c"], out=b["values"].view(-1, 1), row_idx=idx)),
    "vtrace": lambda: ops.vtrace_loss_grads(b["logits"], b["values"], b["action"][:T_, :Em], b["log_prob"][:T_, :Em], b["reward"][:T_, :Em],
                                            b["done"][:T_, :Em], b["d_logits"], b["d_value"], b["metrics"][0], **sysc),
    "backwards": lambda: (ops.mlp_backward(b["sa"], b["arena"], x, b["d_logits"], b["ws_a"], net_grad=b["grads"], row_idx=idx[: T_ * Em]),
                          ops.mlp_backward(b["sc"], b["arena"][b["coff"]:], x, b["d_value"].view(-1, 1), b["ws_c"], net_grad=b["grads"][b["coff"]:],
                                           row_idx=idx)),
    "rmsprop": lambda: ops.clip_adam_step(b["plan"], b["arena"], b["grads"], a_tree.arena_mu, a_tree.arena_nu),
}
stage_us = {}
with torch.cuda.device(dev):
    for name, fn in stages.items():
        ts = []
        for _ in range(60):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ts.append(1e3 * e0.elapsed_time(e1))
        stage_us[name] = float(np.median(ts[10:]))
    # kernel launches of one learner step (two shards, as the actor threads deliver them)
    from stoix_b200.systems.impala.impala_types import ImpalaTransition

    half = E // 2
    shards = [ImpalaTransition(*[b[f][:, k * half:(k + 1) * half].clone() for f in ImpalaTransition._fields]) for k in range(2)]
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        learn(state, shards)
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
               and "memset" not in e.name.lower()]
    copies = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" in e.name.lower()]

props = torch.cuda.get_device_properties(dev)
try:
    import subprocess

    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
except OSError:
    power = "unknown"
print(json.dumps({
    "metric": "env steps/sec Sebulba ff_impala (MLP torso, synthetic Box CPU envs)", "value": impala["env_steps_per_s"], "unit": "env_steps/s",
    "config": {"workload": f"{a.threads} actor threads x {a.envs_per_thread} envs, rollout_len={T}, num_minibatches={a.minibatches}, obs_dim=64, "
                           "MLP[256,256], actor and learner on cuda:0, fp32"},
    "impala": impala, "ppo_same_shape": ppo,
    "impala_minibatch_us": stage_us, "impala_kernel_launches_per_update": len(kernels), "impala_copies_per_update": len(copies),
    "gpu": props.name, "power_limit": power,
    "note": "host-side numpy env stepping is inside the wall clock; PPO runs 4 epochs x num_minibatches Adam steps per update, IMPALA one epoch"}))
