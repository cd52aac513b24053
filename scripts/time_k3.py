"""Per-kernel device times of the bf16 PPO minibatch update at the benchmark shapes (E=4096, T=128, D=64, A=8, mb=32768).

Workload: 64 minibatch steps of `ops.ppo_minibatch_grads` (K3a `tc_ppo_fwd_bwd_kernel`, K3b `tc_dw_kernel`, `tc_reduce_kernel`)
+ `ops.clip_adam_step(prenorm=True)` (`clip_adam_kernel`) after a warm-up.  Two runs: one under torch.profiler (CUDA activities)
for per-kernel device times, one with the profiler off for a CUDA-event time of the whole 64-step loop.  Achieved GB/s and TFLOP/s
use the bytes and FLOPs the kernels need, computed from the shapes by `k3_accounting`.

    python scripts/time_k3.py --out /tmp/time_k3.json
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

E, T, D, A, MB = 4096, 128, 64, 8, 32768
H = 256
STEPS = 64
KERNELS = ("tc_ppo_fwd_bwd_kernel", "tc_dw_kernel", "tc_reduce_kernel", "clip_adam_kernel")
DW_SPLIT = (19, 13, 15)  # K3b's split-K CTAs per dW1 half, dW2, dW0 (stx_tc_ppo.cu kDwCtasW1 / W2 / W0)


def k3_accounting(mb: int = MB, d: int = D, n_params: int = 0, rebuild: bool = True) -> dict:
    """HBM bytes and tensor FLOPs of one minibatch step, per kernel, from the shapes (both networks).

    Bytes are what each kernel has to move: the activations K3a writes and K3b reads in their stored widths (tiled bf16, dz
    padded to 16 columns, the h2 sign mask 32 B per row), the gathered input rows, indices and loss inputs, the fp32 partials.
    rebuild=True is the current layout: K3b's dW1 half-jobs rebuild h1 and dh2 from x, dz and the mask, so those two never
    reach HBM.  rebuild=False is the earlier layout, where K3a stored h1 and dh2 and both dW1 half-jobs streamed all of h1
    and half of dh2.  FLOPs are the MMA work as executed (heads padded to N=16, the input layer to K=64)."""
    w1, w2, w0 = DW_SPLIT
    x_row, act_row, dz_row, mask_row = 2 * d, 2 * H, 2 * 16, H // 8
    # K3a, per row: both nets gather x and read the index twice; the actor reads action, logp, adv, the critic value, target
    k3a_read = 2 * (x_row + 2 * 4) + 3 * 4 + 2 * 4
    if rebuild:  # per net: h2, dh1, dz, mask; xg once (actor CTAs)
        k3a_write = 2 * (2 * act_row + dz_row + mask_row) + x_row
        dw1_read = 2 * (x_row + dz_row + mask_row)  # two half-jobs
    else:  # per net: h1, h2, dh1, dh2, dz; xg once
        k3a_write = 2 * (4 * act_row + dz_row) + x_row
        dw1_read = 2 * (act_row + act_row // 2)
    k3b_read = 2 * (dw1_read + (act_row + dz_row) + (act_row + x_row))  # dW1, dW2 = h2^T dz, dW0 = dh1^T x, per net
    part_floats = 2 * (2 * w1 * 128 * H + w2 * H * 16 + w0 * H * 64)
    db_floats = 2 * 66 * 528
    k3a_flop = 2 * 2 * (64 * H + H * H + H * 16 + 16 * H + H * H)  # G0..G4 per row, both nets
    k3b_flop = 2 * 2 * (H * H + H * 16 + H * 64)
    if rebuild:  # per half-job: h1 half (K=64, N=128) and dh2 (K=16, N=256)
        k3b_flop += 2 * 2 * 2 * (64 * 128 + 16 * H)
    return {
        "tc_ppo_fwd_bwd_kernel": {"bytes": mb * (k3a_read + k3a_write) + 4 * db_floats, "flop": mb * k3a_flop,
                                  "activation_write_bytes": mb * k3a_write},
        "tc_dw_kernel": {"bytes": mb * k3b_read + 4 * part_floats, "flop": mb * k3b_flop, "activation_read_bytes": mb * k3b_read},
        "tc_reduce_kernel": {"bytes": 4 * (part_floats + db_floats) + 4 * n_params, "flop": 0},
        "clip_adam_kernel": {"bytes": 28 * n_params, "flop": 0},
    }


def _gpu_info() -> dict:
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]
    try:
        line = subprocess.run(q, capture_output=True, text=True, check=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in line.split(",")]
        return {"name": name, "power_limit": power, "clocks_max_sm": clock}
    except Exception as e:  # the timings are still worth having; say why the card is unnamed
        return {"error": repr(e)}


def _setup():
    import torch

    from stoix_b200 import ops

    dev = torch.device("cuda:0")
    B = T * E
    g = torch.Generator(device=dev).manual_seed(0)
    sa, sc = ops.MlpSpec((D, H, H, A)), ops.MlpSpec((D, H, H, 1))
    _, coff, total = ops.arena_offsets(sa, sc)
    arena = torch.randn(total, device=dev, generator=g) * 0.05
    shadow = ops.cast_bf16(arena)
    mu, nu = torch.zeros_like(arena), torch.zeros_like(arena)
    obs = torch.randn(B, D, device=dev, generator=g).to(torch.bfloat16)
    action = torch.randint(0, A, (B,), device=dev, generator=g, dtype=torch.int32)
    log_prob = -torch.rand(B, device=dev, generator=g) * 2.0 - 0.5
    value, adv, tgt = (torch.randn(B, device=dev, generator=g) for _ in range(3))
    stats = torch.stack([adv.mean(), 1.0 / adv.std()]).float().contiguous()
    perm = ops.make_permutation(B, 7, 0, device=dev)
    batch = ops.PpoBatch(obs, action, log_prob, value, adv, tgt, stats, perm)
    grads, metrics = torch.zeros(total, device=dev), torch.zeros(8, device=dev)
    ws = ops.ppo_workspace(sa, sc, MB, ops.STX_PREC_BF16, dev)
    plan = ops.AdamPlan([(0, sa.param_count, 3e-4, 0.5), (coff, sc.param_count, 3e-4, 0.5)], dev, steps_per_update=64, num_updates=100)

    def step(i: int) -> None:
        ops.ppo_minibatch_grads(sa, sc, arena, batch, (i % (B // MB)) * MB, MB, 0.2, 0.01, 0.5, True, grads, metrics, ws,
                                ops.STX_PREC_BF16, 1.0, shadow, overwrite=True, adam_scratch=plan.scratch)
        ops.clip_adam_step(plan, arena, grads, mu, nu, params_bf16=shadow, prenorm=True)

    return step, sa.param_count + sc.param_count


def run_once(rebuild: bool) -> dict:
    import torch
    from torch.profiler import ProfilerActivity, profile

    if not torch.cuda.is_available():
        raise SystemExit("time_k3.py measures on a CUDA device; none is visible")
    step, n_params = _setup()
    for i in range(2 * 16):  # warm-up: every minibatch offset once, twice
        step(i)
    torch.cuda.synchronize()

    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for i in range(STEPS):
        step(i)
    ev1.record()
    torch.cuda.synchronize()
    loop_ms = ev0.elapsed_time(ev1)

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(STEPS):
            step(i)
        torch.cuda.synchronize()
    dev_us = {k: 0.0 for k in KERNELS}
    calls = {k: 0 for k in KERNELS}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key:
                dev_us[k] += ev.self_device_time_total
                calls[k] += ev.count
    acc = k3_accounting(n_params=n_params, rebuild=rebuild)
    kernels = {}
    for k in KERNELS:
        us = dev_us[k] / STEPS
        b, f = acc[k]["bytes"], acc[k]["flop"]
        kernels[k] = {"us_per_step": round(us, 2), "launches": calls[k], "mbytes": round(b / 1e6, 2), "gflop": round(f / 1e9, 3),
                      "gb_per_s": round(b / (us * 1e-6) / 1e9, 1) if us > 0 else None,
                      "tflop_per_s": round(f / (us * 1e-6) / 1e12, 1) if us > 0 and f else None}
    return {"split": list(DW_SPLIT), "loop_us_per_step": round(loop_ms / STEPS * 1e3, 2), "steps": STEPS, "kernels": kernels,
            "sum_kernel_us_per_step": round(sum(v["us_per_step"] for v in kernels.values()), 2)}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="JSON output path")
    ap.add_argument("--layout", choices=("rebuild", "stored"), default="rebuild",
                    help="byte accounting of the build under test: rebuild (current) or stored (h1 and dh2 through HBM, earlier builds)")
    args = ap.parse_args()
    res = {"gpu": _gpu_info(), "shape": {"E": E, "T": T, "D": D, "A": A, "mb": MB}, "layout": args.layout,
           "default": run_once(args.layout == "rebuild")}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
