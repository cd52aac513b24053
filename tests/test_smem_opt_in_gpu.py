"""Kernels that take more than 48 KB of dynamic shared memory raise their limit once per device (opt_in_smem,
stx_common.cuh).  The limit is a per-device attribute: a process-wide "done" flag would let only the first device opt in,
and the same launch on a second device would then fail (Sebulba's actor threads each run the bf16 forward on their own GPU).
The bf16 forward and the rollout policy run on cuda:0 and then on cuda:1 with the same inputs: each launches on both and
gives the same bits on both."""
import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O

pytestmark = pytest.mark.gpu

D, A, M, T, E = 64, 8, 1000, 4, 256


def _run(dev, net, x, obs):
    from stoix_b200 import ops

    with torch.cuda.device(dev):
        spec = ops.MlpSpec((D, 256, 256, A))
        params = torch.as_tensor(net.flat(), dtype=torch.float32, device=dev)
        shadow = ops.cast_bf16(params)
        xb = torch.as_tensor(x, device=dev).to(torch.bfloat16)
        out = ops.mlp_forward(spec, params, xb, precision=ops.STX_PREC_BF16, params_bf16=shadow)
        obs_b = torch.as_tensor(obs, device=dev).to(torch.bfloat16).contiguous()
        action = torch.empty((T, E), dtype=torch.int32, device=dev)
        log_prob = torch.empty((T, E), dtype=torch.float32, device=dev)
        counter = torch.zeros(1, dtype=torch.int64, device=dev)
        ops.tc_rollout_policy(spec, params, shadow, obs_b, action, log_prob, 1234, 0, counter)
        torch.cuda.synchronize(dev)
    return {"mlp_forward": out.cpu().numpy(), "action": action.cpu().numpy(), "log_prob": log_prob.cpu().numpy()}


def test_large_smem_kernels_run_on_a_second_device():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    rng = np.random.default_rng(0)
    net = O.init_mlp(rng, [D, 256, 256, A], 1.0)
    x = rng.standard_normal((M, D)).astype(np.float32)
    obs = rng.standard_normal((T, E, D)).astype(np.float32)
    ref = _run(0, net, x, obs)
    got = _run(1, net, x, obs)
    for k in ref:
        assert np.array_equal(got[k], ref[k]), f"{k}: cuda:1 differs from cuda:0"
