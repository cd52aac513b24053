"""The synthetic env's whole-trajectory kernel against T calls of its per-step kernel, and the rollout's once-per-observation
critic values against two full forward passes: every field bit for bit."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from stoix_b200 import ops

    return ops


def _buffers(T, E, D, dev="cuda:0"):
    z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev)
    return {"obs": z(T + 1, E, D, dt=torch.bfloat16), "next_obs": z(T, E, D, dt=torch.bfloat16), "reward": z(T, E),
            "done": z(T, E, dt=torch.uint8), "truncated": z(T, E, dt=torch.uint8), "ep_return": z(T, E),
            "ep_length": z(T, E, dt=torch.int32), "is_terminal": z(T, E, dt=torch.uint8)}


@pytest.mark.parametrize("E,T,D,p_term,p_trunc,counter", [
    (256, 40, 64, 0.05, 0.05, 0),                 # the benchmark's feature width; episodes end and truncate inside the window
    (37, 33, 24, 0.2, 0.1, (1 << 32) - 17),       # ragged env count, 6 feature groups on 8 lanes; the step crosses 2^32
    (130, 7, 8, 0.3, 0.3, (1 << 33) + 5),         # two feature groups, a window shorter than the lanes' outcome batch
    (64, 129, 128, 0.01, 0.02, (1 << 32) - 64),   # 32 feature groups: one env per warp
])
def test_trajectory_matches_per_step_env(E, T, D, p_term, p_trunc, counter):
    ops = _ops()
    dev = "cuda:0"
    seed, step = 0x9E3779B97F4A7C15, 3
    g = torch.Generator(device=dev)
    g.manual_seed(E * 1000 + T)
    obs0 = torch.randn(E, D, device=dev, generator=g).to(torch.bfloat16)
    rr0 = torch.randn(E, device=dev, generator=g)
    rl0 = torch.randint(0, 50, (E,), device=dev, generator=g, dtype=torch.int32)
    ctr = torch.tensor([counter], dtype=torch.int64, device=dev)

    a = _buffers(T, E, D)
    a["obs"][0] = obs0
    rr_a, rl_a = rr0.clone(), rl0.clone()
    ops.synth_env_trajectory(E, D, T, seed, step, p_term, p_trunc, a["obs"], a["next_obs"], a["reward"], a["done"], a["truncated"],
                             a["ep_return"], a["ep_length"], a["is_terminal"], rr_a, rl_a, dev_counter=ctr)

    b = _buffers(T, E, D)
    b["obs"][0] = obs0
    rr_b, rl_b = rr0.clone(), rl0.clone()
    act = torch.zeros(E, dtype=torch.int32, device=dev)
    for t in range(T):
        ops.synth_env_step(E, D, seed, step + t, p_term, p_trunc, act, b["obs"][t + 1], b["next_obs"][t], b["reward"][t], b["done"][t],
                           b["truncated"][t], rr_b, rl_b, b["ep_return"][t], b["ep_length"][t], b["is_terminal"][t], dev_counter=ctr)
    torch.cuda.synchronize()

    ended = b["is_terminal"].bool()
    assert ended.any() and b["truncated"].bool().any() and b["done"].bool().any(), "episodes should end inside the window"
    for k in a:
        assert torch.equal(a[k], b[k]), f"field {k} differs between the trajectory kernel and the per-step env"
    assert torch.equal(rr_a, rr_b) and torch.equal(rl_a, rl_b), "carried episode bookkeeping differs"


@pytest.mark.parametrize("E,T,D", [(256, 24, 64), (128, 13, 8)])
def test_rollout_values_match_two_forward_passes(E, T, D):
    ops = _ops()
    dev = "cuda:0"
    torch.manual_seed(E + T)
    spec = ops.MlpSpec((D, 256, 256, 1))
    params = torch.cat([(torch.randn(D * 256) / D ** 0.5), torch.randn(256) * 0.1, torch.randn(256 * 256) / 16, torch.randn(256) * 0.1,
                        torch.randn(256) / 16, torch.randn(1)]).to(dev)
    shadow = ops.cast_bf16(params)
    a = _buffers(T, E, D)
    a["obs"][0] = torch.randn(E, D, device=dev).to(torch.bfloat16)
    rr, rl = torch.zeros(E, device=dev), torch.zeros(E, dtype=torch.int32, device=dev)
    ops.synth_env_trajectory(E, D, T, 7, 0, 0.05, 0.05, a["obs"], a["next_obs"], a["reward"], a["done"], a["truncated"], a["ep_return"],
                             a["ep_length"], a["is_terminal"], rr, rl)
    value, boot = torch.full((T, E), float("nan"), device=dev), torch.full((T, E), float("nan"), device=dev)
    ops.tc_rollout_values(spec, params, shadow, a["obs"], a["next_obs"], a["is_terminal"], value, boot, ws_key="test-rollout-values")
    n = T * E
    v_ref = ops.mlp_forward(spec, params, a["obs"][:T].reshape(n, D), precision=ops.STX_PREC_BF16, params_bf16=shadow).view(T, E)
    b_ref = ops.mlp_forward(spec, params, a["next_obs"].reshape(n, D), precision=ops.STX_PREC_BF16, params_bf16=shadow).view(T, E)
    torch.cuda.synchronize()
    assert a["is_terminal"].bool().any()
    assert torch.equal(value, v_ref)
    assert torch.equal(boot, b_ref)
