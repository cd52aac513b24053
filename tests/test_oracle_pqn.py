"""CPU checks of the PQN oracle (tests/pqn_oracle.py) against independent computations, and of the PQN configuration."""
import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from tests import pqn_oracle as P


def _torch_mlp(p: O.MLPParams, x: torch.Tensor) -> torch.Tensor:
    """Autograd restatement of MLPTorso(silu, LayerNorm eps 1e-6) + Dense head over float64 leaves."""
    h = x
    n = len(p.W)
    for i in range(n):
        W = torch.tensor(p.W[i], requires_grad=True)
        b = torch.tensor(p.b[i], requires_grad=True)
        p._leaves.append((W, b))
        if p.has_ln(i):
            bias = torch.tensor(p.ln_bias[i], requires_grad=True)
            p._leaves[-1] = (W, b, bias)
            u = h @ W
            z = torch.nn.functional.layer_norm(u, (u.shape[-1],), b, bias, eps=O.LN_EPS)
        else:
            z = h @ W + b
        h = torch.nn.functional.silu(z) if i < n - 1 else z
    return h


@pytest.mark.parametrize("delta", [0.0, 0.5])
@pytest.mark.parametrize("ln", [False, True])
def test_q_loss_gradient_matches_autograd(delta, ln):
    rng = np.random.default_rng(3)
    sizes = [6, 16, 16, 5]
    p = O.init_mlp(rng, sizes, 1.0)
    p = O.MLPParams(p.W, p.b, "silu", [rng.normal(size=s) * 0.1 for s in sizes[1:-1]] + [None] if ln else None)
    if ln:
        p.b[:-1] = [1.0 + 0.1 * rng.normal(size=s) for s in sizes[1:-1]]
    m = 12
    x = rng.normal(size=(m, 6))
    a = rng.integers(0, 5, size=m)
    q, acts = O.mlp_forward(p, x)
    tg = q[np.arange(m), a] + rng.normal(size=m)
    tg[0] = q[0, a[0]]                    # td = 0
    if delta > 0:
        tg[1] = q[1, a[1]] + delta        # |td| = delta exactly
        tg[2] = q[2, a[2]] - delta
    loss, dq = P.q_loss_and_dq(q, a, tg, delta)
    grads = O.mlp_backward(p, acts, dq)

    p._leaves = []
    qt = _torch_mlp(p, torch.tensor(x))
    td = torch.tensor(tg) - qt[torch.arange(m), torch.tensor(a)]
    if delta > 0:
        ax = td.abs()
        quad = torch.clamp(ax, max=delta)
        lt = (0.5 * quad ** 2 + delta * (ax - quad)).mean()
    else:
        lt = (0.5 * td ** 2).mean()
    lt.backward()
    assert abs(float(lt.detach()) - loss) < 1e-12
    for i, leaves in enumerate(p._leaves):
        np.testing.assert_allclose(grads.W[i], leaves[0].grad.numpy(), rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(grads.b[i], leaves[1].grad.numpy(), rtol=1e-9, atol=1e-12)
        if len(leaves) == 3:
            np.testing.assert_allclose(grads.ln_bias[i], leaves[2].grad.numpy(), rtol=1e-9, atol=1e-12)


def test_huber_tie_gives_the_same_value_and_gradient_on_both_branches():
    q = np.array([[0.0, 1.0]])
    for td in (0.5, -0.5):
        loss, dq = P.q_loss_and_dq(q, np.array([1]), np.array([1.0 + td]), 0.5)
        assert loss == 0.5 * 0.25 and dq[0, 1] == -td   # quadratic branch 0.5 td^2, linear branch delta^2 / 2 + 0


def test_radam_restatement_matches_torch_radam_across_the_rectifier_switch():
    rng = np.random.default_rng(0)
    n = 37
    p0 = rng.normal(size=n)
    p = p0.copy()
    st = P.RadamState(np.zeros(n), np.zeros(n))
    tp = torch.tensor(p0.copy(), requires_grad=True)
    opt = torch.optim.RAdam([tp], lr=1e-2, betas=(0.9, 0.999), eps=0.0)
    branches = []
    for step in range(50):
        g = rng.normal(size=n)
        p = P.clip_radam_step(p, g, st, 1e-2, 1e30, b1=0.9, b2=0.999, eps=0.0)
        tp.grad = torch.tensor(g)
        opt.step()
        branches.append(P.radam_rectifier(0.999, step + 1) is not None)
        np.testing.assert_allclose(p, tp.detach().numpy(), rtol=1e-12, atol=1e-14)
    assert branches[:5] == [False] * 5 and all(branches[5:])   # steps 1-5 un-rectified, step 6 the first rectified one


def test_radam_rectifier_in_fp32_is_what_the_kernel_avoids():
    """The relative error of a literal fp32 rectifier (DESIGN.md section 2, tolerance scheme): 1.8e-3 at t = 6, 6e-5 at t = 10."""
    def r32(t):
        f = np.float32
        b2 = f(0.999)
        rho_inf = f(2) / (f(1) - b2) - f(1)
        b2t = b2 ** f(t)
        rho = rho_inf - f(2) * f(t) * b2t / (f(1) - b2t)
        return float(np.sqrt((rho - f(4)) * (rho - f(2)) * rho_inf / ((rho_inf - f(4)) * (rho_inf - f(2)) * rho)))

    rel = lambda t: abs(r32(t) - P.radam_rectifier(float(np.float32(0.999)), t)) / P.radam_rectifier(float(np.float32(0.999)), t)
    assert 1e-3 < rel(6) < 3e-3
    assert 2e-5 < rel(10) < 2e-4


@pytest.mark.parametrize("lam", [0.0, 0.95, 1.0])
def test_lambda_returns_against_a_loop_and_the_gae_identity(lam):
    rng = np.random.default_rng(1)
    T, E, A = 9, 5, 3
    r = rng.normal(size=(T, E))
    d = 0.99 * (rng.random((T, E)) > 0.2)
    q = rng.normal(size=(T, E, A))
    G = P.batch_q_lambda(r, d, q, lam)
    v = q.max(-1)
    # independent loop over n-step returns: G_t = sum_n weights of the n-step bootstrapped returns
    for e in range(E):
        for t in range(T):
            total, w_left, disc, ret = 0.0, 1.0, 1.0, 0.0
            for k in range(t, T):
                ret += disc * r[k, e]
                disc *= d[k, e]
                w = (1 - lam) if k < T - 1 else 1.0
                total += w_left * w * (ret + disc * v[k, e])
                w_left *= lam
            np.testing.assert_allclose(G[t, e], total, rtol=1e-12, atol=1e-12)
    # G = v_tm1 + GAE with v_tm1[t + 1] = v_t[t]
    v_tm1 = np.concatenate([rng.normal(size=(1, E)), v[:-1]], axis=0)
    adv = np.zeros((T, E))
    acc = np.zeros(E)
    for t in range(T - 1, -1, -1):
        acc = r[t] + d[t] * v[t] - v_tm1[t] + d[t] * lam * acc
        adv[t] = acc
    np.testing.assert_allclose(G, v_tm1 + adv, rtol=1e-12, atol=1e-12)


def test_epsilon_schedule_at_update_boundaries():
    from stoix_b200.systems.q_learning import ff_pqn

    s = ff_pqn.linear_schedule(1.0, 0.1, 5.0)
    got = [s(k) for k in range(8)]
    np.testing.assert_array_equal(np.array(got, np.float32), P.epsilon_at(1.0, 0.1, 5.0, True, np.arange(8)))
    assert got[0] == np.float32(1.0) and got[5] == got[7] == np.float32(0.1)
    assert ff_pqn.linear_schedule(1.0, 0.1, 0.0)(3) == np.float32(1.0)
    assert ff_pqn.constant_schedule(0.25)(9) == np.float32(0.25)


def test_epsilon_greedy_oracle_distribution():
    rng = np.random.default_rng(0)
    E, A = 20000, 4
    q = np.tile(np.array([[1.0, 3.0, 3.0, 0.0]], np.float32), (E, 1))
    a = P.epsilon_greedy(q, 0.2, seed=12345, call=7)
    freq = np.bincount(a, minlength=A) / E
    np.testing.assert_allclose(freq, [0.05, 0.45, 0.45, 0.05], atol=0.015)
    assert (P.epsilon_greedy(q, 1.0, 1, 0) != 1).sum() > 0
    np.testing.assert_array_equal(P.epsilon_greedy(q, 0.5, 1, 0, mode=True), np.ones(E, np.int32))
    del rng


def test_default_ff_pqn_composes_and_resolves():
    import stoix  # noqa: F401  (the stoix alias)
    from stoix_b200.config import compose, instantiate
    from stoix_b200.networks.heads import DiscreteQNetworkHead
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    cfg = compose("default_ff_pqn", ["arch.total_num_envs=1024", "arch.total_timesteps=5e5"], config_dir="default/anakin")
    cfg.num_devices = 1
    cfg = check_total_timesteps(cfg, quiet=True)
    assert (cfg.system.rollout_length, cfg.system.epochs, cfg.system.num_minibatches) == (8, 4, 16)
    assert cfg.arch.num_envs == 1024 and cfg.arch.num_updates == 61
    node = cfg.network.actor_network
    assert node.action_head._target_ == "stoix.networks.heads.DiscreteQNetworkHead"
    assert node.pre_torso.activation == "silu" and list(node.pre_torso.layer_sizes) == [256, 256]
    head = instantiate(node.action_head, action_dim=2, epsilon=0.05)
    assert isinstance(head, DiscreteQNetworkHead) and head.out_dim == 2 and head.epsilon == 0.05 and head.kernel_init_scale == 1.0
    import stoix.networks.heads as aliased

    assert aliased.DiscreteQNetworkHead is DiscreteQNetworkHead
    import stoix.systems.q_learning.ff_pqn as launch
    from stoix_b200.systems.q_learning import ff_pqn

    assert launch is ff_pqn


def test_radam_chain_and_bf16_refusal_on_the_host():
    from stoix_b200 import optim
    from stoix_b200.config import compose
    from stoix_b200.systems.q_learning import ff_pqn

    opt = optim.chain(optim.clip_by_global_norm(0.5), optim.radam(5e-4))
    assert opt.rule == "radam" and opt.max_grad_norm == 0.5 and opt.init_lr == 5e-4
    cfg = compose("default_ff_pqn", ["arch.precision=bf16"], config_dir="default/anakin")
    with pytest.raises(ValueError, match="bf16"):
        ff_pqn._refuse_bf16(cfg)
