"""rec_r2d2 on the CPU: the fp64 oracle against torch autograd and its own restatements, the configs, the launch file, the arena
layout with flax's names, and the refusals."""
import numpy as np
import pytest
import torch

from tests import r2d2_oracle as orc


def test_value_transform_round_trips():
    x = np.concatenate([-np.logspace(-8, 6, 57), [0.0], np.logspace(-8, 6, 57)])
    np.testing.assert_allclose(orc.h_inv(orc.h(x)), x, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(orc.h(orc.h_inv(x)), x, rtol=1e-9, atol=1e-12)


def test_stable_transforms_equal_the_published_forms():
    x = np.concatenate([-np.logspace(-3, 8, 45), np.logspace(-3, 8, 45)])
    np.testing.assert_allclose(orc.h_stable(x), orc.h(x), rtol=1e-11)
    np.testing.assert_allclose(orc.h_inv_stable(x), orc.h_inv(x), rtol=1e-9)
    tiny = np.array([1e-30, -1e-20, 1e-12])   # first-order terms: h'(0) = 1/2 + eps, (h^-1)'(0) = 1 / h'(0)
    np.testing.assert_allclose(orc.h_stable(tiny), tiny * (0.5 + orc.TX_EPS), rtol=1e-9)
    np.testing.assert_allclose(orc.h_inv_stable(tiny), tiny / (0.5 + orc.TX_EPS), rtol=1e-9)


def test_n_step_padding_at_the_window_end():
    """seq_len < n - 1 and the last n - 1 targets: r padded with zeros, d with ones, v with its last value."""
    rng = np.random.default_rng(0)
    for seq, n in ((3, 5), (7, 5), (6, 1), (1, 3)):
        r, d, v = rng.normal(size=seq), rng.uniform(0, 1, size=seq), rng.normal(size=seq) * 5
        want = np.zeros(seq)
        for t in range(seq):
            g = v[min(t + n - 1, seq - 1)]
            for i in reversed(range(n)):
                k = t + i
                g = orc.h((r[k] if k < seq else 0.0) + (d[k] if k < seq else 1.0) * orc.h_inv(g))
            want[t] = g
        np.testing.assert_allclose(orc.transformed_n_step_returns(r, d, v, n), want, rtol=1e-12)


def _torch_loss(q, q_tg, action, reward, done, prob, n, gamma, max_abs, beta, stop: bool = True):
    """The reference's _q_loss_fn in torch float64, with the targets under stop_gradient (or, stop=False, differentiable)."""
    T, B, A = q.shape
    eps = orc.TX_EPS
    h = lambda x: torch.sign(x) * (torch.sqrt(torch.abs(x) + 1) - 1) + eps * x
    hi = lambda x: torch.sign(x) * (torch.square(torch.sqrt(1 + 4 * eps * (eps + 1 + torch.abs(x))) / 2 / eps - 1 / 2 / eps) - 1)
    sel = q.argmax(-1)
    v = torch.gather(q_tg[1:], 2, sel[1:, :, None])[..., 0]
    v = v.detach() if stop else v
    r = torch.clamp(reward, -max_abs, max_abs)[:-1]
    d = ((1 - done.double()) * gamma)[:-1]
    seq = T - 1
    r = torch.cat([r, torch.zeros(n - 1, B, dtype=r.dtype)])
    d = torch.cat([d, torch.ones(n - 1, B, dtype=d.dtype)])
    tgt = torch.cat([v[n - 1:], v[-1:].expand(min(n - 1, seq), B)])
    for i in reversed(range(n)):
        tgt = h(r[i:i + seq] + d[i:i + seq] * hi(tgt))
    td = (tgt.detach() if stop else tgt) - torch.gather(q[:-1], 2, action[:-1, :, None].long())[..., 0]
    iw = (1.0 / (prob + 1e-6)) ** beta
    return torch.mean(iw / iw.max() * 0.5 * (td ** 2).sum(0))


@pytest.mark.parametrize("T,B,A,n", [(9, 4, 3, 5), (4, 3, 2, 5), (12, 5, 4, 1)])
def test_loss_oracle_against_autograd(T, B, A, n):
    rng = np.random.default_rng(T * B)
    q, q_tg = rng.normal(size=(T, B, A)) * 3, rng.normal(size=(T, B, A)) * 3
    q[2, 0, :] = 1.0   # a tie: the first maximum
    action, reward = rng.integers(0, A, size=(T, B)), rng.normal(size=(T, B)) * 2
    done = (rng.uniform(size=(T, B)) < 0.2).astype(np.uint8)
    prob = rng.uniform(0.01, 0.2, size=B)
    out = orc.loss(q, q_tg, action, reward, done, prob, n, 0.99, 1.5, 0.9, 0.7)
    qt = torch.tensor(q, requires_grad=True)
    L = _torch_loss(qt, torch.tensor(q_tg), torch.tensor(action), torch.tensor(reward), torch.tensor(done), torch.tensor(prob), n, 0.99, 1.5, 0.7)
    L.backward()
    assert abs(L.item() - out["loss"]) < 1e-12 * max(1.0, abs(out["loss"]))
    np.testing.assert_allclose(out["d_q"], qt.grad.numpy(), rtol=1e-10, atol=1e-14)


@pytest.mark.parametrize("dueling", [False, True])
def test_burn_in_and_targets_get_no_gradient(dueling):
    """The oracle's gradient equals torch autograd of the whole loss with the burn-in carries and the targets under stop_gradient, and
    differs from autograd with either left differentiable, so both stops are in effect (online = target parameters, so a target path
    would reach the same leaves).  The dueling head's gradient is almost all in the value LayerNorm bias (its advantage LayerNorm
    over two actions passes almost none), so the differences are measured on the plain head."""
    lay, net = _layout("gru", dueling=dueling, H=8, sizes=8, D=3)
    rng = np.random.default_rng(1)
    flat = net.init(0, torch.zeros(1, 8), (torch.zeros(1, 1, 3), torch.zeros(1, 1, dtype=torch.bool))).flat.double().numpy()
    flat = flat + 0.05 * rng.normal(size=flat.shape)
    S, B, bi, n = 7, 3, 3, 3
    seq = {"obs": rng.normal(size=(S, B, 3)), "reset": np.zeros((S, B), np.uint8), "carry0": rng.normal(size=(B, 8)) * 0.5,
           "action": rng.integers(0, 2, size=(S, B)), "reward": rng.normal(size=(S, B)), "done": np.zeros((S, B), np.uint8)}
    prob = np.array([0.1, 0.3, 0.2])
    g, _ = orc.q_loss_grad(lay, flat, flat, seq, bi, prob, n, 0.99, 1000.0, 0.9, 0.6)

    def autograd(stop_burn_in: bool, stop_targets: bool) -> np.ndarray:
        p = torch.tensor(flat, requires_grad=True)
        obs, reset, c0 = torch.tensor(seq["obs"]), torch.tensor(seq["reset"]), torch.tensor(seq["carry0"])
        _, c = orc.network(lay, p, obs[:bi], reset[:bi], c0)
        c = c.detach() if stop_burn_in else c
        q, _ = orc.network(lay, p, obs[bi:], reset[bi:], c)
        L = _torch_loss(q, q, torch.tensor(seq["action"][bi:]), torch.tensor(seq["reward"][bi:]), torch.tensor(seq["done"][bi:]),
                        torch.tensor(prob), n, 0.99, 1000.0, 0.6, stop=stop_targets)
        L.backward()
        return p.grad.numpy()

    np.testing.assert_allclose(g, autograd(True, True), rtol=1e-9, atol=1e-13 * np.abs(g).max())
    if not dueling:
        scale = np.abs(g).max()
        assert np.abs(autograd(False, True) - g).max() > 1e-3 * scale    # gradient through the burn-in would change it
        assert np.abs(autograd(True, False) - g).max() > 1e-3 * scale    # so would gradient through the targets
        return
    vb = lay.off_value + lay.spec_value.ln_bias_slices()[-1].start
    assert np.count_nonzero(g[lay.off_value: lay.param_count]) <= 1 and g[vb] != 0.0   # only the value LayerNorm bias of MLPTorso_0


def _layout(cell: str, dueling: bool, H: int = 256, sizes: int = 256, A: int = 2, D: int = 4):
    from stoix_b200.networks.dueling import DuelingQNetwork
    from stoix_b200.networks.heads import DiscreteQNetworkHead
    from stoix_b200.networks.recurrent import RecurrentActor
    from stoix_b200.networks.torso import MLPTorso
    head = DuelingQNetwork(A, 0.1, [sizes], "relu", True) if dueling else DiscreteQNetworkHead(A, 0.1)
    net = RecurrentActor(head, MLPTorso([sizes], "relu", True), H, cell, MLPTorso([sizes], "relu", True))
    return net.layout_for(D), net


def test_arena_layout_and_flax_names():
    lay, net = _layout("gru", dueling=True)
    tree = net.init(0, torch.zeros(1, 256), (torch.zeros(1, 1, 4), torch.zeros(1, 1, dtype=torch.bool)))
    p = tree["params"]
    assert set(p) == {"pre_torso", "ScannedRNN_0", "post_torso", "action_head"}
    ah = p["action_head"]
    assert set(ah) == {"MLPTorso_0", "MLPTorso_1"}
    for br, out in (("MLPTorso_0", 1), ("MLPTorso_1", 2)):
        assert set(ah[br]) == {"Dense_0", "Dense_1", "LayerNorm_0", "LayerNorm_1"}
        assert set(ah[br]["Dense_1"]) == {"kernel"} and tuple(ah[br]["Dense_1"]["kernel"].shape) == (256, out)
        assert set(ah[br]["LayerNorm_1"]) == {"scale", "bias"} and torch.equal(ah[br]["LayerNorm_1"]["scale"], torch.ones(out))
    assert set(p["post_torso"]) == {"Dense_0", "LayerNorm_0"} and set(p["post_torso"]["Dense_0"]) == {"kernel"}
    # [pre | W_h | b_hn | post-torso + advantage branch | value branch]; every float of the arena is in the tree exactly once
    assert lay.spec_post.sizes == (256, 256, 256, 2) and lay.spec_post.ln_final and lay.spec_value.sizes == (256, 256, 1)
    assert lay.param_count == lay.off_value + lay.spec_value.param_count
    seen = torch.zeros(lay.param_count, dtype=torch.int32)
    base = tree.flat.data_ptr()

    def mark(d):
        for v in d.values():
            if isinstance(v, dict):
                mark(v)
            else:
                o = (v.data_ptr() - base) // 4
                idx = o + torch.as_strided(torch.arange(lay.param_count), v.shape, v.stride()).reshape(-1)
                seen[idx] += 1

    mark(p)
    assert bool((seen == 1).all())
    # orthogonal(sqrt 2) final kernels: columns of norm sqrt 2
    np.testing.assert_allclose(torch.linalg.norm(ah["MLPTorso_1"]["Dense_1"]["kernel"], dim=0).numpy(), np.sqrt(2), rtol=1e-5)
    plain, _ = _layout("lstm", dueling=False)
    assert not plain.dueling and plain.spec_post.sizes == (256, 256, 2) and not plain.spec_post.ln_final and plain.S == 512


def test_ln_final_spec_layout():
    """A final LayerNorm gives the last layer W, scale, bias; the specs every other network uses keep their layout."""
    from stoix_b200.ops import MlpSpec
    a, b = MlpSpec((5, 7, 3), "relu", True), MlpSpec((5, 7, 3), "relu", True, ln_final=True)
    assert a.param_count == 5 * 7 + 2 * 7 + 7 * 3 + 3 and b.param_count == a.param_count + 3
    assert a.ln_bias_slices()[-1] is None and b.ln_bias_slices()[-1] == slice(a.param_count, a.param_count + 3)


def test_configs_match_the_reference():
    from stoix_b200.config import compose
    cfg = compose("default_rec_r2d2", [], config_dir="default/anakin")
    want = {"system_name": "r2d2", "rollout_length": 40, "epochs": 32, "warmup_steps": 128, "total_buffer_size": 100_000, "total_batch_size": 32,
            "burn_in_length": 40, "sample_sequence_length": 80, "period": 40, "priority_exponent": 0.9, "importance_sampling_exponent": 0.6,
            "priority_eta": 0.9, "n_step": 5, "q_lr": 1e-4, "tau": 0.005, "gamma": 0.99, "max_grad_norm": 0.5, "decay_learning_rates": False,
            "training_epsilon": 0.1, "evaluation_epsilon": 0.0, "max_abs_reward": 1000.0}
    assert {k: cfg.system[k] for k in want} == want and set(cfg.system) == set(want)
    net = cfg.network.actor_network
    assert net.rnn_layer.cell_type == "gru" and net.rnn_layer.hidden_state_dim == 256
    assert net.action_head._target_ == "stoix.networks.dueling.DuelingQNetwork" and list(net.action_head.layer_sizes) == [256]
    assert net.action_head.use_layer_norm and net.pre_torso.use_layer_norm and net.post_torso.use_layer_norm
    assert cfg.env.scenario.name == "CartPole-v1" if "scenario" in cfg.env else True
    plain = compose("default_rec_r2d2", ["network=rnn_dqn"], config_dir="default/anakin")
    assert plain.network.actor_network.action_head._target_ == "stoix.networks.heads.DiscreteQNetworkHead"


def test_launch_file():
    import stoix.systems.q_learning.rec_r2d2 as launch
    from stoix_b200.systems.q_learning import rec_r2d2
    assert launch is rec_r2d2 and callable(launch.hydra_entry_point)


@pytest.mark.parametrize("overrides,n_devices,match", [
    ([], 3, "buffer size"), (["system.total_buffer_size=99999"], 3, "batch size"),
    (["system.burn_in_length=80"], 1, "burn-in"), (["system.period=41"], 1, "period"), (["arch.precision=bf16"], 1, "bf16"),
    (["system.total_buffer_size=20480"], 1, "fewer than one sequence"), (["network.actor_network.rnn_layer.cell_type=mgu"], 1, "cell_type"),
    (["network.actor_network.action_head._target_=stoix.networks.heads.CategoricalHead"], 1, "action head"),
    (["network.actor_network.action_head.use_layer_norm=False"], 1, "use_layer_norm=True")])
def test_refusals(overrides, n_devices, match):
    from stoix_b200.config import compose
    from stoix_b200.systems.q_learning.rec_r2d2 import refuse_unsupported
    cfg = compose("default_rec_r2d2", overrides, config_dir="default/anakin")
    with pytest.raises(ValueError, match=match):
        refuse_unsupported(cfg, n_devices=n_devices)


def test_sequence_buffer_refusals():
    from stoix_b200.utils.replay import PrioritisedSequenceBuffer
    with pytest.raises(ValueError, match="fewer than one sequence"):
        PrioritisedSequenceBuffer(100, 4, 80, 4, 40, 0.9, 4, 8, "cpu")
    with pytest.raises(ValueError, match="period"):
        PrioritisedSequenceBuffer(400, 4, 80, 4, 101, 0.9, 4, 8, "cpu")


def test_ring_oracle_rule():
    """The oracle's item rule on a ring whose length is not a multiple of the period, through a wrap."""
    ring = orc.Ring(L=11, E=2, S=4, period=3, alpha=0.9)
    assert ring.K == 3
    z = lambda T: dict(reward=np.zeros((T, 2)), carry=np.zeros((T, 2, 1)))
    ring.add(**z(5))      # rows 0..4 written: items starting at 0 (rows 0-3) valid, at 3 (rows 3-6) not
    assert ring.valid_items() == [0, 3]
    ring.add(**z(8))      # rows 5..12 -> w = 2 after a wrap; row 9 starts no item (K p = 9)
    valid = {i % 3 for i in ring.valid_items()}
    assert valid == {1, 2} and ring.w == 2 and ring.c == 11   # start 0 straddles the head (rows 0, 1 new, age 1)
