"""CPU checks of the distributional Q-learning oracle (tests/distq_oracle.py) and of the host side of ff_c51 / ff_qr_dqn."""
import ctypes

import numpy as np
import pytest
import torch

from tests import distq_oracle as D
from tests.dqn_oracle import LossHyper


def _torch_c51(logits_tm1, logits_t, q_sel, atoms, a, r, d):
    """categorical_double_q_learning written out in torch fp64 (the projection as rlax defines it), for autograd."""
    M, A = q_sel.shape
    N = atoms.shape[-1]
    lt1 = logits_tm1.view(M, A, N)
    rows = torch.arange(M)
    p = torch.softmax(logits_t.view(M, A, N)[rows, q_sel.argmax(-1)], -1)
    z_p = torch.clamp(r[:, None] + d[:, None] * atoms, atoms[0], atoms[-1])[:, :, None]
    d_pos = torch.cat([atoms, atoms[:1]])[1:] - atoms
    d_neg = atoms - torch.cat([atoms[-1:], atoms])[:-1]
    d_pos = torch.where(d_pos > 0, 1.0 / d_pos, torch.zeros_like(d_pos))
    d_neg = torch.where(d_neg > 0, 1.0 / d_neg, torch.zeros_like(d_neg))
    delta = z_p - atoms
    s = (delta >= 0).double()
    dh = s * delta * d_pos - (1 - s) * delta * d_neg
    t = (torch.clamp(1 - dh, 0, 1) * p[:, :, None]).sum(1)
    return -(t * torch.log_softmax(lt1[rows, a], -1)).sum(-1)


def _torch_qr(q_tm1, q_t, tau, a, r, d, A, kappa):
    M = q_t.shape[0]
    N = tau.shape[-1]
    rows = torch.arange(M)
    qt = q_t.view(M, A, N)
    target = r[:, None] + d[:, None] * qt[rows, qt.mean(-1).argmax(-1)]
    delta = target[:, None, :] - q_tm1.view(M, A, N)[rows, a][:, :, None]
    w = torch.abs(tau[None, :, None] - (delta < 0).double())
    if kappa > 0:
        ax = delta.abs()
        quad = torch.clamp(ax, max=kappa)
        rho = 0.5 * quad ** 2 + kappa * (ax - quad)
    else:
        rho = delta.abs()
    return (w * rho).mean(-1).sum(-1)


def test_categorical_gradient_matches_autograd():
    rng = np.random.default_rng(0)
    M, A, N = 40, 3, 11
    atoms = np.linspace(-5, 5, N)
    lt1, lt = rng.normal(size=(M, A * N)), rng.normal(size=(M, A * N))
    q_sel = rng.normal(size=(M, A))
    a, r = rng.integers(0, A, M), rng.normal(size=M) * 2
    d = (rng.random(M) < 0.8) * 0.9
    h = LossHyper(gamma=0.9)
    loss, g, t = D.categorical_loss_and_grad(lt1, lt, q_sel, atoms, atoms, a, r, None, h, discount=d)
    x = torch.tensor(lt1, requires_grad=True)
    want = _torch_c51(x, torch.tensor(lt), torch.tensor(q_sel), torch.tensor(atoms), torch.tensor(a), torch.tensor(r), torch.tensor(d))
    want.mean().backward()
    np.testing.assert_allclose(loss, want.detach().numpy(), rtol=1e-12)
    np.testing.assert_allclose(g, x.grad.numpy(), rtol=1e-10, atol=1e-14)
    np.testing.assert_allclose(t.sum(-1), 1.0, rtol=1e-12)


@pytest.mark.parametrize("kappa", [0.0, 1.0])
def test_quantile_gradient_matches_autograd_away_from_ties(kappa):
    rng = np.random.default_rng(1)
    M, A, N = 30, 4, 9
    tau = (np.arange(N) + 0.5) / N
    q1, qt = rng.normal(size=(M, A * N)) * 2, rng.normal(size=(M, A * N)) * 2
    a, r, d = rng.integers(0, A, M), rng.normal(size=M), rng.random(M)
    h = LossHyper(huber=kappa)
    loss, g = D.quantile_loss_and_grad(q1, qt, None, tau, a, r, None, h, A, discount=d)
    x = torch.tensor(q1, requires_grad=True)
    want = _torch_qr(x, torch.tensor(qt), torch.tensor(tau), torch.tensor(a), torch.tensor(r), torch.tensor(d), A, kappa)
    want.mean().backward()
    np.testing.assert_allclose(loss, want.detach().numpy(), rtol=1e-12)
    np.testing.assert_allclose(g, x.grad.numpy(), rtol=1e-10, atol=1e-14)


def test_quantile_ties_follow_the_jax_convention():
    """delta = 0 exactly: the weight is tau_i (delta_neg = (delta < 0)), the |.| slope is +1 (lax.abs's JVP), the Huber slope 0."""
    N, A = 4, 1
    tau = (np.arange(N) + 0.5) / N
    q = np.full((1, N), 3.0)   # every source quantile equals every target quantile: r = 3, d = 0
    for kappa, slope in ((0.0, 1.0), (1.0, 0.0)):
        loss, g = D.quantile_loss_and_grad(q, q, None, tau, [0], [3.0], None, LossHyper(huber=kappa), A, discount=[0.0])
        assert loss[0] == 0.0
        np.testing.assert_allclose(g[0], -tau * slope)   # -(1/N) sum_j tau_i slope / M with M = 1
    # torch's |.| has slope 0 at 0: the oracle deliberately differs from autograd there
    x = torch.zeros(1, requires_grad=True)
    x.abs().sum().backward()
    assert x.grad.item() == 0.0


def test_projection_mass_and_edge_cases():
    atoms = np.linspace(0.0, 10.0, 11)
    rng = np.random.default_rng(2)
    p = rng.random(11)
    p /= p.sum()
    for shift in (0.0, 3.0, 2.5, -50.0, 50.0, 10.0, -10.0):   # on atoms, between, below vmin, above vmax, at both ends
        t = D.l2_project(atoms + shift, p, atoms)
        np.testing.assert_allclose(t.sum(), 1.0, rtol=1e-12)
        assert (t >= 0).all()
    np.testing.assert_allclose(D.l2_project(atoms, p, atoms), p, rtol=1e-12)           # on the atoms: unchanged
    np.testing.assert_allclose(D.l2_project(atoms + 3.0, p, atoms)[3:-1], p[:-4])      # shifted by three atoms
    assert D.l2_project(atoms - 50.0, p, atoms)[0] == pytest.approx(1.0)               # everything below vmin lands on it
    assert D.l2_project(atoms + 50.0, p, atoms)[-1] == pytest.approx(1.0)              # and above vmax on vmax
    mid = D.l2_project(np.full(11, 2.5), p, atoms)                                     # halfway between atoms 2 and 3
    np.testing.assert_allclose(mid[[2, 3]], [0.5, 0.5])


def test_expected_q_values():
    logits = np.log(np.array([[1.0, 1.0, 2.0, 1.0, 3.0, 0.0 + 1e-300]]))
    np.testing.assert_allclose(D.categorical_q_values(logits, [0.0, 1.0, 2.0], 2), [[0.25 * 1.0 + 0.5 * 2.0, 0.75 * 1.0]], rtol=1e-12)
    np.testing.assert_allclose(D.quantile_q_values(np.arange(6.0)[None], 2), [[1.0, 4.0]])


def test_configs_compose_with_the_reference_values():
    from stoix_b200.config import compose

    want = {"ff_c51": dict(rollout_length=1, epochs=1, warmup_steps=16, total_buffer_size=500_000, total_batch_size=256, q_lr=1e-4, tau=0.005,
                           gamma=0.99, max_grad_norm=0.5, training_epsilon=0.1, evaluation_epsilon=0.0, max_abs_reward=1000.0, num_atoms=51,
                           vmin=0.0, vmax=500.0),
            "ff_qr_dqn": dict(rollout_length=1, epochs=1, warmup_steps=32, total_buffer_size=500_000, total_batch_size=256, q_lr=5e-5, tau=0.005,
                              gamma=0.99, max_grad_norm=0.5, training_epsilon=0.1, evaluation_epsilon=0.0, max_abs_reward=1000.0,
                              huber_loss_parameter=1.0, num_quantiles=200)}
    heads = {"ff_c51": ("DistributionalDiscreteQNetwork", dict(vmin=0.0, vmax=500.0, num_atoms=51)),
             "ff_qr_dqn": ("QuantileDiscreteQNetwork", dict(num_quantiles=200))}
    for name, kv in want.items():
        cfg = compose(f"default_{name}", [], config_dir="default/anakin")
        assert cfg.system.system_name == name
        for k, v in kv.items():
            assert float(cfg.system[k]) == pytest.approx(float(v), rel=1e-12), (name, k)
        net = cfg.network.actor_network
        assert list(net.pre_torso.layer_sizes) == [256, 256] and net.pre_torso.activation == "silu" and not net.pre_torso.use_layer_norm
        assert net.action_head._target_ == f"stoix.networks.heads.{heads[name][0]}"
        for k, v in heads[name][1].items():
            assert float(net.action_head[k]) == v, (name, k)
        assert "cartpole" in str(cfg.env).lower()


@pytest.mark.parametrize("name,loss", [("ff_c51", "categorical_double_q_learning"), ("ff_qr_dqn", "quantile_q_learning")])
def test_launch_files_resolve_to_the_implementation(name, loss):
    import importlib

    launch = importlib.import_module(f"stoix.systems.q_learning.{name}")
    impl = importlib.import_module(f"stoix_b200.systems.q_learning.{name}")
    assert launch is impl and impl.LOSS == loss
    for fn in ("get_warmup_fn", "get_learner_fn", "learner_setup", "run_experiment", "hydra_entry_point"):
        assert callable(getattr(impl, fn))

    class Net:
        def apply(self, params, x):
            return ("greedy", params, x)

    assert impl.EvalActorWrapper(Net()).apply(1, 2) == "greedy"


def test_head_widths_and_lecun_normal_init():
    from stoix_b200.networks.base import FeedForwardActor, _lecun_normal
    from stoix_b200.networks.heads import DistributionalDiscreteQNetwork, QuantileDiscreteQNetwork, linspace_f32
    from stoix_b200.networks.torso import MLPTorso

    c51 = DistributionalDiscreteQNetwork(action_dim=4, epsilon=0.1, num_atoms=51, vmin=0.0, vmax=500.0)
    qr = QuantileDiscreteQNetwork(action_dim=8, epsilon=0.1, num_quantiles=200)
    assert c51.out_dim == 204 and qr.out_dim == 1600
    assert c51.atoms_host.dtype == np.float32 and c51.atoms_host[0] == 0.0 and c51.atoms_host[-1] == 500.0
    np.testing.assert_array_equal(c51.atoms_host, linspace_f32(0.0, 500.0, 51))
    np.testing.assert_allclose(c51.atoms_host, np.linspace(0.0, 500.0, 51), rtol=1e-6)
    gen = torch.Generator().manual_seed(0)
    n_in, n_out = 256, 1600
    w = _lecun_normal(gen, n_in, n_out, 1.0).double()
    std = np.sqrt(1.0 / n_in) / 0.87962566103423978
    assert w.abs().max().item() <= 2.0 * std * (1 + 1e-6)
    assert w.var().item() == pytest.approx(1.0 / n_in, rel=0.02)   # variance_scaling(1, fan_in): Var = 1 / fan_in
    # the head's kernel is lecun_normal, the torso's stays orthogonal
    net = FeedForwardActor(action_head=qr, torso=MLPTorso(layer_sizes=[64, 64], activation="silu", use_layer_norm=False))
    tree = net.init(3, torch.zeros(1, 10))
    head = tree["params"]["action_head"]["Dense_0"]["kernel"].double()
    assert tuple(head.shape) == (64, 1600) and head.abs().max().item() <= 2.0 * np.sqrt(1 / 64) / 0.87962566103423978 * (1 + 1e-6)
    k0 = tree["params"]["torso"]["Dense_0"]["kernel"].double()
    gram = (k0 @ k0.t()).numpy()   # orthogonal(scale): n_in = 10 < 64, so the rows are orthogonal with equal norms
    np.testing.assert_allclose(gram, gram[0, 0] * np.eye(10), atol=1e-5)


def test_new_struct_layout_matches_c(tmp_path):
    import os
    import shutil
    import subprocess

    from stoix_b200 import _lib, ops

    cc = shutil.which("cc") or shutil.which("gcc")
    assert cc, "a C compiler is needed to read the C layouts (the CUDA build needs one too)"
    cls = _lib.StxDistQHyper
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "stx.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(StxDistQHyper));']
    lines += [f'  printf("{f} %zu\\n", offsetof(StxDistQHyper, {f}));' for f, _ in cls._fields_]
    lines += ['  printf("categorical %d\\n", (int)STX_DIST_CATEGORICAL);', '  printf("quantile %d\\n", (int)STX_DIST_QUANTILE);',
              '  printf("max_n %d\\n", (int)STX_DIST_MAX_N);', "  return 0;\n}"]
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text("\n".join(lines))
    include = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    subprocess.run([cc, "-std=c11", "-I", include, str(src), "-o", str(exe)], check=True, capture_output=True, text=True)
    got = dict((a, int(b)) for a, b in (l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines()))
    assert got["size"] == ctypes.sizeof(cls)
    for f, _ in cls._fields_:
        assert got[f] == getattr(cls, f).offset, f
    assert got["categorical"] == ops.DIST_KINDS["categorical"] and got["quantile"] == ops.DIST_KINDS["quantile"]
    assert got["max_n"] == ops.DIST_MAX_N


def test_loss_faces_refuse_actions_outside_the_rows():
    from stoix_b200 import ops
    from stoix_b200.utils import loss as L

    M, A, N = 3, 2, 5
    lg, at, r, d = torch.zeros(M, A, N), torch.zeros(M, N), torch.zeros(M), torch.ones(M)
    dist, tau = torch.zeros(M, N, A), torch.zeros(M, N)
    for a in (torch.tensor([0, 2, 1]), torch.tensor([-1, 0, 1])):
        with pytest.raises(ops.StxError, match="a_tm1"):
            L.categorical_double_q_learning(lg, at, a, r, d, lg, at, torch.zeros(M, A))
        with pytest.raises(ops.StxError, match="a_tm1"):
            L.quantile_q_learning(dist, tau, a, r, d, dist, dist, 1.0)


def test_heads_and_losses_are_matched_on_the_host():
    from stoix_b200.config import compose
    from stoix_b200.systems.q_learning import ff_dqn

    for name, loss in (("ff_c51", "categorical_double_q_learning"), ("ff_qr_dqn", "quantile_q_learning")):
        cfg = compose(f"default_{name}", [], config_dir="default/anakin")
        ff_dqn._refuse_unsupported(cfg, loss)   # its own head: accepted
        with pytest.raises(ValueError, match=name):   # a distributional head under a scalar loss names its system
            ff_dqn._refuse_unsupported(cfg)
        with pytest.raises(ValueError, match="bf16"):
            ff_dqn._refuse_unsupported(compose(f"default_{name}", ["arch.precision=bf16"], config_dir="default/anakin"), loss)
        plain = compose("default_ff_dqn", [], config_dir="default/anakin")
        with pytest.raises(ValueError, match="not implemented"):   # the plain head under a distributional loss
            ff_dqn._refuse_unsupported(plain, loss)
    c51 = compose("default_ff_c51", [], config_dir="default/anakin")
    with pytest.raises(ValueError, match="ff_qr_dqn"):   # the other distributional head
        ff_dqn._refuse_unsupported(c51, "quantile_q_learning")
    assert set(ff_dqn.LOSSES) >= {"categorical_double_q_learning", "quantile_q_learning"}
