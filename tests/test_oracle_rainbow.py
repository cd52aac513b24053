"""CPU checks of Rainbow (ff_rainbow): the oracle (tests/rainbow_oracle.py) against torch autograd of the reference formulas, the
buffer rules on hand-built cases, the parameter layout, the configs and launch files, and the ctypes structs against include/stx.h."""
from __future__ import annotations

import ctypes
import importlib

import numpy as np
import pytest
import torch

from tests import rainbow_oracle as R


def _layout(D=5, torso=(6, 7), branch=(8,), A=3, N=4):
    from stoix_b200.networks.dueling import NoisyDistributionalDuelingQNetwork, NoisyLayout
    from stoix_b200.networks.torso import NoisyMLPTorso

    head = NoisyDistributionalDuelingQNetwork(A, 0.0, list(branch), 0.25, num_atoms=N, vmin=0.0, vmax=10.0, activation="silu")
    return NoisyLayout(D, NoisyMLPTorso(list(torso), "silu", sigma_zero=0.25), head), head


@pytest.mark.parametrize("branch", [(8,), (8, 5), ()])
def test_effective_forward_and_fold_match_autograd(branch):
    """The effective arena run as the block MLP equals the reference network, and fold(d effective) equals autograd's (d mu, d sigma)
    under the same noise, through the dueling combine."""
    lay, head = _layout(branch=branch)
    A, N = head.action_dim, head.num_atoms
    rng = np.random.default_rng(len(branch))
    params = rng.normal(size=lay.param_count).astype(np.float32) * 0.5
    nz = rng.normal(size=lay.noise_count).astype(np.float32)
    x = rng.normal(size=(6, 5))
    # the effective arena, run as the StxMlp chain
    eff = R.effective(lay.layers, params, nz, lay.eff_count, np.float64)
    sizes, sl = lay.spec.sizes, lay.spec.layer_slices()
    h = x
    for i in range(len(sizes) - 1):
        h = h @ eff[sl[i][0]].reshape(sizes[i], sizes[i + 1]) + eff[sl[i][1]]
        if i < len(sizes) - 2:
            h = R._silu(h)
    want = R.noisy_forward64(lay.layers, params, nz, x, 2, len(branch))
    np.testing.assert_allclose(h, want, rtol=1e-5, atol=1e-5)
    # autograd of the reference formula: q_logits -> a weighted sum
    p = torch.tensor(params.astype(np.float64), requires_grad=True)
    nzt = torch.tensor(nz.astype(np.float64))
    cot = rng.normal(size=(6, A * N))

    def lin(L, hh):
        n_in, n_out, o = L["in_"], L["out"], L["param"]
        W = n_in * n_out
        mu_w, mu_b = p[o:o + W].view(n_in, n_out), p[o + W:o + W + n_out]
        sg_w, sg_b = p[o + W + n_out:o + 2 * W + n_out].view(n_in, n_out), p[o + 2 * W + n_out:o + 2 * W + 2 * n_out]
        fin, fout = nzt[L["noise"]:L["noise"] + n_in], nzt[L["noise"] + n_in:L["noise"] + n_in + n_out]
        return hh @ (mu_w + sg_w * torch.outer(fin, fout)) + mu_b + sg_b * fout

    hh = torch.tensor(x)
    for L in lay.layers[:2]:
        hh = torch.nn.functional.silu(lin(L, hh))
    br = []
    for b in range(2):
        hb = hh
        for L in lay.layers[2 + b * len(branch): 2 + (b + 1) * len(branch)]:
            hb = torch.nn.functional.silu(lin(L, hb))
        br.append(hb)
    v, adv = lin(lay.layers[-2], br[0]).view(-1, 1, N), lin(lay.layers[-1], br[1]).view(-1, A, N)
    q = (v + adv - adv.mean(1, keepdim=True)).reshape(-1, A * N)
    np.testing.assert_allclose(q.detach().numpy(), R.dueling_combine(want, A, N), rtol=1e-9)
    (q * torch.tensor(cot)).sum().backward()
    # the same gradient by the kernels' route: dueling backward, the block MLP's backward on the effective arena, then fold
    e = torch.tensor(eff, requires_grad=True)
    hh = torch.tensor(x)
    for i in range(len(sizes) - 1):
        hh = hh @ e[sl[i][0]].view(sizes[i], sizes[i + 1]) + e[sl[i][1]]
        if i < len(sizes) - 2:
            hh = torch.nn.functional.silu(hh)
    (hh * torch.tensor(R.dueling_backward(cot, A, N))).sum().backward()
    g = np.zeros(lay.param_count)
    for L in lay.layers:   # fold in float64
        n_in, n_out, o = L["in_"], L["out"], L["param"]
        W = n_in * n_out
        fin, fout = R._f(L, nz.astype(np.float64))
        ge = e.grad.numpy()
        gw = np.stack([ge[L["eff_w"] + r * L["ld"]: L["eff_w"] + r * L["ld"] + n_out] for r in range(n_in)])
        gb = ge[L["eff_b"]: L["eff_b"] + n_out]
        g[o:o + W], g[o + W:o + W + n_out] = gw.reshape(-1), gb
        g[o + W + n_out:o + 2 * W + n_out], g[o + 2 * W + n_out:o + 2 * W + 2 * n_out] = (gw * np.outer(fin, fout)).reshape(-1), gb * fout
    np.testing.assert_allclose(g, p.grad.numpy(), rtol=1e-9, atol=1e-12)
    # and the fp32 fold mirror agrees with it
    np.testing.assert_allclose(R.fold(lay.layers, e.grad.numpy().astype(np.float32), nz, lay.param_count), g, rtol=1e-5, atol=1e-6)


def test_dueling_backward_matches_autograd():
    rng = np.random.default_rng(3)
    A, N = 5, 7
    head = torch.tensor(rng.normal(size=(4, N + A * N)), requires_grad=True)
    v, adv = head[:, None, :N], head[:, N:].view(-1, A, N)
    q = (v + adv - adv.mean(1, keepdim=True)).reshape(-1, A * N)
    cot = rng.normal(size=q.shape)
    (q * torch.tensor(cot)).sum().backward()
    np.testing.assert_allclose(R.dueling_combine(head.detach().numpy(), A, N), q.detach().numpy(), rtol=1e-12)
    np.testing.assert_allclose(R.dueling_backward(cot, A, N), head.grad.numpy(), rtol=1e-12, atol=1e-12)


def test_n_step_return_is_the_discounted_sum_cut_at_done():
    """batch_discounted_returns(r, (1 - done) gamma, 0)[:, 0] written as a backward scan, against the forward sum."""
    rng = np.random.default_rng(4)
    for _ in range(50):
        n = int(rng.integers(1, 7))
        r, d = rng.normal(size=n), (rng.random(n) < 0.3).astype(np.uint8)
        g = torch.zeros((), dtype=torch.float64)
        for k in reversed(range(n)):
            g = torch.tensor(r[k]) + (1.0 - d[k]) * 0.9 * g
        assert R.n_step_return(r, d, 0.9) == pytest.approx(float(g), rel=1e-12, abs=1e-12)
        assert float(R.n_step_return32(r.astype(np.float32), d, 0.9)) == pytest.approx(float(g), rel=1e-5, abs=1e-5)
    assert R.n_step_return(np.array([1.0, 2.0, 4.0]), np.array([0, 1, 0]), 0.5) == 1.0 + 0.5 * 2.0   # cut after the done step


def test_weighted_loss_gradient_matches_autograd():
    """d mean(w loss) / d logits_tm1 = w_i (softmax sum t - t) / M, the projected target held fixed (rlax stops its gradient)."""
    from tests import distq_oracle as DQ
    from tests.dqn_oracle import LossHyper

    rng = np.random.default_rng(5)
    M, A, N = 6, 3, 11
    atoms = np.linspace(-5.0, 5.0, N)
    lt1, lt, q_sel = rng.normal(size=(M, A * N)), rng.normal(size=(M, A * N)), rng.normal(size=(M, A))
    a, r, done = rng.integers(0, A, M), rng.normal(size=M), (rng.random(M) < 0.3).astype(np.uint8)
    w = rng.random(M)
    loss, g, t = DQ.categorical_loss_and_grad(lt1, lt, q_sel, atoms, atoms, a, r, done, LossHyper(gamma=0.9, max_abs_reward=3.0))
    x = torch.tensor(lt1, requires_grad=True)
    la = x.view(M, A, N)[torch.arange(M), torch.tensor(a)]
    per_row = -(torch.tensor(t) * torch.log_softmax(la, -1)).sum(-1)
    np.testing.assert_allclose(per_row.detach().numpy(), loss, rtol=1e-12)
    (torch.tensor(w) * per_row).mean().backward()
    np.testing.assert_allclose(g * w[:, None], x.grad.numpy(), rtol=1e-10, atol=1e-14)


def test_importance_weights_and_beta_schedule():
    p = np.array([0.5, 0.25, 0.125, 0.125])
    np.testing.assert_allclose(R.importance_weights(p, 1.0), [0.25, 0.5, 1.0, 1.0])
    np.testing.assert_allclose(R.importance_weights(p, 0.0), 1.0)
    assert R.beta_at(0, 0.4, 100) == pytest.approx(0.4) and R.beta_at(50, 0.4, 100) == pytest.approx(0.7)
    assert R.beta_at(1000, 0.4, 100) == 1.0 and R.beta_at(7, 0.4, 0) == 0.4
    # the normalised weight does not depend on the total
    np.testing.assert_allclose(R.importance_weights(p * 3.0, 0.6), R.importance_weights(p, 0.6))


def _fill(ring: R.PrioRing, T: int, base: float):
    E, D = ring.E, ring.D
    obs = (base + np.arange(T * E * D, dtype=np.float32)).reshape(T, E, D)
    return obs, np.full((T, E), int(base) % 3, np.int32), np.full((T, E), base, np.float32), np.zeros((T, E), np.uint8), obs + 0.5


def test_buffer_validity_on_add_across_the_wrap():
    """L = 6, n = 3: valid items are those whose 3 rows are written and do not straddle the write head; an add re-prices the items it
    touched with the max priority and zeroes the ones it broke."""
    ring = R.PrioRing(6, 2, 1, 3, 1.0)
    ring.add(*_fill(ring, 2, 0.0))
    assert ring.prio.sum() == 0.0                      # two rows: no sequence of three yet
    ring.add(*_fill(ring, 2, 10.0))                    # rows 0..3 written, head at 4
    valid = [p for p in range(6) if ring.prio[p] > 0]
    assert valid == [0, 1] and ring.prio[6:].tolist() == ring.prio[:6].tolist()
    ring.set_priorities([0, 1], np.array([4.0, 2.0]))
    ring.add(*_fill(ring, 3, 20.0))                    # rows 4, 5, 0 overwritten, head at 1
    # valid starts: ages >= 2 -> p in {1, 2, 3, 4}... with c = 6: age(p) = (0 - p) mod 6
    assert [p for p in range(6) if ring.prio[p] > 0] == [1, 2, 3, 4]
    assert ring.prio[1] == 2.0                         # rows 1, 2, 3: untouched, keeps its priority
    assert ring.prio[2] == ring.prio[3] == ring.prio[4] == 4.0   # touched by the add: max priority (4 ** 1)
    assert ring.prio[0] == 0.0 and ring.prio[5] == 0.0  # straddles the head / incomplete


def test_buffer_sampling_and_set_priorities_rules():
    ring = R.PrioRing(4, 1, 1, 1, 0.5)
    ring.add(*_fill(ring, 4, 1.0))
    ring.set_priorities([0, 1, 2, 3, 1], np.array([1.0, 4.0, 16.0, 9.0, 25.0]))   # duplicate 1: the last (25) wins
    np.testing.assert_allclose(ring.prio, [1.0, 5.0, 4.0, 3.0])
    assert ring.maxp == 5.0
    # stratified: slice r of 4 of the total 13
    np.testing.assert_array_equal(ring.sample(np.array([0.0, 0.5, 0.5, 0.99])), [0, 1, 2, 3])
    ring.set_priorities([2], np.array([0.0]))
    assert 2 not in ring.sample(np.linspace(0.01, 0.99, 4))


def test_tree_size():
    assert R.tree_floats(1) == 1 and R.tree_floats(32) == 33 and R.tree_floats(33) == 33 + 2 + 1
    assert R.tree_floats(10**6) == 10**6 + 31250 + 977 + 31 + 1


def test_parameter_layout_follows_the_flax_tree():
    lay, head = _layout(D=4, torso=(256, 256), branch=(512,), A=2, N=51)
    names = ["/".join(L["path"]) for L in lay.layers]
    assert names == ["torso/NoisyLinear_0", "torso/NoisyLinear_1", "action_head/NoisyMLPTorso_0/NoisyLinear_0", "action_head/NoisyMLPTorso_1/NoisyLinear_0",
                     "action_head/NoisyLinear_0", "action_head/NoisyLinear_1"]
    assert lay.spec.sizes == (4, 256, 256, 1024, 51 + 2 * 51) and lay.spec.activation == "silu"
    per = [2 * L["in_"] * L["out"] + 2 * L["out"] for L in lay.layers]
    assert lay.param_count == sum(per) and [L["param"] for L in lay.layers] == list(np.cumsum([0] + per[:-1]))
    # the blocks the layers write never overlap, and the off-diagonal blocks of the output layer are not written
    cover = np.zeros(lay.eff_count, np.int32)
    for L in lay.layers:
        for r in range(L["in_"]):
            cover[L["eff_w"] + r * L["ld"]: L["eff_w"] + r * L["ld"] + L["out"]] += 1
        cover[L["eff_b"]: L["eff_b"] + L["out"]] += 1
    assert cover.max() == 1
    out_w = lay.spec.layer_slices()[3][0]
    blk = cover[out_w].reshape(1024, 153)
    assert blk[:512, :51].all() and blk[512:, 51:].all() and not blk[:512, 51:].any() and not blk[512:, :51].any()


def test_init_values():
    """sigma = sigma_zero / sqrt(fan_in) with the owning module's sigma_zero: the torso's and the output layers' 0.25, and the branches'
    0.5 (the reference's branches receive sigma_zero in the kernel_init slot and keep NoisyMLPTorso's default)."""
    from stoix_b200.networks.dueling import NoisyFeedForwardActor
    from stoix_b200.networks.torso import NoisyMLPTorso

    lay, head = _layout(D=4, torso=(64,), branch=(32,), A=2, N=5)
    net = NoisyFeedForwardActor(head, NoisyMLPTorso([64], "silu", sigma_zero=0.25))
    tree = net.init(7, torch.zeros(1, 4, dtype=torch.float32))
    sig = lambda s0, n_in: float(np.float32(s0) / np.sqrt(np.float32(n_in)))
    l0 = tree["params"]["torso"]["NoisyLinear_0"]
    assert torch.all(l0["bias"] == 0) and torch.all(l0["sigma_w"] == sig(0.25, 4)) and torch.all(l0["sigma_b"] == sig(0.25, 4))
    for b in ("NoisyMLPTorso_0", "NoisyMLPTorso_1"):
        br = tree["params"]["action_head"][b]["NoisyLinear_0"]
        assert torch.all(br["sigma_w"] == sig(0.5, 64)) and torch.all(br["sigma_b"] == sig(0.5, 64)) and torch.all(br["bias"] == 0)
    assert head.branch.sigma_zero == 0.5 and head.sigma_zero == 0.25
    for name, cols in (("NoisyLinear_0", 5), ("NoisyLinear_1", 10)):
        out = tree["params"]["action_head"][name]
        assert out["kernel"].shape == (32, cols) and torch.all(out["sigma_w"] == sig(0.25, 32)) and torch.all(out["sigma_b"] == sig(0.25, 32))
        assert float(out["kernel"].abs().max()) <= 2.0 * np.sqrt(1.0 / 32) / 0.87962566103423978 + 1e-6   # truncated lecun_normal


def test_configs_carry_the_reference_values():
    from stoix_b200.config import compose

    cfg = compose("default_ff_rainbow", [], config_dir="default/anakin")
    s = cfg.system
    want = dict(system_name="ff_rainbow", rollout_length=4, epochs=128, warmup_steps=16, total_buffer_size=1_000_000, total_batch_size=512,
                priority_exponent=0.5, importance_sampling_exponent=0.4, n_step=5, q_lr=6.25e-5, tau=0.005, gamma=0.99, max_grad_norm=0.5,
                decay_learning_rates=False, training_epsilon=0.0, evaluation_epsilon=0.0, max_abs_reward=1000.0, num_atoms=51, vmin=0.0, vmax=500.0,
                sigma_zero=0.25)
    for k, v in want.items():
        assert s[k] == v, k
    net = cfg.network.actor_network
    assert net.pre_torso._target_ == "stoix.networks.torso.NoisyMLPTorso" and list(net.pre_torso.layer_sizes) == [256, 256]
    assert net.action_head._target_ == "stoix.networks.dueling.NoisyDistributionalDuelingQNetwork" and list(net.action_head.layer_sizes) == [512]
    assert net.pre_torso.activation == net.action_head.activation == "silu"


def test_launch_file_is_the_implementation():
    mod = importlib.import_module("stoix.systems.q_learning.ff_rainbow")
    impl = importlib.import_module("stoix_b200.systems.q_learning.ff_rainbow")
    assert mod is impl
    for name in ("get_warmup_fn", "get_learner_fn", "learner_setup", "run_experiment", "hydra_entry_point"):
        assert callable(getattr(impl, name))


@pytest.mark.parametrize("override, match", [(["arch.precision=bf16"], "bf16"), (["network=mlp_c51"], "not implemented"),
                                             (["network.actor_network.pre_torso.use_layer_norm=True"], "use_layer_norm"),
                                             (["network.actor_network.action_head.use_layer_norm=True"], "use_layer_norm")])
def test_refusals_on_the_host(override, match):
    from stoix_b200.config import compose
    from stoix_b200.systems.q_learning import ff_rainbow

    cfg = compose("default_ff_rainbow", override, config_dir="default/anakin")
    with pytest.raises(ValueError, match=match):
        ff_rainbow._refuse_unsupported(cfg)


def test_rainbow_struct_layouts_match_c(tmp_path):
    import os
    import shutil
    import subprocess

    from stoix_b200 import _lib

    cc = shutil.which("cc") or shutil.which("gcc")
    assert cc, "a C compiler is needed to read the C layouts (the CUDA build needs one too)"
    structs = {"StxNoisyLayer": _lib.StxNoisyLayer, "StxNoisyNet": _lib.StxNoisyNet, "StxReplayPrioritised": _lib.StxReplayPrioritised}
    c_name = lambda f: "in" if f == "in_" else f
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "stx.h"', "int main(void) {"]
    for name, cls in structs.items():
        lines.append(f'  printf("{name} size %zu\\n", sizeof({name}));')
        for field, _ in cls._fields_:
            lines.append(f'  printf("{name} {field} %zu\\n", offsetof({name}, {c_name(field)}));')
    lines += ['  printf("const max_layers %d\\n", STX_NOISY_MAX_LAYERS);', '  printf("const fanout %d\\n", STX_PRIO_FANOUT);', "  return 0;\n}"]
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text("\n".join(lines))
    include = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    subprocess.run([cc, "-std=c11", "-I", include, str(src), "-o", str(exe)], check=True, capture_output=True, text=True)
    got = {}
    for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines():
        a, b, v = line.split()
        got[(a, b)] = int(v)
    for name, cls in structs.items():
        assert got[(name, "size")] == ctypes.sizeof(cls), name
        for field, _ in cls._fields_:
            assert got[(name, field)] == getattr(cls, field).offset, (name, field)
    assert got[("const", "max_layers")] == _lib.STX_NOISY_MAX_LAYERS and got[("const", "fanout")] == _lib.STX_PRIO_FANOUT
