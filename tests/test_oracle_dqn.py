"""CPU checks of the DQN-family oracle (tests/dqn_oracle.py) against autograd of the reference formulas, of the discrete ring
oracle, and of the four configurations, launch files and C struct layouts."""
import ctypes

import numpy as np
import pytest
import torch

from tests import dqn_oracle as Q

RULES = ["q_learning", "double_q_learning", "munchausen_q_learning", "q_learning_reg"]


def _autograd_loss(rule, q_tm1, q_t, q_aux, a, reward, done, h: Q.LossHyper):
    """The reference's _q_loss_fn restated literally in torch (ff_dqn.py:156-176, utils/loss.py:106-223), float64."""
    q_tm1 = torch.tensor(q_tm1, dtype=torch.float64, requires_grad=True)
    q_t = torch.tensor(q_t, dtype=torch.float64)
    at = torch.tensor(a)
    discount = 1.0 - torch.tensor(done, dtype=torch.float64)
    d_t = discount * h.gamma
    r_t = torch.clamp(torch.tensor(reward, dtype=torch.float64), -h.max_abs_reward, h.max_abs_reward)
    idx = torch.arange(len(a))
    if rule in ("q_learning", "q_learning_reg"):
        target = r_t + d_t * q_t.max(-1).values
    elif rule == "double_q_learning":
        target = r_t + d_t * q_t[idx, torch.tensor(q_aux).argmax(-1)]
    else:
        qa_t = torch.tensor(q_aux, dtype=torch.float64)
        m = h.tau * torch.log_softmax(qa_t / h.tau, dim=-1)
        m_a = torch.clamp((torch.nn.functional.one_hot(at, q_tm1.shape[-1]) * m).sum(-1), min=h.clip_value_min, max=0.0)
        next_v = h.tau * torch.logsumexp(q_t / h.tau, dim=-1)
        target = r_t + h.alpha * m_a + d_t * next_v
    td = target.detach() - q_tm1[idx, at]
    if h.huber > 0:   # rlax.huber_loss
        ax = td.abs()
        quad = torch.clamp(ax, max=h.huber)
        loss = (0.5 * quad ** 2 + h.huber * (ax - quad)).mean()
    else:             # rlax.l2_loss
        loss = (0.5 * td ** 2).mean()
    if rule == "q_learning_reg":
        loss = h.reg * q_tm1[idx, at].mean() + loss
    loss.backward()
    return float(loss.detach()), q_tm1.grad.numpy()


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("huber", [0.0, 1.0])
def test_loss_gradient_matches_autograd(rule, huber):
    rng = np.random.default_rng(RULES.index(rule) * 10 + int(huber))
    M, A = 64, 5
    h = Q.LossHyper(gamma=0.97, max_abs_reward=2.0, huber=huber, tau=0.03, alpha=0.9, clip_value_min=-1e3, reg=0.1)
    q_tm1 = rng.normal(size=(M, A))
    q_t = rng.normal(size=(M, A))
    q_aux = rng.normal(size=(M, A))
    if rule == "munchausen_q_learning":   # |q / tau| ~ 1e3, and clip_value_min active on some rows
        q_t, q_aux = q_t * 30.0, q_aux * 30.0
        h.clip_value_min = -20.0
    a = rng.integers(0, A, size=M)
    reward = rng.normal(size=M) * 3.0      # a third of the rows clipped
    done = (rng.random(M) < 0.2).astype(np.uint8)
    want_loss, want_dq = _autograd_loss(rule, q_tm1, q_t, q_aux, a, reward, done, h)
    loss, dq = Q.loss_and_dq(rule, q_tm1, q_t, q_aux, a, reward, done, h)
    assert abs(loss - want_loss) <= 1e-12 * max(1.0, abs(want_loss))
    np.testing.assert_allclose(dq, want_dq, rtol=1e-12, atol=1e-15)
    assert (np.abs(reward) > h.max_abs_reward).any() and done.any()
    if rule == "munchausen_q_learning":
        z = q_aux / h.tau
        log_pi = h.tau * (z - z.max(-1, keepdims=True) - np.log(np.exp(z - z.max(-1, keepdims=True)).sum(-1, keepdims=True)))
        assert (log_pi[np.arange(M), a] < h.clip_value_min).any()


def test_double_q_takes_the_first_maximal_selector():
    h = Q.LossHyper(gamma=1.0)
    q_t = np.array([[1.0, 2.0, 3.0]])
    sel = np.array([[5.0, 5.0, 1.0]])
    loss, dq = Q.loss_and_dq("double_q_learning", np.zeros((1, 3)), q_t, sel, np.array([2]), np.zeros(1), np.zeros(1, np.uint8), h)
    assert dq[0, 2] == -1.0 and loss == 0.5


def test_ring_oracle_keeps_the_newest_rows():
    ring = Q.Ring(5, 1)
    for start, n in ((0, 3), (3, 4), (7, 9)):
        v = np.arange(start, start + n, dtype=np.float32)
        ring.add(v[:, None], v.astype(np.int32), v, np.zeros(n, np.uint8), v[:, None] + 0.5)
    assert ring.size == 5 and ring.pos == (16 % 5)
    assert sorted(ring.reward.tolist()) == [11.0, 12.0, 13.0, 14.0, 15.0]
    assert ring.reward[(15) % 5] == 15.0
    j = Q.uniform_indices(1001, 7, 123, 4)
    assert j.min() >= 0 and j.max() < 7 and len(np.unique(j)) == 7


def test_configs_compose_with_the_reference_values():
    from stoix_b200.config import compose

    want = {
        "default_ff_dqn": dict(system_name="ff_dqn", rollout_length=2, epochs=16, warmup_steps=16, total_buffer_size=1_000_000, total_batch_size=512,
                               q_lr=5e-4, tau=0.005, gamma=0.99, max_grad_norm=0.5, training_epsilon=0.1, evaluation_epsilon=0.0,
                               max_abs_reward=1000.0, huber_loss_parameter=0.0),
        "default_ff_mdqn": dict(system_name="ff_mdqn", rollout_length=1, epochs=1, warmup_steps=16, total_buffer_size=500_000, total_batch_size=256,
                                q_lr=1e-4, tau=0.005, huber_loss_parameter=1.0, entropy_temperature=0.03, munchausen_coefficient=0.9,
                                clip_value_min=-1e3),
        "default_ff_dqn_reg": dict(system_name="ff_dqn_reg", rollout_length=1, epochs=1, total_buffer_size=50_000, total_batch_size=256, q_lr=1e-5,
                                   huber_loss_parameter=1.0, regularizer_coeff=0.1),
    }
    want["default_ff_ddqn"] = want["default_ff_dqn"]   # the reference's default_ff_ddqn composes system: q_learning/ff_dqn
    for name, kv in want.items():
        cfg = compose(name, [], config_dir="default/anakin")
        for k, v in kv.items():
            got = cfg.system[k]
            assert (got == v) if isinstance(v, str) else float(got) == pytest.approx(float(v), rel=1e-12), (name, k, got, v)
        assert cfg.system.decay_learning_rates is False or str(cfg.system.decay_learning_rates) == "False"
        assert cfg.network.actor_network.action_head._target_ == "stoix.networks.heads.DiscreteQNetworkHead"
        assert cfg.env.env_name.lower().startswith("cartpole") or "cartpole" in str(cfg.env).lower()


@pytest.mark.parametrize("name,loss", [("ff_dqn", "q_learning"), ("ff_ddqn", "double_q_learning"), ("ff_mdqn", "munchausen_q_learning"),
                                       ("ff_dqn_reg", "q_learning_reg")])
def test_launch_files_resolve_to_the_implementation(name, loss):
    import importlib

    launch = importlib.import_module(f"stoix.systems.q_learning.{name}")
    impl = importlib.import_module(f"stoix_b200.systems.q_learning.{name}")
    assert launch is impl
    assert getattr(impl, "LOSS", "q_learning") == loss
    for fn in ("get_warmup_fn", "get_learner_fn", "learner_setup", "run_experiment", "hydra_entry_point"):
        assert callable(getattr(impl, fn))


def test_bf16_and_dueling_heads_are_refused_on_the_host():
    from stoix_b200.config import compose
    from stoix_b200.systems.q_learning import ff_dqn

    with pytest.raises(ValueError, match="bf16"):
        ff_dqn._refuse_unsupported(compose("default_ff_dqn", ["arch.precision=bf16"], config_dir="default/anakin"))
    cfg = compose("default_ff_dqn", [], config_dir="default/anakin")
    cfg.network.actor_network.action_head._target_ = "stoix.networks.heads.DuelingQNetworkHead"
    with pytest.raises(ValueError, match="not implemented"):
        ff_dqn._refuse_unsupported(cfg)


def test_new_struct_layouts_match_c(tmp_path):
    """Size and every field offset of the ctypes structs against what the C compiler makes of include/stx.h, and the STX_Q_* rule
    numbers against ops.Q_RULES."""
    import os
    import shutil
    import subprocess

    from stoix_b200 import _lib, ops

    cc = shutil.which("cc") or shutil.which("gcc")
    assert cc, "a C compiler is needed to read the C layouts (the CUDA build needs one too)"
    structs = {"StxReplayDiscrete": _lib.StxReplayDiscrete, "StxQTdHyper": _lib.StxQTdHyper}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "stx.h"', "int main(void) {"]
    for name, cls in structs.items():
        lines.append(f'  printf("{name} size %zu\\n", sizeof({name}));')
        for field, _ in cls._fields_:
            lines.append(f'  printf("{name} {field} %zu\\n", offsetof({name}, {field}));')
    lines += [f'  printf("rule {k} %d\\n", (int){c});' for k, c in (("q_learning", "STX_Q_DQN"), ("double_q_learning", "STX_Q_DOUBLE"),
                                                                    ("munchausen_q_learning", "STX_Q_MUNCHAUSEN"), ("q_learning_reg", "STX_Q_DQN_REG"))]
    lines.append("  return 0;\n}")
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
    for k, v in ops.Q_RULES.items():
        assert got[("rule", k)] == v, k


def test_loss_faces_refuse_actions_outside_the_rows():
    from stoix_b200 import ops
    from stoix_b200.utils import loss as L

    q, r, d = torch.zeros(3, 2), torch.zeros(3), torch.ones(3)
    for a in (torch.tensor([0, 2, 1]), torch.tensor([-1, 0, 1])):
        with pytest.raises(ops.StxError, match="a_tm1"):
            L.q_learning(q, a, r, d, q, 0.0)
        with pytest.raises(ops.StxError, match="a_tm1"):
            L.double_q_learning(q, q, a, r, d, q, 0.0)
        with pytest.raises(ops.StxError, match="a_tm1"):
            L.munchausen_q_learning(q, q, a, r, d, q, 0.03, 0.9, -1e3, 0.0)
