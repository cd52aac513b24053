"""C51 and QR-DQN on the GPU through the C ABI and the learner, against the NumPy oracle (tests/distq_oracle.py)."""
import importlib

import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from stoix_b200 import ops
from stoix_b200.config import DictConfig
from stoix_b200.networks.heads import linspace_f32
from tests import distq_oracle as D
from tests import dqn_oracle as Q
from tests import pqn_oracle as P
from tests.test_dqn_gpu import _learner, _ring_equals

pytestmark = pytest.mark.gpu

f64 = lambda t: t.detach().double().cpu().numpy()
t_ = lambda x: torch.tensor(x, device="cuda")
SYSTEMS = {"ff_c51": "categorical_double_q_learning", "ff_qr_dqn": "quantile_q_learning"}
# odd N on both sides of every launch-form switch (32 / 64 / 128 threads per row), the reference's 51 and 200, and a larger N
NS = [31, 33, 51, 63, 65, 127, 129, 200, 513]


def _close(got, want, rtol=1e-4, err_msg=""):
    np.testing.assert_allclose(got, want, rtol=rtol, atol=rtol * max(np.abs(want).max(), 1e-30), err_msg=err_msg)


def test_dist_q_values_against_the_oracle():
    rng = np.random.default_rng(0)
    for M, A, N in ((1000, 2, 51), (333, 8, 200), (7, 3, 1)):
        head = (rng.normal(size=(M, A * N)) * 3).astype(np.float32)
        atoms = linspace_f32(-10.0, 10.0, N)
        _close(f64(ops.dist_q_values("categorical", t_(head), A, N, t_(atoms))), D.categorical_q_values(head, atoms, A), 1e-5)
        _close(f64(ops.dist_q_values("quantile", t_(head), A, N)), D.quantile_q_values(head, A), 1e-5)


def _c51_case(rng, M, A, N):
    """Selector ties, done rows, rewards clipped to 30 and past the +-10 support, targets exactly on atoms (done rows with r = atom)."""
    atoms = linspace_f32(-10.0, 10.0, N)
    lt1, lt = (rng.normal(size=(M, A * N)) * 2).astype(np.float32), (rng.normal(size=(M, A * N)) * 2).astype(np.float32)
    q_sel = (rng.integers(0, 3, size=(M, A)) * 0.5).astype(np.float32)
    a = rng.integers(0, A, size=M).astype(np.int32)
    r = (rng.normal(size=M) * 3).astype(np.float32)
    r[::7] = 40.0
    r[1::7] = -40.0
    done = (rng.random(M) < 0.25).astype(np.uint8)
    on = np.arange(2, M, 7)
    done[on] = 1
    r[on] = atoms[rng.integers(0, N, size=len(on))]
    return atoms, lt1, lt, q_sel, a, r, done


def _qr_case(rng, M, A, N):
    """Selector ties (action 1 a copy of action 0 on a third of the rows), done rows, clipped rewards."""
    q1, qt = (rng.normal(size=(M, A * N)) * 2).astype(np.float32), (rng.normal(size=(M, A * N)) * 2).astype(np.float32)
    ties = np.arange(0, M, 3)
    qt.reshape(M, A, N)[ties, 1] = qt.reshape(M, A, N)[ties, 0]
    a = rng.integers(0, A, size=M).astype(np.int32)
    r = (rng.normal(size=M) * 3).astype(np.float32)
    done = (rng.random(M) < 0.25).astype(np.uint8)
    tau = ((np.arange(N, dtype=np.float32) + np.float32(0.5)) / np.float32(N)).astype(np.float32)
    return q1, qt, a, r, done, tau


@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("A", [2, 8])
def test_categorical_loss_kernel_against_the_oracle(N, A):
    rng = np.random.default_rng(N * 10 + A)
    M = 300
    atoms, lt1, lt, q_sel, a, r, done = _c51_case(rng, M, A, N)
    h = Q.LossHyper(gamma=0.99, max_abs_reward=30.0)
    hy = ops.dist_q_hyper(gamma=h.gamma, max_abs_reward=h.max_abs_reward)
    runs = []
    for _ in range(2):
        g, metrics, rows = torch.full((M, A * N), 9.0, device="cuda"), torch.zeros(2, device="cuda"), torch.zeros(M, device="cuda")
        ops.categorical_q_loss_grads(t_(lt1), t_(lt), t_(q_sel), t_(atoms), t_(atoms), t_(a), t_(r), hy, g, metrics, done=t_(done), loss_rows=rows,
                                     weight=0.5)
        runs.append((g, metrics, rows))
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(runs[0], runs[1]))   # two launches: the same bits
    loss, want, _ = D.categorical_loss_and_grad(lt1, lt, q_sel, atoms, atoms, a, r, done, h)
    _close(f64(runs[0][0]), want)
    _close(f64(runs[0][2]), loss)
    np.testing.assert_allclose(runs[0][1][0].item(), 0.5 * loss.mean(), rtol=1e-5)
    assert runs[0][1][1].item() == 0.0
    assert (q_sel == q_sel.max(1, keepdims=True)).sum(1).max() > 1


@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("A", [2, 8])
@pytest.mark.parametrize("kappa", [0.0, 1.0])
def test_quantile_loss_kernel_against_the_oracle(N, A, kappa):
    rng = np.random.default_rng(N * 10 + A + int(kappa) * 1000)
    M = 200
    q1, qt, a, r, done, tau = _qr_case(rng, M, A, N)
    h = Q.LossHyper(gamma=0.99, max_abs_reward=2.0, huber=kappa)
    hy = ops.dist_q_hyper(gamma=h.gamma, max_abs_reward=h.max_abs_reward, huber_delta=kappa)
    runs = []
    for _ in range(2):
        g, metrics, rows = torch.full((M, A * N), 9.0, device="cuda"), torch.zeros(2, device="cuda"), torch.zeros(M, device="cuda")
        ops.quantile_q_loss_grads(t_(q1), t_(qt), t_(tau), t_(a), t_(r), hy, g, metrics, A, done=t_(done), loss_rows=rows, weight=0.5)
        runs.append((g, metrics, rows))
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(runs[0], runs[1]))
    loss, want = D.quantile_loss_and_grad(q1, qt, None, tau, a, r, done, h, A)
    _close(f64(runs[0][0]), want)
    _close(f64(runs[0][2]), loss)
    np.testing.assert_allclose(runs[0][1][0].item(), 0.5 * loss.mean(), rtol=1e-5)


def test_quantile_kernel_tie_conventions():
    """delta = 0 exactly in every pair: weight tau_i, and slope +1 for |.| (JAX), 0 for Huber."""
    N, M = 6, 3
    q = np.full((M, 2 * N), 3.0, np.float32)
    tau = ((np.arange(N, dtype=np.float32) + 0.5) / N).astype(np.float32)
    for kappa, slope in ((0.0, 1.0), (1.0, 0.0)):
        g, metrics = torch.zeros(M, 2 * N, device="cuda"), torch.zeros(1, device="cuda")
        ops.quantile_q_loss_grads(t_(q), t_(q), t_(tau), t_(np.zeros(M, np.int32)), t_(np.full(M, 3.0, np.float32)), ops.dist_q_hyper(huber_delta=kappa),
                                  g, metrics, 2, discount=t_(np.zeros(M, np.float32)))
        np.testing.assert_allclose(f64(g)[:, :N], np.broadcast_to(-tau * slope / M, (M, N)), rtol=1e-6)
        assert (f64(g)[:, N:] == 0).all() and metrics.item() == 0.0


def test_n_above_the_shared_memory_bound_is_refused():
    M, A, N = 4, 2, ops.DIST_MAX_N + 1
    z = torch.zeros(M, A * N, device="cuda")
    i, f, m = torch.zeros(M, dtype=torch.int32, device="cuda"), torch.zeros(M, device="cuda"), torch.zeros(1, device="cuda")
    with pytest.raises(ops.StxError, match="shared memory"):
        ops.quantile_q_loss_grads(z, z, torch.zeros(N, device="cuda"), i, f, ops.dist_q_hyper(), z.clone(), m, A, discount=f)
    with pytest.raises(ops.StxError, match="shared memory"):
        ops.categorical_q_loss_grads(z, z, torch.zeros(M, A, device="cuda"), torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda"), i, f,
                                     ops.dist_q_hyper(), z.clone(), m, discount=f)


def test_loss_faces_match_the_oracle():
    from stoix_b200.utils import loss as L

    rng = np.random.default_rng(4)
    M, A, N = 200, 3, 51
    atoms, lt1, lt, q_sel, a, r, _ = _c51_case(rng, M, A, N)
    d_t = (rng.random(M) * 0.99).astype(np.float32)
    rows_atoms = np.broadcast_to(atoms, (M, N)).copy()
    got = L.categorical_double_q_learning(t_(lt1.reshape(M, A, N)), t_(rows_atoms), t_(a), t_(r), t_(d_t), t_(lt.reshape(M, A, N)), t_(rows_atoms),
                                          t_(q_sel))
    want, _, _ = D.categorical_loss_and_grad(lt1, lt, q_sel, atoms, atoms, a, r, None, Q.LossHyper(), discount=d_t)
    assert tuple(got.shape) == (M,)
    _close(f64(got), want)
    q1, qt, a, r, _, tau = _qr_case(rng, M, A, N)
    sel = (rng.normal(size=(M, A * N))).astype(np.float32)
    swap = lambda x: t_(x.reshape(M, A, N).transpose(0, 2, 1).copy())   # the reference's (M, N, A)
    for kappa in (0.0, 1.0):
        got = L.quantile_q_learning(swap(q1), t_(np.broadcast_to(tau, (M, N)).copy()), t_(a), t_(r), t_(d_t), swap(sel), swap(qt), kappa)
        want, _ = D.quantile_loss_and_grad(q1, qt, sel, tau, a, r, None, Q.LossHyper(huber=kappa), A, discount=d_t)
        np.testing.assert_allclose(got.item(), want.mean(), rtol=1e-5)


def _support(system, learn_or_head):
    head = learn_or_head
    if system == "ff_c51":
        return head.atoms_host.astype(np.float64)
    return ((np.arange(head.num_quantiles, dtype=np.float32) + np.float32(0.5)) / np.float32(head.num_quantiles)).astype(np.float64)


@pytest.mark.parametrize("system", list(SYSTEMS))
def test_epoch_gradient_teacher_forced(system):
    """ff_dqn.batch_grads with the distributional loss on given batches: two shards (weight 1/2 each, the first overwrites a dirty
    arena) against the fp64 oracle, 1e-5 norm-wise; bit-identical on repeat."""
    from stoix_b200.networks.heads import DistributionalDiscreteQNetwork, QuantileDiscreteQNetwork
    from stoix_b200.systems.q_learning import ff_dqn

    loss = SYSTEMS[system]
    rng = np.random.default_rng(len(system))
    Dm, A, N, M = 10, 3, (11 if system == "ff_c51" else 13), 384
    head = DistributionalDiscreteQNetwork(A, 0.1, N, -10.0, 10.0) if system == "ff_c51" else QuantileDiscreteQNetwork(A, 0.1, N)
    spec = ops.MlpSpec((Dm, 64, 64, A * N), activation="silu", use_layer_norm=False)
    sizes = list(spec.sizes)
    on = (rng.normal(size=spec.param_count) * 0.2).astype(np.float32)
    tg = (on + rng.normal(size=spec.param_count) * 0.02).astype(np.float32)
    h = Q.LossHyper(gamma=0.99, max_abs_reward=2.0, huber=1.0 if system == "ff_qr_dqn" else 0.0)
    cfg = DictConfig({"system": {"gamma": 0.99, "max_abs_reward": 2.0, "huber_loss_parameter": 1.0}})
    hyper = ff_dqn.loss_hyper(loss, cfg, head, torch.device("cuda"))
    support = _support(system, head)
    on_p = O.MLPParams.from_flat(on.astype(np.float64), sizes, "silu", False)
    tg_p = O.MLPParams.from_flat(tg.astype(np.float64), sizes, "silu", False)
    batches, want, lsum = [], np.zeros(spec.param_count), 0.0
    for _ in range(2):
        obs, nxt = rng.normal(size=(M, Dm)).astype(np.float32), rng.normal(size=(M, Dm)).astype(np.float32)
        a = rng.integers(0, A, size=M).astype(np.int32)
        r = (rng.normal(size=M) * 3).astype(np.float32)
        d = (rng.random(M) < 0.2).astype(np.uint8)
        batches.append(ff_dqn.Batch(t_(np.concatenate([obs, nxt])), t_(a), t_(r), t_(d)))
        l, g = D.batch_grad(loss, on_p, tg_p, obs, nxt, a, r, d, h, support, A)
        want += 0.5 * g
        lsum += 0.5 * l
    work = ff_dqn.make_work(spec, M, "cuda", A if system == "ff_c51" else None)
    got = []
    for _ in range(2):
        grads, metric = torch.full((spec.param_count,), 7.0, device="cuda"), torch.zeros(1, device="cuda")
        ff_dqn.batch_grads(loss, spec, t_(on), t_(tg), batches, hyper, grads, metric, work)
        got.append((grads, metric))
    torch.cuda.synchronize()
    assert torch.equal(got[0][0], got[1][0]) and torch.equal(got[0][1], got[1][1])
    g = f64(got[0][0])
    assert np.linalg.norm(g - want) <= 1e-5 * np.linalg.norm(want), np.linalg.norm(g - want) / np.linalg.norm(want)
    np.testing.assert_allclose(got[0][1].item(), lsum, rtol=1e-5)


_SMALL = ["env.kwargs.obs_dim=8", "env.kwargs.num_actions=4", "network.actor_network.pre_torso.layer_sizes=[32,32]", "system.q_lr=1e-2",
          "system.warmup_steps=3", "system.total_buffer_size=400", "system.max_abs_reward=1.5", "system.tau=0.3"]
_HEAD = {"ff_c51": ["system.num_atoms=11", "system.vmin=-3", "system.vmax=3"], "ff_qr_dqn": ["system.num_quantiles=13"]}


@pytest.mark.parametrize("system", list(SYSTEMS))
def test_three_updates_eager_and_graph_match_the_oracle(system):
    """Three whole updates (eager, graph capture, replay): every rollout and warm-up action re-drawn from the expected Q, the ring
    after the add bit-exact, and online and target parameters against the oracle on the same sampled indices."""
    loss = SYSTEMS[system]
    E, T, epochs, M = 64, 2, 3, 96
    cfg, learn, eval_net, state, _ = _learner(system, E, T, epochs, M, _SMALL + _HEAD[system])
    cfg.arch.num_updates_per_eval = 1
    sysc = cfg.system
    head = eval_net.actor.action_head
    kind = "categorical" if system == "ff_c51" else "quantile"
    A, N = head.action_dim, head.out_dim // head.action_dim
    support = _support(system, head)
    atoms = t_(head.atoms_host) if system == "ff_c51" else None
    spec = state.params.online.spec
    sizes, n = list(spec.sizes), spec.param_count
    h = Q.LossHyper(gamma=float(sysc.gamma), max_abs_reward=float(sysc.max_abs_reward), huber=float(sysc.get("huber_loss_parameter", 0.0)))
    expected = (lambda x: D.categorical_q_values(x, support, A)) if system == "ff_c51" else (lambda x: D.quantile_q_values(x, A))
    buf = state.buffer_state[0]
    ring = buf.ring
    W = int(sysc.warmup_steps)
    ref = Q.Ring(ring.capacity, ring.obs_dim)
    for name in ("obs", "next_obs", "action", "reward", "done"):
        getattr(ref, name)[:] = getattr(ring, name).cpu().numpy()
    ref.pos, ref.size = W * E, W * E
    online, target = f64(state.params.online.flat)[:n], f64(state.params.target.flat)[:n]
    assert (online == target).all()
    st = O.AdamState(np.zeros(n), np.zeros(n))
    eps = np.float32(sysc.training_epsilon)
    init = O.MLPParams.from_flat(online, sizes, "silu", False)
    for t in range(W):
        rows = slice(t * E, (t + 1) * E)
        q_w = ops.dist_q_values(kind, ops.mlp_forward(spec, state.params.online.flat, ring.obs[rows]), A, N, atoms)
        _close(f64(q_w), expected(O.mlp_forward(init, f64(ring.obs[rows]))[0]), 1e-4)
        np.testing.assert_array_equal(ring.action[rows].cpu().numpy(), P.epsilon_greedy(q_w.cpu().numpy(), eps, int(state.key[1]), t),
                                      err_msg=f"warm-up step {t}")
    for k in range(3):
        pre = O.MLPParams.from_flat(f64(state.params.online.flat)[:n], sizes, "silu", False)
        call0 = int(buf.counter.item())
        out = learn(state)
        torch.cuda.synchronize()
        assert (learn.built["graph"] is not None) == (k >= 1)
        ro = learn.built["shards"][0]
        _close(f64(ro.q).reshape(T * E, -1), expected(O.mlp_forward(pre, f64(ro.obs[:T]).reshape(T * E, -1))[0]), 1e-4)
        for t in range(T):
            want = P.epsilon_greedy(ro.q[t].cpu().numpy(), eps, int(state.key[0]), t + k * T)
            np.testing.assert_array_equal(ro.action[t].cpu().numpy(), want, err_msg=f"update {k} step {t}")
        ref.add(ro.obs[:T].cpu().numpy(), ro.action.cpu().numpy(), ro.reward.cpu().numpy(), ro.done.cpu().numpy(), ro.next_obs.cpu().numpy())
        _ring_equals(ring, ref)
        eps_batches = [[ref.sample(M, buf.seed, call0 + ep)[:5]] for ep in range(epochs)]
        online, target = D.distq_update(loss, online, target, st, eps_batches, h, support, A, float(sysc.q_lr), float(sysc.max_grad_norm),
                                        float(sysc.tau), sizes)
        np.testing.assert_allclose(f64(out.learner_state.params.online.flat)[:n], online, rtol=1e-4, atol=2e-6, err_msg=f"online, update {k}")
        np.testing.assert_allclose(f64(out.learner_state.params.target.flat)[:n], target, rtol=1e-4, atol=2e-6, err_msg=f"target, update {k}")
        state = out.learner_state
    assert out.train_metrics["q_loss"].shape == (1, epochs)
    assert int(state.params.online.arena_counts[0]) == 3 * epochs


@pytest.mark.parametrize("system", list(SYSTEMS))
def test_graph_replays_draw_fresh_actions_and_indices(system):
    cfg, learn, _, state, _ = _learner(system, 64, 2, 2, 64, _SMALL + _HEAD[system], U=2)
    cfg.arch.num_updates_per_eval = 1
    seen = []
    for _ in range(3):
        state = learn(state).learner_state
        torch.cuda.synchronize()
        ros, bts = learn.built["shards"], learn.built["batches"]
        seen.append((ros[0].action.clone(), bts[0].xs.clone()))
        assert not torch.equal(ros[0].obs, ros[1].obs) and not torch.equal(bts[0].xs, bts[1].xs)
    assert not torch.equal(seen[1][0], seen[2][0]) and not torch.equal(seen[1][1], seen[2][1])


@pytest.mark.parametrize("system", list(SYSTEMS))
def test_bf16_is_refused(system):
    with pytest.raises(ValueError, match="bf16"):
        _learner(system, 64, 2, 2, 64, _SMALL + _HEAD[system] + ["arch.precision=bf16"])


def test_c51_learner_refuses_the_plain_head():
    with pytest.raises(ValueError, match="not implemented"):
        _learner("ff_c51", 64, 2, 2, 64, _SMALL + ["network=mlp_dqn"])


_ENTRY = ["env=synthetic/box", "env.kwargs.obs_dim=8", "env.kwargs.num_actions=3", "env.kwargs.p_term=0.05", "arch.total_num_envs=16",
          "system.rollout_length=2", "system.epochs=2", "system.total_batch_size=32", "system.total_buffer_size=400", "system.warmup_steps=3",
          "arch.total_timesteps=128", "network.actor_network.pre_torso.layer_sizes=[32,32]", "arch.num_evaluation=2", "arch.absolute_metric=True",
          "logger.checkpointing.save_model=True", "arch.num_eval_episodes=4", "arch.max_eval_steps=50", "logger.use_console=False"]


@pytest.mark.parametrize("system", list(SYSTEMS))
def test_entry_point_runs_evaluates_and_checkpoints(system, tmp_path, monkeypatch):
    from stoix_b200.config import compose

    torch.cuda.set_device(0)
    monkeypatch.chdir(tmp_path)
    cfg = compose(f"default_{system}", _ENTRY + _HEAD[system], config_dir="default/anakin")
    mod = importlib.import_module(f"stoix_b200.systems.q_learning.{system}")
    assert np.isfinite(mod.hydra_entry_point(cfg))
    saved = sorted(tmp_path.glob(f"checkpoints/{cfg.system.system_name}/*/*.pt"))
    assert saved, "no checkpoint written"
    blob = torch.load(saved[-1], map_location="cpu")
    assert set(blob) >= {"params", "mu", "nu", "counts"} and torch.isfinite(blob["params"]).all()


@pytest.mark.parametrize("system", list(SYSTEMS))
def test_cartpole_learns(system):
    """CartPole at test_dqn_gpu.test_cartpole_learns's schedule (1024 envs, T = 2, 16 epochs of batch 512, tau 0.005, lr 5e-4,
    epsilon 0.1), 192 updates, evaluated greedily every 16 updates; the system's own head (C51: 51 atoms on [0, 500]; QR-DQN: 200
    quantiles, kappa 1).  The best greedy evaluation and the training episodes of the last 16 updates are read.  Measured on an
    H100 80GB HBM3 at 700 W with this seed: ff_c51 evaluations 9.2, 19.5, 176.2, 142.0, 107.3, 200.1, 255.0, 258.2, 259.1, 270.2,
    270.9, 273.9, training return 216.8; ff_qr_dqn 9.4, 9.2, 9.2, 10.2, 189.1, 286.1, 226.6, 245.7, 249.0, 269.9, 273.1, 276.1,
    training return 238.9.  Bars: the DQN family's 150 and 80."""
    from stoix_b200 import random as srandom
    from stoix_b200.evaluator import get_distribution_act_fn, get_ff_evaluator_fn

    sched = ["system.q_lr=5e-4", "system.warmup_steps=16"]
    cfg, learn, eval_net, state, eval_env = _learner(system, 1024, 2, 16, 512, sched, env_name="gymnax/cartpole", updates=400)
    cfg.arch.num_updates_per_eval = 16
    evaluator = get_ff_evaluator_fn(eval_env, get_distribution_act_fn(cfg, eval_net.apply), cfg)
    evals = []
    for k in range(12):
        out = learn(state)
        state = out.learner_state
        evals.append(float(evaluator(state.params.online, srandom.PRNGKey(k))["episode_return"].mean()))
    em = out.episode_metrics
    train_return = float(em["episode_return"][em["is_terminal_step"]].mean())
    print(f"[{system} cartpole] greedy evaluations {[round(r, 1) for r in evals]}, training return {train_return:.1f}")
    assert max(evals) > 150.0 and train_return > 80.0


@pytest.mark.parametrize("system", list(SYSTEMS))
def test_two_rank_updates_match_the_oracle(system, tmp_path):
    """Two torchrun ranks, three whole updates with the NCCL gradient all-reduce inside the captured step; each rank's parameters
    against the oracle with a gloo gradient exchange, and the arenas bit-identical across the ranks."""
    import json
    import os
    import subprocess
    import sys

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (NCCL refuses two ranks on one device)")
    from tests.test_dqn_gpu import WORKER

    head = _HEAD[system]
    script = WORKER.replace("SYSTEM", system).replace('"system.huber_loss_parameter=1.0"]', '"system.huber_loss_parameter=1.0"] + ' + repr(head))
    script = script.replace("from tests import dqn_oracle as Q", "from tests import dqn_oracle as Q\nfrom tests import distq_oracle as DQ")
    script = script.replace(
        "online, target = Q.dqn_update(learn.loss, online, target, st, batches, h, float(s.q_lr), float(s.max_grad_norm), float(s.tau), sizes, \"silu\",\n"
        "                                  False, grad_sync=grad_sync)",
        "hd = learn.built['hyper']\n"
        "    online, target = DQ.distq_update(learn.loss, online, target, st, batches, h, hd.support.double().cpu().numpy(), hd.A, float(s.q_lr),\n"
        "                                     float(s.max_grad_norm), float(s.tau), sizes, grad_sync=grad_sync)")
    assert "DQ.distq_update" in script
    (tmp_path / "worker.py").write_text(script)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(29541 + list(SYSTEMS).index(system)), str(tmp_path / "worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=240, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    res = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    assert res["oracle_ok_all_ranks"], res
    assert res["params_identical_across_ranks"] and res["metrics_identical_across_ranks"] and res["shards_differ"] and res["graph"], res
