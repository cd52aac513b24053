"""GPU checks of Rainbow (ff_rainbow) against tests/rainbow_oracle.py: the noise draw, the effective weights and the fold, the dueling
combine, the weighted C51 kernel at every launch form, the prioritised ring (add across the wrap, stratified sampling, priorities,
determinism), a teacher-forced epoch gradient, eager / captured / replayed updates, the refusals, the entry point and CartPole."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from stoix_b200 import ops
from stoix_b200.networks.heads import linspace_f32
from tests import distq_oracle as DQ
from tests import rainbow_oracle as R
from tests.dqn_oracle import LossHyper
from tests.test_oracle_rainbow import _layout

pytestmark = pytest.mark.gpu

f64 = lambda t: t.double().cpu().numpy()
t_ = lambda x: torch.tensor(x, device="cuda")


def _close(got, want, rtol=1e-4, err_msg=""):
    np.testing.assert_allclose(got, want, rtol=rtol, atol=rtol * max(np.abs(want).max(), 1e-30), err_msg=err_msg)


def test_noise_kernel_draws_the_oracle_noise_and_fresh_noise_per_call():
    lay, _ = _layout()
    params = torch.zeros(lay.param_count, device="cuda")
    eff, noise = lay.scratch("cuda")
    ctr = torch.tensor([3], dtype=torch.int64, device="cuda")
    lay.weights(params, eff, noise, seed=1234, offset=2, dev_counter=ctr)
    # normal2's logf / sincospif against NumPy's float32 log and float64 cos: within an ulp or two, not bit for bit
    np.testing.assert_allclose(f64(noise), R.noise(1234, 5, lay.noise_count), atol=2e-6, rtol=0)
    n5 = noise.clone()
    ops.counter_add(ctr, 1)
    lay.weights(params, eff, noise, seed=1234, offset=2, dev_counter=ctr)
    np.testing.assert_allclose(f64(noise), R.noise(1234, 6, lay.noise_count), atol=2e-6, rtol=0)
    assert not torch.equal(noise, n5)
    lay.weights(params, eff, noise, seed=1234, offset=5)   # the same call index without a counter: the same bits
    assert torch.equal(noise, n5)


@pytest.mark.parametrize("branch", [(8,), (8, 5)])
def test_effective_weights_and_fold_are_exact(branch):
    """Parameters in 1/8 steps, injected noise in 1/4 steps: every product and sum is exact, so the kernels equal the oracle bit for bit,
    and the zero blocks of the block-diagonal layers stay zero."""
    lay, _ = _layout(branch=branch)
    rng = np.random.default_rng(11)
    params = (rng.integers(-16, 17, size=lay.param_count) / 8).astype(np.float32)
    nz = (rng.integers(-8, 9, size=lay.noise_count) / 4).astype(np.float32)
    eff, noise = lay.scratch("cuda")
    noise.copy_(t_(nz))
    lay.weights(t_(params), eff, noise, draw=False)
    np.testing.assert_array_equal(eff.cpu().numpy(), R.effective(lay.layers, params, nz, lay.eff_count))
    g_eff = (rng.integers(-16, 17, size=lay.eff_count) / 16).astype(np.float32)
    grad = torch.full((lay.param_count,), 7.0, device="cuda")
    lay.fold(t_(g_eff), noise, grad, overwrite=True)
    want = R.fold(lay.layers, g_eff, nz, lay.param_count)
    np.testing.assert_array_equal(grad.cpu().numpy(), want)
    lay.fold(t_(g_eff), noise, grad, overwrite=False)
    np.testing.assert_array_equal(grad.cpu().numpy(), 2 * want)


@pytest.mark.parametrize("A", [2, 3, 4, 18])
def test_dueling_combine_and_backward(A):
    rng = np.random.default_rng(A)
    M, N = 37, 51
    head = (rng.integers(-64, 65, size=(M, N + A * N)) / 4).astype(np.float32)
    dq = (rng.integers(-64, 65, size=(M, A * N)) / 4).astype(np.float32)
    q, dh = ops.dueling_combine(t_(head), A, N), ops.dueling_backward(t_(dq), A, N)
    if A in (2, 4):   # the mean divides by a power of two: exact
        np.testing.assert_array_equal(f64(q), R.dueling_combine(head, A, N))
        np.testing.assert_array_equal(f64(dh), R.dueling_backward(dq, A, N))
    else:
        _close(f64(q), R.dueling_combine(head, A, N), 1e-6)
        _close(f64(dh), R.dueling_backward(dq, A, N), 1e-6)


@pytest.mark.parametrize("N", [31, 51, 63, 65, 129, 513])
def test_weighted_c51_kernel(N):
    """Weights of one give the unweighted kernel's bits; other weights scale each row's gradient and the metric, and loss_rows stays
    the unweighted loss."""
    from tests.test_distq_gpu import _c51_case

    rng = np.random.default_rng(N)
    M, A = 300, 3
    atoms, lt1, lt, q_sel, a, r, done = _c51_case(rng, M, A, N)
    h = LossHyper(gamma=0.99, max_abs_reward=30.0)
    hy = ops.dist_q_hyper(gamma=h.gamma, max_abs_reward=h.max_abs_reward)

    def run(w):
        g, metrics, rows = torch.full((M, A * N), 9.0, device="cuda"), torch.zeros(2, device="cuda"), torch.zeros(M, device="cuda")
        ops.categorical_q_loss_grads(t_(lt1), t_(lt), t_(q_sel), t_(atoms), t_(atoms), t_(a), t_(r), hy, g, metrics, done=t_(done), loss_rows=rows,
                                     weight=0.5, row_weight=None if w is None else t_(w))
        return g, metrics, rows

    base, ones = run(None), run(np.ones(M, np.float32))
    assert all(torch.equal(x, y) for x, y in zip(base, ones))
    w = rng.random(M).astype(np.float32)
    g, metrics, rows = run(w)
    assert all(torch.equal(x, y) for x, y in zip((g, metrics, rows), run(w)))
    loss, want, _ = DQ.categorical_loss_and_grad(lt1, lt, q_sel, atoms, atoms, a, r, done, h)
    _close(f64(g), want * w[:, None])
    _close(f64(rows), loss)
    np.testing.assert_allclose(metrics[0].item(), 0.5 * (w * loss).mean(), rtol=1e-5)


def test_weighted_c51_kernel_per_row_support_and_discount():
    """The (M, N) atoms form and the direct discount input of the weighted loss: weights of one give the unweighted bits, other
    weights scale each row's gradient."""
    from tests.test_distq_gpu import _c51_case

    rng = np.random.default_rng(7)
    M, A, N = 200, 4, 51
    atoms, lt1, lt, q_sel, a, r, done = _c51_case(rng, M, A, N)
    z_tm1 = (atoms[None, :] + rng.integers(-4, 5, size=(M, 1)).astype(np.float32)).astype(np.float32)
    z_t = (atoms[None, :] * np.float32(0.5) + rng.integers(-4, 5, size=(M, 1)).astype(np.float32)).astype(np.float32)
    disc = (rng.random(M) * 0.99).astype(np.float32)
    h = LossHyper(gamma=0.99, max_abs_reward=30.0)
    hy = ops.dist_q_hyper(gamma=h.gamma, max_abs_reward=h.max_abs_reward)

    def run(w):
        g, metrics, rows = torch.full((M, A * N), 9.0, device="cuda"), torch.zeros(2, device="cuda"), torch.zeros(M, device="cuda")
        ops.categorical_q_loss_grads(t_(lt1), t_(lt), t_(q_sel), t_(z_tm1), t_(z_t), t_(a), t_(r), hy, g, metrics, discount=t_(disc), loss_rows=rows,
                                     row_weight=None if w is None else t_(w))
        return g, metrics, rows

    assert all(torch.equal(x, y) for x, y in zip(run(None), run(np.ones(M, np.float32))))
    w = rng.random(M).astype(np.float32)
    g, metrics, rows = run(w)
    loss, want, _ = DQ.categorical_loss_and_grad(lt1, lt, q_sel, z_tm1, z_t, a, r, None, h, discount=disc)
    _close(f64(g), want * w[:, None])
    _close(f64(rows), loss)
    np.testing.assert_allclose(metrics[0].item(), (w * loss).mean(), rtol=1e-5)


def _ring_case(L=6, E=3, D=2, n=3, alpha=1.0):
    return ops.PrioritisedRing(L, E, D, n, alpha, "cuda"), R.PrioRing(L, E, D, n, alpha)


def _batch(rng, T, E, D):
    obs = rng.integers(-8, 9, size=(T, E, D)).astype(np.float32)
    return (obs, rng.integers(0, 4, size=(T, E)).astype(np.int32), rng.integers(-4, 5, size=(T, E)).astype(np.float32),
            (rng.random((T, E)) < 0.2).astype(np.uint8), obs + np.float32(0.5))


def _check_tree(ring: ops.PrioritisedRing):
    """Every parent is the sum of its children in index order (fp32), the leaves first."""
    tree = ring.tree.cpu().numpy()
    c, off = ring.envs * ring.length, 0
    while c > 1:
        nxt = (c + 31) // 32
        for k in range(nxt):
            s = np.float32(0)
            for v in tree[off + 32 * k: off + min(32 * k + 32, c)]:
                s = np.float32(s + v)
            assert tree[off + c + k] == s
        off, c = off + c, nxt


def test_ring_add_across_the_wrap_and_validity():
    ring, ref = _ring_case()
    rng = np.random.default_rng(1)
    for T in (2, 2, 4, 1, 7, 3):   # the fourth add wraps, the fifth writes more rows than the ring holds
        b = _batch(rng, T, 3, 2)
        ops.replay_add_prioritised(ring, *(t_(x) for x in b))
        ref.add(*b)
        np.testing.assert_array_equal(ring.priorities.cpu().numpy(), ref.prio.astype(np.float32), err_msg=f"T={T}")
        np.testing.assert_array_equal(ring.obs.cpu().numpy(), ref.obs)
        np.testing.assert_array_equal(ring.reward.cpu().numpy(), ref.reward)
        assert ring.state.tolist() == [ref.w, ref.c]
        _check_tree(ring)
        if T == 4:   # give some items other priorities: later adds must keep the untouched ones
            idx = np.nonzero(ref.prio)[0][:3].astype(np.int32)
            pr = np.array([2.0, 4.0, 0.5], np.float32)
            ops.replay_set_priorities(ring, t_(idx), t_(pr))
            ref.set_priorities(idx, pr)


def test_stratified_sampling_is_exact_on_power_of_two_priorities():
    ring, ref = _ring_case(L=8, E=4, D=3, n=3)
    rng = np.random.default_rng(2)
    for T in (5, 4):
        b = _batch(rng, T, 4, 3)
        ops.replay_add_prioritised(ring, *(t_(x) for x in b))
        ref.add(*b)
    valid = np.nonzero(ref.prio)[0].astype(np.int32)
    pr = (2.0 ** rng.integers(-3, 4, size=len(valid))).astype(np.float32)
    ops.replay_set_priorities(ring, t_(valid), t_(pr))
    ref.set_priorities(valid, pr)
    M = 16
    u = (rng.integers(0, 8, size=M) / 8).astype(np.float32)
    out = dict(obs=torch.zeros(2 * M, 3, device="cuda"), action=torch.zeros(M, dtype=torch.int32, device="cuda"),
               reward=torch.zeros(M, device="cuda"), done=torch.zeros(M, dtype=torch.uint8, device="cuda"),
               idx=torch.zeros(M, dtype=torch.int32, device="cuda"), prob=torch.zeros(M, device="cuda"), weight=torch.zeros(M, device="cuda"))
    count = torch.tensor([25], dtype=torch.int32, device="cuda")
    ops.replay_sample_prioritised(ring, M, 0, out["obs"][:M], out["obs"][M:], out["action"], out["reward"], out["done"], out["idx"], out["prob"],
                                  out["weight"], 0.9, 0.4, 100.0, count=count, u_in=t_(u))
    idx = ref.sample(u)
    np.testing.assert_array_equal(out["idx"].cpu().numpy(), idx)
    total = ref.prio.sum()
    np.testing.assert_array_equal(out["prob"].cpu().numpy(), (ref.prio[idx] / total).astype(np.float32))
    for m, i in enumerate(idx):
        o, a, _, d, nxt, r, dn = ref.transition(i, 0.9)
        np.testing.assert_array_equal(out["obs"][m].cpu().numpy(), o)
        np.testing.assert_array_equal(out["obs"][M + m].cpu().numpy(), nxt)
        assert out["action"][m].item() == a and bool(out["done"][m].item()) == d
        assert out["reward"][m].item() == float(R.n_step_return32(r, dn, 0.9))
    beta = R.beta_at(25, 0.4, 100.0)
    np.testing.assert_allclose(f64(out["weight"]), R.importance_weights(ref.prio[idx] / total, beta), rtol=2e-6)
    # Philox uniforms: the oracle's stream
    ctr = torch.tensor([4], dtype=torch.int64, device="cuda")
    ops.replay_sample_prioritised(ring, M, 99, out["obs"][:M], out["obs"][M:], out["action"], out["reward"], out["done"], out["idx"], out["prob"],
                                  out["weight"], 0.9, 0.4, 100.0, offset=1, dev_counter=ctr)
    np.testing.assert_array_equal(out["idx"].cpu().numpy(), ref.sample(R.prio_uniforms(99, 5, M)))


def test_set_priorities_duplicates_determinism_and_max():
    ring, ref = _ring_case(L=40, E=50, D=1, n=2, alpha=0.5)
    rng = np.random.default_rng(3)
    b = _batch(rng, 40, 50, 1)
    ops.replay_add_prioritised(ring, *(t_(x) for x in b))
    ref.add(*b)
    idx = rng.integers(0, 2000, size=512).astype(np.int32)
    idx[100:110] = idx[0]   # duplicates: the last occurrence (row 109) wins
    pr = rng.random(512).astype(np.float32) * 4
    snap = ring.tree.clone(), ring.max_priority.clone()
    ops.replay_set_priorities(ring, t_(idx), t_(pr))
    first = ring.tree.clone(), ring.max_priority.clone()
    ring.tree.copy_(snap[0]), ring.max_priority.copy_(snap[1])
    ops.replay_set_priorities(ring, t_(idx), t_(pr))
    assert torch.equal(ring.tree, first[0]) and torch.equal(ring.max_priority, first[1])   # two launches: the same bits
    ref.set_priorities(idx, pr)
    np.testing.assert_allclose(ring.priorities.cpu().numpy(), ref.prio, rtol=1e-6)
    assert ring.priorities[int(idx[0])].item() == pytest.approx(float(pr[109]) ** 0.5, rel=1e-6)
    assert ring.max_priority.item() == pytest.approx(ref.maxp, rel=1e-6)
    _check_tree(ring)


_SMALL = ["env=synthetic/box", "env.kwargs.obs_dim=8", "env.kwargs.num_actions=3", "network.actor_network.pre_torso.layer_sizes=[32,32]",
          "network.actor_network.action_head.layer_sizes=[16]", "system.num_atoms=11", "system.vmin=-5.0", "system.vmax=5.0", "system.q_lr=1e-3",
          "system.warmup_steps=6", "system.total_buffer_size=640", "system.n_step=3", "system.max_abs_reward=3.0", "system.tau=0.3",
          "logger.use_console=False", "arch.num_evaluation=1"]


def _learner(E, T, epochs, batch, extra=(), updates=40, U=1, env_name=None):
    from stoix_b200 import random as srandom
    from stoix_b200.config import compose
    from stoix_b200.systems.q_learning import ff_rainbow
    from stoix_b200.utils import make_env
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    ov = list(_SMALL) + [f"arch.total_num_envs={E * U}", f"arch.update_batch_size={U}", f"system.rollout_length={T}", f"system.epochs={epochs}",
                         f"system.total_batch_size={batch * U}", f"arch.total_timesteps={E * U * T * updates}"] + list(extra)
    if env_name:
        ov.append(f"env={env_name}")
    cfg = compose("default_ff_rainbow", ov, config_dir="default/anakin")
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, eval_env = make_env.make(cfg)
    keys = srandom.split(srandom.PRNGKey(3), 3)
    learn, eval_net, state = ff_rainbow.learner_setup(env, tuple(keys), cfg)
    return cfg, learn, eval_net, state, eval_env


def _grad64(lay, params: np.ndarray, nz: np.ndarray, x: np.ndarray, cot: np.ndarray, A: int, N: int) -> np.ndarray:
    """d sum(q_logits * cot) / d (mu, sigma) of the reference network in float64 (torch autograd), under the noise nz; the layout's
    torso layers first, then one layer per branch, then the two output layers."""
    p = torch.tensor(np.asarray(params, np.float64), requires_grad=True)
    nzt = torch.tensor(np.asarray(nz, np.float64))

    def lin(L, hh):
        n_in, n_out, o = L["in_"], L["out"], L["param"]
        W = n_in * n_out
        fin, fout = nzt[L["noise"]:L["noise"] + n_in], nzt[L["noise"] + n_in:L["noise"] + n_in + n_out]
        return hh @ (p[o:o + W].view(n_in, n_out) + p[o + W + n_out:o + 2 * W + n_out].view(n_in, n_out) * torch.outer(fin, fout)) + \
            p[o + W:o + W + n_out] + p[o + 2 * W + n_out:o + 2 * W + 2 * n_out] * fout

    silu = torch.nn.functional.silu
    hh = torch.tensor(np.asarray(x, np.float64))
    for L in lay.layers[:-4]:
        hh = silu(lin(L, hh))
    v = lin(lay.layers[-2], silu(lin(lay.layers[-4], hh))).view(-1, 1, N)
    adv = lin(lay.layers[-1], silu(lin(lay.layers[-3], hh))).view(-1, A, N)
    q = (v + adv - adv.mean(1, keepdim=True)).reshape(-1, A * N)
    (q * torch.tensor(np.asarray(cot, np.float64))).sum().backward()
    return p.grad.numpy()


def test_teacher_forced_epoch_gradient():
    """One epoch's gradient (two shards) against torch autograd of the reference loss in float64, with the noise each kernel drew read
    back and the sampled batch taken as given; the new priorities are each shard's own unweighted losses."""
    from stoix_b200.systems.q_learning import ff_rainbow as FR

    cfg, learn, _, state, _ = _learner(16, 2, 1, 32, U=2)
    learn.ensure_built(state)
    b = learn.built
    lay = b["layout"]
    A, N = 3, 11
    online, target = state.params.online.flat.clone(), state.params.target.flat.clone()
    target.add_(0.01)   # a target unlike the online network
    rng = np.random.default_rng(5)
    for u, bt in enumerate(b["batches"]):
        bt.xs.copy_(t_(rng.normal(size=bt.xs.shape).astype(np.float32)))
        bt.action.copy_(t_(rng.integers(0, A, size=32).astype(np.int32)))
        bt.reward.copy_(t_(rng.normal(size=32).astype(np.float32) * 2))
        bt.done.copy_(t_((rng.random(32) < 0.2).astype(np.uint8)))
        bt.idx.copy_(t_(rng.permutation(100)[:32].astype(np.int32)))
        bt.weight.copy_(t_(rng.random(32).astype(np.float32)))
    seeds = [11, 12]
    h = LossHyper(gamma=float(cfg.system.gamma), max_abs_reward=3.0)
    atoms = linspace_f32(-5.0, 5.0, N).astype(np.float64)
    for u, bt in enumerate(b["batches"]):   # each shard alone (U = 1 inside batch_grads): its whole gradient
        grads, metric = torch.zeros_like(b["grads"]), torch.zeros(1, device="cuda")
        FR.batch_grads(lay, online, target, [bt], [state.buffer_state[u]], b["head"], b["hyper"], [seeds[u]], 7, None, grads, metric, b["work"])
        nz = [f64(b["work"].eff[k][1]) for k in range(3)]
        for k in range(3):
            np.testing.assert_allclose(nz[k], R.noise(seeds[u], 7 + k, lay.noise_count), atol=2e-6)
        M = 32
        xs = f64(bt.xs)
        on64, tg64 = f64(online), f64(target)
        q_t = R.dueling_combine(R.noisy_forward64(lay.layers, tg64, nz[1], xs[M:], 2, 1), A, N)
        q_s = R.dueling_combine(R.noisy_forward64(lay.layers, on64, nz[2], xs[M:], 2, 1), A, N)
        sel = DQ.categorical_q_values(q_s, atoms, A)
        a, r, d, w = f64(bt.action).astype(np.int64), f64(bt.reward), f64(bt.done), f64(bt.weight)
        lt1 = R.dueling_combine(R.noisy_forward64(lay.layers, on64, nz[0], xs[:M], 2, 1), A, N)
        loss, g, _ = DQ.categorical_loss_and_grad(lt1, q_t, sel, atoms, atoms, a, r, d, h)
        _close(f64(b["work"].loss_rows), loss, 1e-4)
        _close(state.buffer_state[u].ring.priorities[f64(bt.idx).astype(np.int64)].double().cpu().numpy(), loss ** 0.5, 1e-4)
        # d mean(w loss) / d params through the dueling combine and the noisy layers, by autograd of the float64 network
        want = _grad64(lay, on64, nz[0], xs[:M], g * w[:, None], A, N)
        _close(f64(grads[:lay.param_count]), want, 2e-4)
        np.testing.assert_allclose(metric.item(), (w * loss).mean(), rtol=1e-4)


def test_three_updates_eager_captured_and_replayed_match_the_oracle(monkeypatch):
    """Three whole updates (eager, graph capture, replay), two shards, two epochs each, against the oracle: every rollout Q row
    re-computed under its noise draw (call t of the shard's stream) and every action re-drawn; the ring replayed through its adds,
    wrap included; every epoch's Philox uniforms re-drawn and sampled from the oracle's priorities (a sample may differ only where
    its draw lies within rounding of a slice boundary, and then the learner's is kept); the n-step rows, p_i and the importance
    weights with beta at the Adam count; the three noisy forwards (calls T + 3 ep + k), the weighted loss and its gradient by
    autograd, the new priorities, clip + Adam and Polyak.  Online and target arenas and the ring's priorities are compared after
    every update."""
    from oracle import ppo_oracle as O
    from stoix_b200.utils import replay as RP
    from tests import pqn_oracle as P

    E, T, epochs, M, U = 16, 2, 2, 32, 2
    rec: dict = {}
    orig = RP.PrioritisedTrajectoryBuffer.sample_into

    def recording(self, *args, **kw):   # the learner's sample of each epoch, copied on the stream (and so into the graph)
        orig(self, *args, **kw)
        r = rec.setdefault(id(self), {"n": 0, "idx": torch.zeros(epochs, M, dtype=torch.int32, device="cuda"),
                                      "weight": torch.zeros(epochs, M, device="cuda"), "reward": torch.zeros(epochs, M, device="cuda"),
                                      "done": torch.zeros(epochs, M, dtype=torch.uint8, device="cuda"), "xs": torch.zeros(epochs, 2 * M, 8, device="cuda")})
        ep = r["n"] % epochs
        r["n"] += 1
        r["idx"][ep].copy_(args[5]), r["weight"][ep].copy_(args[7]), r["reward"][ep].copy_(args[3]), r["done"][ep].copy_(args[4])
        r["xs"][ep, :M].copy_(args[0]), r["xs"][ep, M:].copy_(args[1])

    monkeypatch.setattr(RP.PrioritisedTrajectoryBuffer, "sample_into", recording)
    cfg, learn, _, state, _ = _learner(E, T, epochs, M, ["system.total_buffer_size=320"], U=U)   # 10 ring rows per shard: update 3 wraps
    cfg.arch.num_updates_per_eval = 1
    learn.ensure_built(state)
    b = learn.built
    lay, head = b["layout"], b["head"]
    A, N = head.action_dim, head.num_atoms
    atoms = head.atoms_host.astype(np.float64)
    sysc = cfg.system
    gamma, tau = float(sysc.gamma), float(sysc.tau)
    h = LossHyper(gamma=gamma, max_abs_reward=float(sysc.max_abs_reward))
    beta0, steps = float(sysc.importance_sampling_exponent), float(int(cfg.arch.num_updates) * epochs)
    n = lay.param_count
    M62 = (1 << 62) - 1
    nseed = [(state.key[2] + u) & M62 for u in range(U)]
    bufs = state.buffer_state
    refs = []
    for buf in bufs:
        rg = buf.ring
        ref = R.PrioRing(rg.length, rg.envs, rg.obs_dim, rg.n_step, rg.priority_exponent)
        for name in ("obs", "next_obs", "action", "reward", "done"):
            getattr(ref, name)[:] = getattr(rg, name).cpu().numpy()
        ref.w, ref.c = (int(x) for x in rg.state.tolist())
        ref.prio, ref.maxp = f64(rg.priorities), float(rg.max_priority.item())
        refs.append(ref)
    online, target = f64(state.params.online.flat)[:n], f64(state.params.target.flat)[:n]
    st = O.AdamState(np.zeros(n), np.zeros(n))
    fwd = lambda params, nz, x: R.dueling_combine(R.noisy_forward64(lay.layers, params, nz, x, len(lay.layers) - 4, 1), A, N)
    flips = 0
    for k in range(3):
        ctr0 = k * (T + 3 * epochs)
        calls0 = [int(buf.counter.item()) for buf in bufs]
        pre = online.copy()
        out = learn(state)
        torch.cuda.synchronize()
        assert (b["graph"] is not None) == (k >= 1)
        for u in range(U):
            ro = b["shards"][u]
            for t in range(T):
                q = DQ.categorical_q_values(fwd(pre, R.noise(nseed[u], ctr0 + t, lay.noise_count), f64(ro.obs[t])), atoms, A)
                _close(f64(ro.q[t]), q, 1e-4, err_msg=f"update {k} shard {u} step {t}")
                np.testing.assert_array_equal(ro.action[t].cpu().numpy(), P.epsilon_greedy(ro.q[t].cpu().numpy(), 0.0, int(state.key[0]) + u, t + k * T))
            refs[u].add(ro.obs[:T].cpu().numpy(), ro.action.cpu().numpy(), ro.reward.cpu().numpy(), ro.done.cpu().numpy(), ro.next_obs.cpu().numpy())
            np.testing.assert_array_equal(bufs[u].ring.obs.cpu().numpy(), refs[u].obs)
        for ep in range(epochs):
            beta = R.beta_at(k * epochs + ep, beta0, steps)
            grads = []
            for u in range(U):
                ref, r = refs[u], rec[id(bufs[u])]
                draws = R.prio_uniforms(bufs[u].seed, calls0[u] + ep, M)
                want_idx, got_idx = ref.sample(draws), r["idx"][ep].cpu().numpy().astype(np.int64)
                total, cum = ref.prio.sum(), np.cumsum(ref.prio)
                for m in np.nonzero(want_idx != got_idx)[0]:
                    v = (m + float(draws[m])) * total / M
                    assert abs(v - cum[min(want_idx[m], got_idx[m])]) <= 1e-4 * total, (k, ep, u, m)
                    flips += 1
                idx = got_idx
                trs = [ref.transition(i, gamma) for i in idx]
                obs, nxt = np.stack([x[0] for x in trs]), np.stack([x[4] for x in trs])
                a, d = np.array([x[1] for x in trs]), np.array([x[3] for x in trs], np.float64)
                r32 = np.array([R.n_step_return32(x[5], x[6], gamma) for x in trs], np.float32)
                np.testing.assert_array_equal(r["xs"][ep].cpu().numpy(), np.concatenate([obs, nxt]))
                np.testing.assert_array_equal(r["reward"][ep].cpu().numpy(), r32)
                np.testing.assert_array_equal(r["done"][ep].cpu().numpy(), d.astype(np.uint8))
                w = R.importance_weights(ref.prio[idx] / total, beta)
                _close(f64(r["weight"][ep]), w, 1e-4, err_msg=f"weights, update {k} epoch {ep} shard {u}")
                nz = [R.noise(nseed[u], ctr0 + T + 3 * ep + j, lay.noise_count) for j in range(3)]
                sel = DQ.categorical_q_values(fwd(online, nz[2], nxt), atoms, A)
                loss, g, _ = DQ.categorical_loss_and_grad(fwd(online, nz[0], obs), fwd(target, nz[1], nxt), sel, atoms, atoms, a, r32, d, h)
                grads.append(_grad64(lay, online, nz[0], obs, g * w[:, None], A, N))
                ref.set_priorities(idx, loss)
            online, _ = O.clip_adam_step(online, np.mean(grads, axis=0), st, float(sysc.q_lr), float(sysc.max_grad_norm), float(np.float32(0.9)),
                                         float(np.float32(0.999)), float(np.float32(1e-5)))
            target = tau * online + (1.0 - tau) * target
        state = out.learner_state
        np.testing.assert_allclose(f64(state.params.online.flat)[:n], online, rtol=1e-4, atol=2e-6, err_msg=f"online, update {k}")
        np.testing.assert_allclose(f64(state.params.target.flat)[:n], target, rtol=1e-4, atol=2e-6, err_msg=f"target, update {k}")
        for u in range(U):
            _close(f64(bufs[u].ring.priorities), refs[u].prio, 1e-3, err_msg=f"priorities, update {k} shard {u}")
        assert b["noise_ctr"].item() == (k + 1) * (T + 3 * epochs)
    assert int(state.params.online.arena_counts[0]) == 3 * epochs and refs[0].w < 6   # the ring wrapped
    print(f"[ff_rainbow three updates] samples kept from the learner at a slice boundary: {flips}")


def test_three_updates_eager_captured_and_replayed_agree_and_draw_fresh_noise():
    """The same learner run eagerly three times and as (eager, capture, replay) gives the same arenas, rings and metrics bit for bit;
    every update draws new noise and new samples, and the parameters move."""
    runs = []
    for graph in (False, True):
        cfg, learn, _, state, _ = _learner(16, 2, 2, 32, [f"arch.cuda_graph={graph}"])
        cfg.arch.num_updates_per_eval = 1
        snaps = []
        for _ in range(3):
            out = learn(state)
            state = out.learner_state
            b = learn.built
            snaps.append((state.params.online.arena.clone(), state.params.target.arena.clone(), state.buffer_state[0].ring.tree.clone(),
                          b["work"].eff[0][1].clone(), b["batches"][0].idx.clone(), out.train_metrics["q_loss"].clone()))
        assert b["noise_ctr"].item() == 3 * (2 + 3 * 2) and (b["graph"] is not None) == graph
        runs.append(snaps)
    for k in range(3):
        assert all(torch.equal(x, y) for x, y in zip(runs[0][k], runs[1][k])), f"update {k}"
    for k in (1, 2):
        assert not torch.equal(runs[1][k][3], runs[1][k - 1][3])   # fresh noise on every replay
        assert not torch.equal(runs[1][k][4], runs[1][k - 1][4])   # fresh samples on every replay
        assert not torch.equal(runs[1][k][0], runs[1][k - 1][0])
    assert all(torch.isfinite(s[0]).all() for s in runs[1])


def test_bf16_and_other_heads_are_refused():
    with pytest.raises(ValueError, match="bf16"):
        _learner(16, 2, 1, 32, ["arch.precision=bf16"])
    with pytest.raises(ValueError, match="not implemented"):
        _learner(16, 2, 1, 32, ["network=mlp_c51"])
    with pytest.raises(ValueError, match="use_layer_norm"):
        _learner(16, 2, 1, 32, ["network.actor_network.pre_torso.use_layer_norm=True"])


def test_eval_network_uses_one_fixed_noise_draw():
    cfg, learn, eval_net, state, _ = _learner(16, 2, 1, 32)
    obs = torch.randn(64, 8, device="cuda")
    q1 = eval_net.apply(state.params.online, obs).preferences.clone()
    q2 = eval_net.apply(state.params.online, obs).preferences.clone()
    assert torch.equal(q1, q2)
    q3 = eval_net.actor.apply(state.params.online, obs, seed=eval_net.noise_seed, offset=1)[0].preferences
    assert not torch.equal(q1, q3)


def test_entry_point_runs_evaluates_and_checkpoints(tmp_path, monkeypatch):
    from stoix_b200.config import compose
    from stoix_b200.systems.q_learning import ff_rainbow

    torch.cuda.set_device(0)
    monkeypatch.chdir(tmp_path)
    cfg = compose("default_ff_rainbow", _SMALL + ["arch.total_num_envs=16", "system.rollout_length=2", "system.epochs=2", "system.total_batch_size=32",
                                                  "arch.total_timesteps=128", "arch.num_evaluation=2", "arch.absolute_metric=True",
                                                  "logger.checkpointing.save_model=True", "arch.num_eval_episodes=4", "arch.max_eval_steps=50"],
                  config_dir="default/anakin")
    assert np.isfinite(ff_rainbow.hydra_entry_point(cfg))
    saved = sorted(tmp_path.glob(f"checkpoints/{cfg.system.system_name}/*/*.pt"))
    assert saved, "no checkpoint written"


def test_cartpole_learns():
    """CartPole at the reference's Rainbow defaults except the schedule (1024 envs, T = 2, 16 epochs of batch 512, lr 5e-4), 192
    updates, evaluated greedily (with the fixed evaluation noise) every 16 updates.  Measured on an H100 80GB HBM3 at 700 W with this
    seed: evaluations 139.7, 57.8, 261.7, 189.0, 89.2, 57.9, 63.6, 223.4, 288.1, 499.8, 500.0, 500.0, training return 144.0.
    Bar: the DQN family's 150 for the best evaluation."""
    from stoix_b200 import random as srandom
    from stoix_b200.evaluator import get_distribution_act_fn, get_ff_evaluator_fn
    from stoix_b200.config import compose
    from stoix_b200.systems.q_learning import ff_rainbow
    from stoix_b200.utils import make_env
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    cfg = compose("default_ff_rainbow", ["arch.total_num_envs=1024", "system.rollout_length=2", "system.epochs=16", "system.total_batch_size=512",
                                         "system.q_lr=5e-4", "arch.total_timesteps=819200", "arch.num_evaluation=1", "logger.use_console=False"],
                  config_dir="default/anakin")
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, eval_env = make_env.make(cfg)
    learn, eval_net, state = ff_rainbow.learner_setup(env, tuple(srandom.split(srandom.PRNGKey(3), 3)), cfg)
    cfg.arch.num_updates_per_eval = 16
    evaluator = get_ff_evaluator_fn(eval_env, get_distribution_act_fn(cfg, eval_net.apply), cfg)
    evals = []
    for k in range(12):
        out = learn(state)
        state = out.learner_state
        evals.append(float(evaluator(state.params.online, srandom.PRNGKey(k))["episode_return"].mean()))
    em = out.episode_metrics
    train_return = float(em["episode_return"][em["is_terminal_step"]].mean())
    print(f"[ff_rainbow cartpole] greedy evaluations {[round(r, 1) for r in evals]}, training return {train_return:.1f}")
    assert max(evals) > 150.0


def test_two_ranks_run_the_captured_update(tmp_path):
    """Two torchrun ranks run the entry point (NCCL all-reduce inside the captured step)."""
    import os
    import subprocess
    import sys

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (NCCL refuses two ranks on one device)")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    ov = _SMALL + ["arch.total_num_envs=32", "system.rollout_length=2", "system.epochs=2", "system.total_batch_size=64", "arch.total_timesteps=512",
                   "arch.num_evaluation=2", "arch.num_eval_episodes=4", "arch.max_eval_steps=50"]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port", "29561",
           os.path.join(root, "stoix", "systems", "q_learning", "ff_rainbow.py")] + ov
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
