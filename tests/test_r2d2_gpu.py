"""rec_r2d2 kernels and learner on the GPU against tests/r2d2_oracle.py: the prioritised sequence ring, the value transform, the fused
loss, the dueling head with its final LayerNorm, teacher-forced gradients and one optimiser step, whole updates (eager, captured,
replayed), the entry point and learning on CartPole."""
import numpy as np
import pytest
import torch

from tests import r2d2_oracle as orc

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda")


def _ops():
    from stoix_b200 import ops
    return ops


def _batch(T, E, D, Cd, g):
    return dict(obs=torch.randn(T, E, D, generator=g), action=torch.randint(0, 5, (T, E), generator=g, dtype=torch.int32),
                reward=torch.randn(T, E, generator=g), done=torch.randint(0, 2, (T, E), generator=g, dtype=torch.uint8),
                truncated=torch.randint(0, 2, (T, E), generator=g, dtype=torch.uint8), reset=torch.randint(0, 2, (T, E), generator=g, dtype=torch.uint8),
                carry=torch.randn(T, E, Cd, generator=g))


@pytest.mark.parametrize("L,E,S,p,adds", [(11, 3, 4, 3, [5, 8, 2]),        # L % p != 0, a wrap
                                          (97, 4, 80, 40, [128, 40, 40, 40, 40]),   # the reference default's ring: warm-up wraps it
                                          (8, 2, 3, 1, [3, 13, 1]),         # period 1, T > L
                                          (12, 2, 6, 4, [4, 4, 4, 4])])
def test_ring_add_sample_and_set_priorities(L, E, S, p, adds):
    """Rows, carries at item starts, priorities after every add, stratified draws with injected uniforms and set_priorities with
    duplicate indices, all exactly against the oracle."""
    dev, ops = _dev(), _ops()
    D, Cd = 5, 6
    ring, ref = ops.R2d2Ring(L, E, D, Cd, S, p, 0.9, dev), orc.Ring(L, E, S, p, 0.9)
    g = torch.Generator().manual_seed(L * 31 + E)
    for T in adds:
        bt = _batch(T, E, D, Cd, g)
        ops.r2d2_ring_add(ring, *(bt[k].to(dev) for k in ("obs", "action", "reward", "done", "truncated", "reset", "carry")))
        ref.add(**{k: v.numpy() for k, v in bt.items()})
        torch.cuda.synchronize()
        assert ring.state.tolist() == [ref.w, ref.c]
        np.testing.assert_array_equal(ring.priorities.cpu().numpy(), ref.leaves.astype(np.float32))
    for name in ("obs", "action", "reward", "done", "truncated", "reset"):
        np.testing.assert_array_equal(getattr(ring, name).cpu().numpy(), ref.rows[name])
    np.testing.assert_array_equal(ring.carry.cpu().numpy(), ref.carry)
    assert ref.valid_items()
    # raise some priorities (duplicates: the last occurrence wins), then draw with injected uniforms
    items = np.array(ref.valid_items())
    idx = np.concatenate([items, items[:2]]).astype(np.int32)
    pr = np.abs(np.random.default_rng(L).normal(size=idx.size)).astype(np.float32) + 0.1
    ops.r2d2_ring_set_priorities(ring, torch.tensor(idx, device=dev), torch.tensor(pr, device=dev))
    ref.set_priorities(idx, pr)
    torch.cuda.synchronize()
    np.testing.assert_allclose(ring.priorities.cpu().numpy(), ref.leaves, rtol=1e-6)   # powf: within an ulp or two of numpy's
    assert abs(float(ring.max_priority.item()) - ref.max_priority) <= 1e-6 * ref.max_priority
    ref.leaves = ring.priorities.cpu().numpy().astype(np.float64)   # the draws below are checked exactly on the device's leaves
    B = 9
    u = torch.rand(B, generator=g)
    u[0], u[-1] = 0.0, 0.9999999
    out = dict(obs=torch.zeros(S, B, D), action=torch.zeros(S, B, dtype=torch.int32), reward=torch.zeros(S, B), done=torch.zeros(S, B, dtype=torch.uint8),
               reset=torch.zeros(S, B, dtype=torch.uint8), carry0=torch.zeros(B, Cd), idx=torch.zeros(B, dtype=torch.int32), prob=torch.zeros(B))
    out = {k: v.to(dev) for k, v in out.items()}
    ops.r2d2_ring_sample(ring, 0, *out.values(), u_in=u.to(dev))
    torch.cuda.synchronize()
    want = ref.sample_items(u.numpy())
    np.testing.assert_array_equal(out["idx"].cpu().numpy(), want)
    np.testing.assert_array_equal(out["prob"].cpu().numpy(), ref.probabilities(want))
    for b, i in enumerate(want):
        seq = ref.sequence(i)
        for name in ("obs", "action", "reward", "done", "reset"):
            np.testing.assert_array_equal(out[name][:, b].cpu().numpy(), seq[name])
        np.testing.assert_array_equal(out["carry0"][b].cpu().numpy(), seq["carry0"])
    # Philox draws: fresh items per call of the device counter, every one a valid item
    ctr = torch.zeros(1, dtype=torch.int64, device=dev)
    seen = []
    for _ in range(3):
        ops.r2d2_ring_sample(ring, 7, *out.values(), dev_counter=ctr)
        ops.counter_add(ctr, 1)
        seen.append(out["idx"].cpu().numpy().copy())
    assert set(np.concatenate(seen)) <= set(ref.valid_items())


def test_ring_without_a_valid_item():
    """At the reference default (L = 97, S = 80, period 40) the head often sits where no item has S rows behind it: every draw is then
    item 0 with p = 0, and the loss's importance weights stay finite."""
    dev, ops = _dev(), _ops()
    ring, ref = ops.R2d2Ring(97, 2, 3, 4, 80, 40, 0.9, dev), orc.Ring(97, 2, 80, 40, 0.9)
    g = torch.Generator().manual_seed(5)
    for T in (128, 40):
        bt = _batch(T, 2, 3, 4, g)
        ops.r2d2_ring_add(ring, *(bt[k].to(dev) for k in ("obs", "action", "reward", "done", "truncated", "reset", "carry")))
        ref.add(**{k: v.numpy() for k, v in bt.items()})
    assert ref.valid_items() == [] and not ring.priorities.any()
    B = 4
    out = [torch.zeros(80, B, 3), torch.zeros(80, B, dtype=torch.int32), torch.zeros(80, B), torch.zeros(80, B, dtype=torch.uint8),
           torch.zeros(80, B, dtype=torch.uint8), torch.zeros(B, 4), torch.full((B,), 5, dtype=torch.int32), torch.ones(B)]
    out = [t.to(dev) for t in out]
    ops.r2d2_ring_sample(ring, 3, *out)
    assert out[6].tolist() == [0] * B and out[7].tolist() == [0.0] * B
    q = torch.randn(41, B, 2, device=dev)
    d_q, pr, m = torch.zeros_like(q), torch.zeros(B, device=dev), torch.zeros(6, device=dev)
    ops.r2d2_loss_grads(q, q.clone(), out[1][39:], out[2][39:], out[3][39:], out[7], d_q, pr, m, n=5, gamma=0.99, max_abs_reward=1000.0, eta=0.9,
                        beta0=0.6)
    assert torch.isfinite(d_q).all() and torch.isfinite(m).all()


def test_value_transform_against_fp64():
    dev, ops = _dev(), _ops()
    x = np.concatenate([[0.0, 1e-6, -1e-6, 1e-30, -3e-8], np.linspace(-2, 2, 81), np.logspace(-7, 7, 60), -np.logspace(-7, 7, 60), [3e9, -3e9]])
    x32 = torch.tensor(x, dtype=torch.float32, device=dev)
    xs = x32.double().cpu().numpy()
    for inv, f in ((False, orc.h_stable), (True, orc.h_inv_stable)):
        got = ops.r2d2_value_transform(x32, inverse=inv).double().cpu().numpy()
        want = f(xs)
        np.testing.assert_allclose(got, want, rtol=2e-6, atol=0)   # relative everywhere, including near 0 where the published forms cancel
    np.testing.assert_allclose(ops.r2d2_value_transform(ops.r2d2_value_transform(x32), inverse=True).double().cpu().numpy(), xs, rtol=1e-5, atol=1e-37)


def _loss_inputs(T, B, A, seed):
    g = torch.Generator().manual_seed(seed)
    q, q_tg = torch.randn(T, B, A, generator=g) * 3, torch.randn(T, B, A, generator=g) * 3
    q[1:, 0, :] = 0.5            # ties in the selector: the first maximum
    q[3, 1, 1:] = q[3, 1, 0]
    action = torch.randint(0, A, (T, B), generator=g, dtype=torch.int32)
    reward = torch.randn(T, B, generator=g) * 4
    reward[0, 0] = 5000.0        # clipped at max_abs_reward
    done = (torch.rand(T, B, generator=g) < 0.15).to(torch.uint8)
    done[T - 3, :] = 1           # done inside the last n-step windows
    prob = torch.rand(B, generator=g) * 0.05 + 1e-4
    return q, q_tg, action, reward, done, prob


@pytest.mark.parametrize("T,B,A,n", [(40, 32, 2, 5), (9, 5, 4, 5), (4, 3, 3, 5), (17, 64, 6, 1)])
def test_loss_against_oracle(T, B, A, n):
    """The fused loss: d Q, priorities, TD errors and metrics against the oracle; weights through the device's beta schedule; a second
    launch gives the same bits."""
    dev, ops = _dev(), _ops()
    q, q_tg, action, reward, done, prob = _loss_inputs(T, B, A, T * B)
    count = torch.tensor([7], dtype=torch.int32, device=dev)
    beta = orc.beta_at(7, 0.6, 20.0)
    outs = []
    for _ in range(2):
        d_q, pr, metrics, td = torch.zeros(T, B, A, device=dev), torch.zeros(B, device=dev), torch.zeros(6, device=dev), torch.zeros(T - 1, B, device=dev)
        ops.r2d2_loss_grads(q.to(dev), q_tg.to(dev), action.to(dev), reward.to(dev), done.to(dev), prob.to(dev), d_q, pr, metrics, n=n, gamma=0.99,
                            max_abs_reward=1000.0, eta=0.9, beta0=0.6, beta_steps=20.0, count=count, td=td)
        outs.append((d_q.cpu(), pr.cpu(), metrics.cpu(), td.cpu()))
    for x, y in zip(*outs):
        assert torch.equal(x, y)
    ref = orc.loss(q.numpy(), q_tg.numpy(), action.numpy(), reward.numpy(), done.numpy(), prob.numpy(), n, 0.99, 1000.0, 0.9, beta)
    d_q, pr, metrics, td = (x.double().numpy() for x in outs[0])
    scale = np.abs(ref["td"]).max()
    np.testing.assert_allclose(td, ref["td"], rtol=1e-4, atol=1e-5 * scale)
    np.testing.assert_allclose(d_q, ref["d_q"], rtol=1e-4, atol=1e-5 * np.abs(ref["d_q"]).max())
    np.testing.assert_allclose(pr, ref["priorities"], rtol=1e-4, atol=1e-6 * scale)
    np.testing.assert_allclose(metrics, ref["metrics"], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("A", [2, 7])
def test_dueling_head_forward_and_backward(A):
    """The post-torso + advantage branch as one MLP with a final LayerNorm, the combine with the value LayerNorm bias, and the backward
    against float64 autograd of the reference's DuelingQNetwork; every value-branch gradient but that bias is exactly zero."""
    dev, ops = _dev(), _ops()
    from tests.test_oracle_r2d2 import _layout
    lay, net = _layout("gru", dueling=True, H=64, sizes=48, A=A)
    tree = net.init(3, torch.zeros(1, 64), (torch.zeros(1, 1, 4), torch.zeros(1, 1, dtype=torch.bool)))
    flat = tree.flat.clone()
    # seeded: a row whose two pre-norm advantages nearly tie sits where a LayerNorm over two values is ill-conditioned (its gradient
    # grows as eps / gap^3), and fp32 against fp64 there can differ by more than the tolerance; these draws keep away from that
    g0 = torch.Generator().manual_seed(11 + A)
    flat[lay.off_post:lay.off_value] += 0.05 * torch.randn(lay.off_value - lay.off_post, generator=g0)   # LayerNorm scales / biases off 1 / 0
    flat[lay.off_value:] += 0.1 * torch.randn(lay.param_count - lay.off_value, generator=g0)
    M = 333
    x = torch.randn(M, 64, generator=g0)
    dq = torch.randn(M, A, generator=g0)
    fd, xd = flat.to(dev), x.to(dev)
    ws = ops.mlp_train_workspace(lay.spec_post, M, dev)
    adv = ops.mlp_forward_train(lay.spec_post, lay.blocks(fd)[3], xd, ws)
    q = ops.dueling_q(adv, lay.value_bias(fd))
    grads = torch.zeros(lay.param_count, device=dev)
    d_adv = torch.zeros(M, A, device=dev)
    ops.dueling_q_backward(dq.to(dev), d_adv, lay.value_bias(grads), weight=0.5)
    ops.mlp_backward(lay.spec_post, lay.blocks(fd)[3], xd, d_adv, ws, net_grad=lay.blocks(grads)[3], grad_weight=0.5)
    torch.cuda.synchronize()
    f64 = flat.double().requires_grad_(True)
    out = orc._mlp(lay.spec_post, lay.blocks(f64)[3], x.double())
    # the value branch in full, on the post-torso output: its final LayerNorm over one element returns its bias
    sp = lay.spec_post
    torso = ops.MlpSpec(sp.sizes[:2] + (1,), "relu", True)            # post-torso layer 0 (+ an unused head)
    p64 = lay.blocks(f64)[3]
    h1 = torch.relu(torch.nn.functional.layer_norm(x.double() @ p64[torso.layer_slices()[0][0]].view(64, 48), (48,), p64[torso.layer_slices()[0][1]],
                                                   p64[torso.ln_bias_slices()[0]], eps=1e-6))
    v = orc._mlp(lay.spec_value, f64[lay.off_value:], h1)
    q64 = v + (out - out.mean(-1, keepdim=True))
    (0.5 * (q64 * dq.double()).sum()).backward()
    np.testing.assert_allclose(q.cpu().double().numpy(), q64.detach().numpy(), rtol=1e-4, atol=1e-5)
    g = grads.cpu().double().numpy()
    gw = f64.grad.numpy()
    np.testing.assert_allclose(g[lay.off_post:lay.param_count], gw[lay.off_post:lay.param_count], rtol=2e-3, atol=2e-4 * np.abs(gw).max())
    vb = lay.off_value + lay.spec_value.ln_bias_slices()[-1].start
    rest = np.delete(g[lay.off_value:lay.param_count], vb - lay.off_value)
    assert not rest.any() and g[vb] != 0.0
    # autograd through torch's one-element LayerNorm leaves rounding residue only (the exact gradient is zero)
    assert np.abs(np.delete(gw[lay.off_value:lay.param_count], vb - lay.off_value)).max() < 1e-10 * abs(gw[vb])


def _config(overrides=()):
    from stoix_b200.config import compose
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps
    cfg = compose("default_rec_r2d2", ["arch.total_num_envs=16", "arch.total_timesteps=~", "arch.num_updates=4", "arch.num_evaluation=1",
                                       "system.epochs=2", "system.rollout_length=8", "system.period=4", "system.sample_sequence_length=12",
                                       "system.burn_in_length=4", "system.warmup_steps=20", "system.total_buffer_size=384", "system.total_batch_size=6",
                                       "arch.num_eval_episodes=4", "logger.use_console=False", *overrides], config_dir="default/anakin")
    cfg.num_devices = 1
    return check_total_timesteps(cfg, quiet=True)


def _setup(overrides=()):
    from stoix_b200 import random as srandom
    from stoix_b200.systems.q_learning import rec_r2d2
    from stoix_b200.utils import make_env as environments
    cfg = _config(overrides)
    env, _ = environments.make(config=cfg)
    key, _, q_key = srandom.split(srandom.PRNGKey(cfg.arch.seed), num=3)
    learn, net, state = rec_r2d2.learner_setup(env, (key, q_key), cfg)
    return cfg, learn, state


_NETS = [(), ("network=rnn_dqn",), ("network.actor_network.rnn_layer.cell_type=lstm",),
         ("network=rnn_dqn", "network.actor_network.rnn_layer.cell_type=lstm")]


@pytest.mark.parametrize("overrides", _NETS)
def test_teacher_forced_gradients_and_optimiser_step(overrides):
    """One epoch on a sampled batch with injected uniforms: the device's gradient against float64 autograd of the reference's loss fed the
    same batch (burn-in and targets under stop_gradient), the priorities, and the parameters after the clip + Adam step and Polyak."""
    dev = _dev()
    cfg, learn, state = _setup(overrides)
    learn.ensure_built(state)
    b = learn.built
    lay, bt, buf = b["layout"], b["batches"][0], state.buffer_state[0]
    sysc = cfg.system
    B = int(sysc.batch_size)
    buf.sample_into(bt.obs, bt.action, bt.reward, bt.done, bt.reset, bt.carry0, bt.idx, bt.prob, u_in=torch.rand(B, device=dev))
    online, target = state.params.online, state.params.target
    target.arena.add_(1e-3 * torch.randn_like(target.arena))      # target != online
    p0, t0 = online.arena.clone(), target.arena.clone()
    learn.update_epoch(state, 0, sample=False)
    torch.cuda.synchronize()
    seq = {k: getattr(bt, k).cpu().numpy() for k in ("obs", "action", "reward", "done", "reset", "carry0")}
    P = lay.param_count
    g, ref = orc.q_loss_grad(lay, p0[:P].double().cpu().numpy(), t0[:P].double().cpu().numpy(), seq, int(sysc.burn_in_length),
                             bt.prob.cpu().numpy(), int(sysc.n_step), float(sysc.gamma), float(sysc.max_abs_reward), float(sysc.priority_eta),
                             orc.beta_at(0, float(sysc.importance_sampling_exponent), float(cfg.arch.num_updates) * int(sysc.epochs)))
    gd = b["grads"][:P].double().cpu().numpy()
    np.testing.assert_allclose(gd, g, rtol=2e-3, atol=2e-4 * np.abs(g).max())
    np.testing.assert_allclose(b["work"].priorities.cpu().numpy(), ref["priorities"], rtol=1e-3, atol=1e-5)
    np.testing.assert_allclose(b["metrics"][0].cpu().double().numpy(), ref["metrics"], rtol=1e-3, atol=1e-5)
    new, _, _ = orc.clip_adam(p0[:P].double().cpu().numpy(), gd, np.zeros(P), np.zeros(P), 0, float(sysc.q_lr), float(sysc.max_grad_norm))
    np.testing.assert_allclose(online.arena[:P].double().cpu().numpy(), new, rtol=1e-5, atol=1e-6)
    tau = float(sysc.tau)
    np.testing.assert_allclose(target.arena[:P].double().cpu().numpy(), (1 - tau) * t0[:P].double().cpu().numpy() + tau * new, rtol=1e-5, atol=1e-6)
    if lay.dueling:   # the value branch moves only through its final LayerNorm bias
        vb = lay.off_value + lay.spec_value.ln_bias_slices()[-1].start
        moved = (online.arena[lay.off_value:P] != p0[lay.off_value:P]).nonzero().flatten().cpu().tolist()
        assert moved == [vb - lay.off_value]


@pytest.mark.parametrize("overrides", [(), ("network.actor_network.rnn_layer.cell_type=lstm",)])
def test_updates_eager_captured_replayed(overrides):
    """Three whole updates (eager, captured, replayed): finite metrics, the parameters and target move, and replays draw fresh sequences."""
    _dev()
    from stoix_b200.systems import anakin
    cfg, learn, state = _setup(overrides)
    learn.ensure_built(state)
    b = learn.built
    seen = []
    for k in range(3):
        p, t = state.params.online.arena.clone(), state.params.target.arena.clone()
        anakin.update_once(b, True, learn.update_step, state, state.buffer_state, int(cfg.system.rollout_length) * int(cfg.arch.num_envs))
        torch.cuda.synchronize()
        assert torch.isfinite(b["metrics"]).all()
        assert not torch.equal(state.params.online.arena, p) and not torch.equal(state.params.target.arena, t)
        seen.append(b["batches"][0].obs.clone())
    assert b["graph"] is not None
    assert not torch.equal(seen[1], seen[2])


def test_eager_and_replayed_update_bit_identical():
    """The same updates run eagerly and replayed from a captured graph from the same state give the same bits."""
    _dev()
    from stoix_b200.systems import anakin
    outs = []
    for use_graph in (False, True):
        cfg, learn, state = _setup()
        learn.ensure_built(state)
        b = learn.built
        items = int(cfg.system.rollout_length) * int(cfg.arch.num_envs)
        for _ in range(3):
            anakin.update_once(b, use_graph, learn.update_step, state, state.buffer_state, items)
        torch.cuda.synchronize()
        outs.append((state.params.online.arena.clone(), state.params.target.arena.clone(), b["metrics"].clone(),
                     state.buffer_state[0].ring.tree.clone(), b["shards"][0].h_cur.clone()))
    for x, y in zip(*outs):
        assert torch.equal(x, y)


_ENTRY = ["arch.total_num_envs=16", "arch.total_timesteps=~", "arch.num_updates=4", "arch.num_evaluation=2", "system.epochs=2",
          "system.rollout_length=8", "system.period=4", "system.sample_sequence_length=12", "system.burn_in_length=4", "system.warmup_steps=20",
          "system.total_buffer_size=384", "system.total_batch_size=6", "arch.absolute_metric=True", "logger.checkpointing.save_model=True",
          "arch.num_eval_episodes=4", "arch.max_eval_steps=50", "logger.use_console=False", "logger.checkpointing.save_args.checkpoint_uid=warm",
          "logger.checkpointing.load_args.checkpoint_uid=warm"]


def test_entry_point_with_checkpoint_and_warm_start(tmp_path, monkeypatch):
    """The entry point runs, checkpoints the online network, and a warm start loads those parameters into both arenas."""
    _dev()
    from stoix_b200 import random as srandom
    from stoix_b200.config import compose
    from stoix_b200.systems.q_learning import rec_r2d2
    from stoix_b200.utils import make_env
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    torch.cuda.set_device(0)
    monkeypatch.chdir(tmp_path)
    assert np.isfinite(rec_r2d2.hydra_entry_point(compose("default_rec_r2d2", _ENTRY, config_dir="default/anakin")))
    saved = sorted(q for q in tmp_path.glob("checkpoints/*/warm/*.pt") if q.stem.isdigit())
    assert saved, "no checkpoint written"
    blob = torch.load(saved[-1], map_location="cpu")
    cfg = compose("default_rec_r2d2", _ENTRY + ["logger.checkpointing.load_model=True"], config_dir="default/anakin")
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, _ = make_env.make(cfg)
    keys = srandom.split(srandom.PRNGKey(0), 2)
    _, _, state = rec_r2d2.learner_setup(env, (keys[0], keys[1]), cfg)
    P = state.params.online.layout.param_count
    assert torch.equal(state.params.online.flat.cpu(), blob["params"][:P])
    assert torch.equal(state.params.target.flat.cpu(), blob["params"][:P])


def test_cartpole_learning():
    """rec_r2d2 on CartPole at the reference default with the plain Q head (network=rnn_dqn), 1e7 steps.  Measured on an H100 80GB
    HBM3 at 700 W: 363.8 (absolute metric; 500 with period 1); a random policy scores about 20.  The bar is 150.

    The default dueling head does not learn CartPole here: with A = 2 the advantage branch's final LayerNorm maps the two pre-norm
    values to +-1 (times its scale, plus its bias) whatever their size, so almost no gradient reaches below it, and the value branch's
    one-element LayerNorm outputs a constant.  Measured: 9.4 at 1e7 steps with either period.  The reference's network has the same
    LayerNorms; that it fails the same way is argued from that, not measured."""
    _dev()
    from stoix_b200.systems.q_learning import rec_r2d2
    r = rec_r2d2.hydra_entry_point(overrides=["network=rnn_dqn", "logger.use_console=False"])
    print(f"rec_r2d2 (rnn_dqn) CartPole evaluation: {r:.1f}")
    assert r >= 150.0


def test_two_ranks():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import os
    import subprocess
    import sys
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nproc_per_node=2", "-m", "stoix_b200.systems.q_learning.rec_r2d2", "arch.total_num_envs=32",
           "arch.total_timesteps=~", "arch.num_updates=2", "arch.num_evaluation=1", "system.epochs=2", "system.rollout_length=8", "system.period=4",
           "system.sample_sequence_length=12", "system.burn_in_length=4", "system.warmup_steps=20", "system.total_buffer_size=768",
           "system.total_batch_size=6", "arch.num_eval_episodes=4", "logger.use_console=False"]
    r = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ), timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
