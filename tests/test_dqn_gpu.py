"""The DQN family on the GPU through the C ABI and the learner, against the NumPy oracle (tests/dqn_oracle.py)."""
import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from stoix_b200 import ops
from tests import dqn_oracle as Q
from tests import pqn_oracle as P

pytestmark = pytest.mark.gpu

f64 = lambda t: t.detach().double().cpu().numpy()
RULES = ["q_learning", "double_q_learning", "munchausen_q_learning", "q_learning_reg"]
SYSTEMS = {"ff_dqn": "q_learning", "ff_ddqn": "double_q_learning", "ff_mdqn": "munchausen_q_learning", "ff_dqn_reg": "q_learning_reg"}


def _ring_equals(ring: ops.DiscreteReplayRing, ref: Q.Ring) -> None:
    np.testing.assert_array_equal(ring.obs.cpu().numpy(), ref.obs)
    np.testing.assert_array_equal(ring.next_obs.cpu().numpy(), ref.next_obs)
    np.testing.assert_array_equal(ring.action.cpu().numpy(), ref.action)
    np.testing.assert_array_equal(ring.reward.cpu().numpy(), ref.reward)
    np.testing.assert_array_equal(ring.done.cpu().numpy(), ref.done)
    assert ring.state.cpu().tolist() == [ref.pos, ref.size]


def test_discrete_ring_bit_exact():
    """Adds that wrap around and one with more rows than slots; samples from the Philox words, equal to stx_uniform_indices."""
    rng = np.random.default_rng(0)
    cap, D = 1000, 7
    ring, ref = ops.DiscreteReplayRing(cap, D, "cuda"), Q.Ring(cap, D)
    seed, M = 0x1234_5678_9AB, 777
    ctr = torch.tensor([5], dtype=torch.int64, device="cuda")
    for T, E in ((3, 100), (4, 256), (1, 1500), (2, 333)):
        obs = rng.normal(size=(T, E, D)).astype(np.float32)
        nxt = rng.normal(size=(T, E, D)).astype(np.float32)
        act = rng.integers(0, 9, size=(T, E)).astype(np.int32)
        rew = rng.normal(size=(T, E)).astype(np.float32)
        done = (rng.random((T, E)) < 0.3).astype(np.uint8)
        t = lambda x: torch.tensor(x, device="cuda")
        ops.replay_add_discrete(ring, t(obs), t(act), t(rew), t(done), t(nxt))
        ref.add(obs, act, rew, done, nxt)
        _ring_equals(ring, ref)
        xs = torch.empty(2 * M, D, device="cuda")
        a, r, d, idx = (torch.empty(M, dtype=dt, device="cuda") for dt in (torch.int32, torch.float32, torch.uint8, torch.int32))
        ops.replay_sample_discrete(ring, M, seed, xs[:M], xs[M:], a, r, d, offset=2, dev_counter=ctr, idx_out=idx)
        o_w, n_w, a_w, r_w, d_w, j_w = ref.sample(M, seed, 2 + 5)
        np.testing.assert_array_equal(idx.cpu().numpy(), j_w)
        np.testing.assert_array_equal(idx.cpu().numpy(), ops.uniform_indices(M, ring.state[1:2], seed, 2, dev_counter=ctr).cpu().numpy())
        np.testing.assert_array_equal(xs[:M].cpu().numpy(), o_w)
        np.testing.assert_array_equal(xs[M:].cpu().numpy(), n_w)
        for got, want in ((a, a_w), (r, r_w), (d, d_w)):
            np.testing.assert_array_equal(got.cpu().numpy(), want)
    idx_in = torch.tensor(rng.integers(0, cap, size=M).astype(np.int32), device="cuda")   # injected indices
    ops.replay_sample_discrete(ring, M, seed, xs[:M], xs[M:], a, r, d, idx_in=idx_in)
    np.testing.assert_array_equal(r.cpu().numpy(), ref.reward[idx_in.cpu().numpy()])


def _loss_case(rule, rng, M, A):
    """Q rows with argmax ties (DDQN), done rows (terminal and truncated alike), clipped rewards; MDQN at |q / tau| ~ 1e3."""
    q_tm1 = rng.normal(size=(M, A)).astype(np.float32)
    q_t = rng.normal(size=(M, A)).astype(np.float32)
    q_aux = rng.normal(size=(M, A)).astype(np.float32)
    if rule == "double_q_learning":
        q_aux = (rng.integers(0, 3, size=(M, A)) * 0.5).astype(np.float32)
    if rule == "munchausen_q_learning":
        q_t, q_aux = q_t * 30, q_aux * 30
    action = rng.integers(0, A, size=M).astype(np.int32)
    reward = (rng.normal(size=M) * 3).astype(np.float32)
    done = (rng.random(M) < 0.25).astype(np.uint8)
    return q_tm1, q_t, q_aux, action, reward, done


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("huber", [0.0, 1.0])
def test_loss_kernel_against_the_oracle(rule, huber):
    rng = np.random.default_rng(RULES.index(rule) * 7 + int(huber))
    M, A = 3000, 6
    h = Q.LossHyper(gamma=0.99, max_abs_reward=2.0, huber=huber, tau=0.03, alpha=0.9, clip_value_min=-20.0, reg=0.1)
    q_tm1, q_t, q_aux, action, reward, done = _loss_case(rule, rng, M, A)
    hy = ops.q_td_hyper(gamma=h.gamma, max_abs_reward=h.max_abs_reward, huber_delta=huber, entropy_temperature=h.tau,
                        munchausen_coefficient=h.alpha, clip_value_min=h.clip_value_min, regularizer_coeff=h.reg if rule == "q_learning_reg" else 0.0)
    t = lambda x: torch.tensor(x, device="cuda")
    aux = t(q_aux) if rule in ("double_q_learning", "munchausen_q_learning") else None
    runs = []
    for _ in range(2):
        dq, metrics = torch.full((M, A), 9.0, device="cuda"), torch.zeros(2, device="cuda")
        ops.q_td_loss_grads(rule, t(q_tm1), t(q_t), t(action), t(reward), hy, dq, metrics, done=t(done), q_aux=aux, weight=0.5)
        runs.append((dq, metrics))
    torch.cuda.synchronize()
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    # the oracle on the fp32 inputs, with the fp32 discount the kernel forms
    loss, want = Q.loss_and_dq(rule, q_tm1, q_t.astype(np.float64), None if aux is None else q_aux.astype(np.float64), action, reward, done, h)
    np.testing.assert_allclose(f64(runs[0][0]), want, rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(runs[0][1][0].item(), 0.5 * loss, rtol=1e-5)
    assert runs[0][1][1].item() == 0.0
    if rule == "double_q_learning":   # ties among the selector's maxima: the first index (jnp.argmax)
        assert (q_aux == q_aux.max(1, keepdims=True)).sum(1).max() > 1


def test_loss_faces_match_the_oracle():
    from stoix_b200.utils import loss as L

    rng = np.random.default_rng(9)
    M, A = 500, 4
    t = lambda x: torch.tensor(x, device="cuda")
    q_tm1, q_t, q_aux, a, r, _ = _loss_case("munchausen_q_learning", rng, M, A)
    d_t = (rng.random(M) * 0.99).astype(np.float32)
    h = Q.LossHyper(huber=1.0, tau=0.03, alpha=0.9, clip_value_min=-1e3)
    for rule, got in (("q_learning", L.q_learning(t(q_tm1), t(a), t(r), t(d_t), t(q_t), 1.0)),
                      ("double_q_learning", L.double_q_learning(t(q_tm1), t(q_t), t(a), t(r), t(d_t), t(q_aux), 1.0)),
                      ("munchausen_q_learning", L.munchausen_q_learning(t(q_tm1), t(q_aux), t(a), t(r), t(d_t), t(q_t), 0.03, 0.9, -1e3, 1.0))):
        want, _ = Q.loss_and_dq(rule, q_tm1, q_t, q_aux, a, r, None, h, discount=d_t)
        np.testing.assert_allclose(got.item(), want, rtol=1e-5, err_msg=rule)


@pytest.mark.parametrize("rule", RULES)
def test_epoch_gradient_teacher_forced(rule):
    """ff_dqn.batch_grads, the learner's gradient of one epoch, on given batches: two shards (weight 1/2 each, the first overwrites
    a dirty arena) against the fp64 oracle, 1e-5 norm-wise; bit-identical on repeat."""
    from stoix_b200.systems.q_learning import ff_dqn

    rng = np.random.default_rng(RULES.index(rule))
    D, A, M = 10, 5, 384
    spec = ops.MlpSpec((D, 64, 64, A), activation="silu", use_layer_norm=False)
    sizes = list(spec.sizes)
    on = (rng.normal(size=spec.param_count) * 0.2).astype(np.float32)
    tg = (on + rng.normal(size=spec.param_count) * 0.02).astype(np.float32)
    h = Q.LossHyper(gamma=0.99, max_abs_reward=2.0, huber=1.0, tau=0.5, alpha=0.9, clip_value_min=-1e3, reg=0.1)
    hy = ops.q_td_hyper(gamma=h.gamma, max_abs_reward=h.max_abs_reward, huber_delta=h.huber, entropy_temperature=h.tau, munchausen_coefficient=h.alpha,
                        clip_value_min=h.clip_value_min, regularizer_coeff=h.reg if rule == "q_learning_reg" else 0.0)
    on_p = O.MLPParams.from_flat(on.astype(np.float64), sizes, "silu", False)
    tg_p = O.MLPParams.from_flat(tg.astype(np.float64), sizes, "silu", False)
    t = lambda x: torch.tensor(x, device="cuda")
    batches, want, loss = [], np.zeros(spec.param_count), 0.0
    for _ in range(2):
        obs, nxt = rng.normal(size=(M, D)).astype(np.float32), rng.normal(size=(M, D)).astype(np.float32)
        a = rng.integers(0, A, size=M).astype(np.int32)
        r = (rng.normal(size=M) * 3).astype(np.float32)
        d = (rng.random(M) < 0.2).astype(np.uint8)
        batches.append(ff_dqn.Batch(t(np.concatenate([obs, nxt])), t(a), t(r), t(d)))
        l, g = Q.batch_grad(rule, on_p, tg_p, obs, nxt, a, r, d, h)
        want += 0.5 * g
        loss += 0.5 * l
    work = ff_dqn.make_work(spec, M, "cuda")
    got = []
    for _ in range(2):
        grads, metric = torch.full((spec.param_count,), 7.0, device="cuda"), torch.zeros(1, device="cuda")
        ff_dqn.batch_grads(rule, spec, t(on), t(tg), batches, hy, grads, metric, work)
        got.append((grads, metric))
    torch.cuda.synchronize()
    assert torch.equal(got[0][0], got[1][0]) and torch.equal(got[0][1], got[1][1])
    g = f64(got[0][0])
    assert np.linalg.norm(g - want) <= 1e-5 * np.linalg.norm(want), np.linalg.norm(g - want) / np.linalg.norm(want)
    np.testing.assert_allclose(got[0][1].item(), loss, rtol=1e-5)


def _learner(system, E, T, epochs, batch, extra=(), env_name="synthetic/box", updates=40, U=1):
    import importlib

    from stoix_b200 import random as srandom
    from stoix_b200.config import compose
    from stoix_b200.utils import make_env
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    mod = importlib.import_module(f"stoix_b200.systems.q_learning.{system}")
    ov = [f"env={env_name}", f"arch.total_num_envs={E * U}", f"arch.update_batch_size={U}", f"system.rollout_length={T}", f"system.epochs={epochs}",
          f"system.total_batch_size={batch * U}", f"arch.total_timesteps={E * U * T * updates}", "arch.num_evaluation=1",
          "logger.use_console=False"] + list(extra)
    cfg = compose(f"default_{system}", ov, config_dir="default/anakin")
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, eval_env = make_env.make(cfg)
    keys = srandom.split(srandom.PRNGKey(3), 2)
    learn, eval_net, state = mod.learner_setup(env, (keys[0], keys[1]), cfg)
    return cfg, learn, eval_net, state, eval_env


_SMALL = ["env.kwargs.obs_dim=8", "env.kwargs.num_actions=4", "network.actor_network.pre_torso.layer_sizes=[32,32]", "system.q_lr=1e-2",
          "system.warmup_steps=3", "system.total_buffer_size=400", "system.max_abs_reward=1.5", "system.tau=0.3"]


@pytest.mark.parametrize("system", list(SYSTEMS))
@pytest.mark.parametrize("huber", [0.0, 1.0])
def test_three_updates_eager_and_graph_match_the_oracle(system, huber):
    """Three whole updates (eager, graph capture, replay): every rollout action re-drawn from the stored Q rows, the ring after the
    add bit-exact (the warm-up rows included), and online and target parameters against the oracle, which samples the same
    indices from its own copy of the ring."""
    rule = SYSTEMS[system]
    E, T, epochs, M = 64, 2, 3, 96
    extra = _SMALL + [f"system.huber_loss_parameter={huber}"] + (["system.entropy_temperature=0.5"] if rule == "munchausen_q_learning" else [])
    cfg, learn, _, state, _ = _learner(system, E, T, epochs, M, extra)
    cfg.arch.num_updates_per_eval = 1
    sysc = cfg.system
    spec = state.params.online.spec
    sizes, n = list(spec.sizes), spec.param_count
    h = Q.LossHyper(gamma=float(sysc.gamma), max_abs_reward=float(sysc.max_abs_reward), huber=huber, tau=float(sysc.get("entropy_temperature", 0.03)),
                    alpha=float(sysc.get("munchausen_coefficient", 0.9)), clip_value_min=float(sysc.get("clip_value_min", -1e3)),
                    reg=float(sysc.get("regularizer_coeff", 0.0)))
    buf = state.buffer_state[0]
    ring = buf.ring
    W = int(sysc.warmup_steps)
    assert ring.state.cpu().tolist() == [W * E, W * E]   # the warm-up rows are in the ring before the first update
    ref = Q.Ring(ring.capacity, ring.obs_dim)
    for name in ("obs", "next_obs", "action", "reward", "done"):
        getattr(ref, name)[:] = getattr(ring, name).cpu().numpy()
    ref.pos, ref.size = W * E, W * E
    online, target = f64(state.params.online.flat)[:n], f64(state.params.target.flat)[:n]
    assert (online == target).all()
    st = O.AdamState(np.zeros(n), np.zeros(n))
    eps = np.float32(sysc.training_epsilon)
    # the warm-up rows: each step's actions re-drawn from Q(initial parameters, obs) with the warm-up seed, call t; the rows chain
    # into one trajectory per env (obs[t + 1] = next_obs[t] wherever step t did not end an episode)
    init = O.MLPParams.from_flat(online, sizes, "silu", False)
    for t in range(W):
        rows = slice(t * E, (t + 1) * E)
        q_w = ops.mlp_forward(spec, state.params.online.flat, ring.obs[rows])
        np.testing.assert_allclose(f64(q_w), O.mlp_forward(init, f64(ring.obs[rows]))[0], rtol=1e-5, atol=1e-5)
        np.testing.assert_array_equal(ring.action[rows].cpu().numpy(), P.epsilon_greedy(q_w.cpu().numpy(), eps, int(state.key[1]), t),
                                      err_msg=f"warm-up step {t}")
        if t + 1 < W:
            cont = ring.done[rows].cpu().numpy() == 0
            assert cont.any()
            np.testing.assert_array_equal(ring.obs[t * E + E:(t + 2) * E].cpu().numpy()[cont], ring.next_obs[rows].cpu().numpy()[cont])
    for k in range(3):
        pre = O.MLPParams.from_flat(f64(state.params.online.flat)[:n], sizes, "silu", False)
        call0 = int(buf.counter.item())
        out = learn(state)
        torch.cuda.synchronize()
        assert (learn.built["graph"] is not None) == (k >= 1)
        ro = learn.built["rollouts"][0]
        q_roll, _ = O.mlp_forward(pre, f64(ro.obs[:T]).reshape(T * E, -1))
        np.testing.assert_allclose(f64(ro.q).reshape(T * E, -1), q_roll, rtol=1e-5, atol=1e-5)
        for t in range(T):
            want = P.epsilon_greedy(ro.q[t].cpu().numpy(), eps, int(state.key[0]), t + k * T)
            np.testing.assert_array_equal(ro.action[t].cpu().numpy(), want, err_msg=f"update {k} step {t}")
        ref.add(ro.obs[:T].cpu().numpy(), ro.action.cpu().numpy(), ro.reward.cpu().numpy(), ro.done.cpu().numpy(), ro.next_obs.cpu().numpy())
        _ring_equals(ring, ref)
        assert (ro.done.cpu().numpy() == (ro.terminated.cpu().numpy() | ro.truncated.cpu().numpy())).all()
        eps_batches = [[ref.sample(M, buf.seed, call0 + ep)[:5]] for ep in range(epochs)]
        online, target = Q.dqn_update(rule, online, target, st, eps_batches, h, float(sysc.q_lr), float(sysc.max_grad_norm), float(sysc.tau), sizes,
                                      "silu", False)
        np.testing.assert_allclose(f64(out.learner_state.params.online.flat)[:n], online, rtol=1e-4, atol=2e-6, err_msg=f"online, update {k}")
        np.testing.assert_allclose(f64(out.learner_state.params.target.flat)[:n], target, rtol=1e-4, atol=2e-6, err_msg=f"target, update {k}")
        assert int(buf.counter.item()) == call0 + epochs
        state = out.learner_state
    assert out.train_metrics["q_loss"].shape == (1, epochs)
    assert set(out.episode_metrics) >= {"episode_return", "episode_length", "is_terminal_step"}
    assert int(state.params.online.arena_counts[0]) == 3 * epochs
    assert buf.added == (W + 3 * T) * E


def test_graph_replays_draw_fresh_actions_and_indices_and_shards_differ():
    cfg, learn, _, state, _ = _learner("ff_dqn", 64, 2, 2, 64, _SMALL, U=2)
    cfg.arch.num_updates_per_eval = 1
    seen = []
    for _ in range(3):
        state = learn(state).learner_state
        torch.cuda.synchronize()
        ros, bts = learn.built["rollouts"], learn.built["batches"]
        seen.append((ros[0].action.clone(), bts[0].xs.clone()))
        assert not torch.equal(ros[0].obs, ros[1].obs) and not torch.equal(bts[0].xs, bts[1].xs)
    assert not torch.equal(seen[1][0], seen[2][0]) and not torch.equal(seen[1][1], seen[2][1])


def test_bf16_is_refused():
    with pytest.raises(ValueError, match="bf16"):
        _learner("ff_dqn", 64, 2, 2, 64, _SMALL + ["arch.precision=bf16"])


@pytest.mark.parametrize("system", ["ff_dqn", "ff_ddqn"])
def test_cartpole_learns(system):
    """CartPole at the reference's hyper-parameters (1024 envs, T = 2, 16 epochs of batch 512, tau 0.005, lr 5e-4, epsilon 0.1),
    192 updates, evaluated greedily every 16 updates.  A uniform policy returns about 22, and greedy returns swing between
    evaluations, so the test reads the best one and the training episodes of the last 16 updates.  Measured on an H100 80GB HBM3
    with this seed: ff_dqn evaluations 10.1, 11.9, 13.7, 15.1, 152.0, 241.7, 186.4, 220.8, 217.2, 215.2, 283.3, 318.4, training
    return 211.8; ff_ddqn 9.8, 10.7, 13.6, 14.7, 25.0, 267.9, 181.6, 210.6, 190.3, 220.9, 283.7, 315.9, training return 208.4.
    Bars: 150 and 80."""
    from stoix_b200 import random as srandom
    from stoix_b200.evaluator import get_distribution_act_fn, get_ff_evaluator_fn

    cfg, learn, eval_net, state, eval_env = _learner(system, 1024, 2, 16, 512, [], env_name="gymnax/cartpole", updates=400)
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


WORKER = r'''
import os, sys, json
import numpy as np
import torch, torch.distributed as dist
sys.path.insert(0, os.getcwd())
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
cpu_group = dist.new_group(backend="gloo")       # carries the ORACLE's gradient exchange (CPU tensors)
from oracle import ppo_oracle as O
from tests import dqn_oracle as Q
from stoix_b200 import random as srandom
from stoix_b200.config import compose
from stoix_b200.systems.q_learning import SYSTEM as mod
from stoix_b200.utils import make_env
from stoix_b200.utils.total_timestep_checker import check_total_timesteps
E, T, epochs, M, n_upd = 64, 2, 3, 96, 3
cfg = compose("default_SYSTEM", ["env=synthetic/box", f"arch.total_num_envs={E * world}", f"system.rollout_length={T}", f"system.epochs={epochs}",
                                 f"system.total_batch_size={M * world}", f"arch.total_timesteps={E * world * T * n_upd}", "arch.num_evaluation=1",
                                 "logger.use_console=False", "env.kwargs.obs_dim=8", "env.kwargs.num_actions=4",
                                 "network.actor_network.pre_torso.layer_sizes=[32,32]", "system.q_lr=1e-2", "system.warmup_steps=3",
                                 f"system.total_buffer_size={400 * world}", "system.max_abs_reward=1.5", "system.tau=0.3",
                                 "system.huber_loss_parameter=1.0"], config_dir="default/anakin")
cfg.num_devices, cfg.rank = world, rank
cfg = check_total_timesteps(cfg, quiet=True)
assert cfg.arch.num_envs == E and cfg.arch.num_updates == n_upd
env, _ = make_env.make(cfg)
keys = srandom.split(srandom.PRNGKey(cfg.arch.seed), 2)
learn, _, state = mod.learner_setup(env, (keys[0], keys[1]), cfg)
assert int(cfg.system.batch_size) == M
cfg.arch.num_updates_per_eval = 1
f64 = lambda t: t.detach().double().cpu().numpy()
s = cfg.system
h = Q.LossHyper(gamma=float(s.gamma), max_abs_reward=float(s.max_abs_reward), huber=1.0, tau=float(s.get("entropy_temperature", 0.03)),
                alpha=float(s.get("munchausen_coefficient", 0.9)), clip_value_min=float(s.get("clip_value_min", -1e3)),
                reg=float(s.get("regularizer_coeff", 0.0)))
spec = state.params.online.spec
sizes, n = list(spec.sizes), spec.param_count

def grad_sync(g):   # pmean over "device": SUM over the ranks, then 1/world
    t = torch.from_numpy(np.ascontiguousarray(g, np.float64))
    dist.all_reduce(t, op=dist.ReduceOp.SUM, group=cpu_group)
    return t.numpy() / world

def gather_equal(x):
    xs = [torch.empty_like(x) for _ in range(world)]
    dist.all_gather(xs, x)
    return all(torch.equal(xs[0], y) for y in xs)

buf = state.buffer_state[0]
ring = buf.ring
ok, why, worst = True, "", 0.0
identical = gather_equal(state.params.online.arena) and gather_equal(state.params.target.arena)   # same initial parameters
for upd in range(n_upd):   # eager, graph capture, graph replay
    ref = Q.Ring(ring.capacity, ring.obs_dim)
    for name in ("obs", "next_obs", "action", "reward", "done"):
        getattr(ref, name)[:] = getattr(ring, name).cpu().numpy()
    ref.pos, ref.size = (int(v) for v in ring.state.cpu().tolist())
    online, target = f64(state.params.online.flat)[:n], f64(state.params.target.flat)[:n]   # every update checked on its own
    st = O.AdamState(f64(state.opt_states.mu)[:n], f64(state.opt_states.nu)[:n], upd * epochs)
    call0 = int(buf.counter.item())
    out = learn(state); state = out.learner_state
    torch.cuda.synchronize()
    ro = learn.built["rollouts"][0]
    ref.add(ro.obs[:T].cpu().numpy(), ro.action.cpu().numpy(), ro.reward.cpu().numpy(), ro.done.cpu().numpy(), ro.next_obs.cpu().numpy())
    batches = [[ref.sample(M, buf.seed, call0 + ep)[:5]] for ep in range(epochs)]
    online, target = Q.dqn_update(learn.loss, online, target, st, batches, h, float(s.q_lr), float(s.max_grad_norm), float(s.tau), sizes, "silu",
                                  False, grad_sync=grad_sync)
    for name, got, want in (("online", f64(state.params.online.flat)[:n], online), ("target", f64(state.params.target.flat)[:n], target)):
        err = float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))
        worst = max(worst, err)
        if not np.allclose(got, want, rtol=1e-4, atol=2e-6):
            ok, why = False, f"update {upd}: {name} max relative parameter error {err:.3e}"
    identical = identical and gather_equal(state.params.online.arena) and gather_equal(state.params.target.arena)
loss = out.train_metrics["q_loss"].reshape(-1).contiguous()
obs_sum = learn.built["rollouts"][0].obs[:T].sum()
sums = [torch.empty_like(obs_sum) for _ in range(world)]
dist.all_gather(sums, obs_sum)
flags = torch.tensor([1.0 if ok else 0.0], device="cuda")
dist.all_reduce(flags, op=dist.ReduceOp.MIN)
metrics_identical = gather_equal(loss)
if rank == 0:
    print(json.dumps({"oracle_ok_all_ranks": bool(flags.item() == 1.0), "why": why, "worst": worst, "params_identical_across_ranks": identical,
                      "metrics_identical_across_ranks": metrics_identical, "shards_differ": len({float(x) for x in sums}) == world,
                      "graph": learn.built["graph"] is not None, "counts": state.params.online.arena_counts.cpu().tolist()}))
dist.barrier(); torch.cuda.synchronize(); sys.stdout.flush(); os._exit(0)  # NCCL teardown can hang at exit here
'''


@pytest.mark.parametrize("system", ["ff_dqn", "ff_ddqn", "ff_mdqn", "ff_dqn_reg"])
def test_two_rank_updates_match_the_oracle(system, tmp_path):
    """Two torchrun ranks, three whole updates (eager, capture, replay) with the NCCL all-reduces of the gradient and the metrics
    inside the captured step.  Each rank replays its own rollout and ring samples through the oracle with the gradient exchange as
    a gloo all-reduce (SUM, then 1/world): online and target parameters rtol 1e-4 atol 2e-6 per update.  Online and target arenas
    (from the identical initial parameters on) and the averaged q_loss metrics bit-identical across the ranks after every update;
    the ranks' rollouts differ."""
    import json
    import os
    import subprocess
    import sys

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (NCCL refuses two ranks on one device)")
    script = tmp_path / "worker.py"
    script.write_text(WORKER.replace("SYSTEM", system))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(29531 + list(SYSTEMS).index(system)), str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=240, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    res = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    print(res)
    assert res["oracle_ok_all_ranks"], res
    assert res["params_identical_across_ranks"] and res["metrics_identical_across_ranks"] and res["shards_differ"] and res["graph"], res
    assert res["counts"] == [3 * 3, 3 * 3], res
