"""PQN on the GPU through the C ABI and the learner, against the NumPy oracle (tests/pqn_oracle.py)."""
import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from stoix_b200 import ops
from tests import pqn_oracle as P

pytestmark = pytest.mark.gpu

f64 = lambda t: t.detach().double().cpu().numpy()


def _ties_q(rng, E, A):
    """Q rows on a coarse grid, so that exact ties are common."""
    return torch.tensor(rng.integers(0, 3, size=(E, A)).astype(np.float32) * 0.5, device="cuda")


@pytest.mark.parametrize("A", [2, 5, 32])
@pytest.mark.parametrize("eps", [0.0, 0.1, 1.0])
def test_epsilon_greedy_actions_bit_exact(A, eps):
    rng = np.random.default_rng(A)
    E = 1003
    q = _ties_q(rng, E, A)
    seed, offset, ctr = 0x1234_5678_9ABC, 5, torch.tensor([3], dtype=torch.int64, device="cuda")
    sched = ops.epsilon_schedule_struct(eps, eps, 0.0, 1, decay=False)
    eps_out = torch.empty(E, device="cuda")
    a = ops.epsilon_greedy(q, sched, seed=seed, offset=offset, dev_counter=ctr, epsilon_out=eps_out)
    want = P.epsilon_greedy(q.cpu().numpy(), np.float32(eps), seed, offset + 3)
    np.testing.assert_array_equal(a.cpu().numpy(), want)
    assert (eps_out.cpu().numpy() == np.float32(eps)).all()
    np.testing.assert_array_equal(ops.epsilon_greedy(q, sched, mode=True).cpu().numpy(), P.epsilon_greedy(q.cpu().numpy(), eps, 0, 0, mode=True))
    if eps == 0.0:  # never explores: always a maximal index
        qn = q.cpu().numpy()
        assert (qn[np.arange(E), a.cpu().numpy()] == qn.max(1)).all()


@pytest.mark.parametrize("decay,ts", [(True, 7.5), (True, 0.0), (True, -2.0), (False, 10.0)])
def test_device_epsilon_equals_the_fp32_schedule(decay, ts):
    q = torch.zeros(4, 3, device="cuda")
    spu = 6
    sched = ops.epsilon_schedule_struct(1.0, 0.05, ts, spu, decay=decay)
    for count in [0, 5, 6, 11, 12, 30, 42, 47, 48, 60, 1000]:
        c = torch.tensor([count], dtype=torch.int32, device="cuda")
        eo, uo = torch.empty(4, device="cuda"), torch.empty(4, dtype=torch.int32, device="cuda")
        ops.epsilon_greedy(q, sched, count=c, epsilon_out=eo, update_no_out=uo)
        assert int(uo[0]) == count // spu
        assert eo[0].item() == P.epsilon_at(1.0, 0.05, ts, decay, count // spu).item(), (count, eo[0].item())


@pytest.mark.parametrize("lam", [0.0, 0.95, 1.0])
@pytest.mark.parametrize("T", [1, 8, 128])
@pytest.mark.parametrize("E", [37, 256])
def test_q_lambda_both_faces(lam, T, E):
    rng = np.random.default_rng(T * 1000 + E)
    A = 6
    q = rng.normal(size=(T, E, A)).astype(np.float32)
    r = rng.normal(size=(T, E)).astype(np.float32)
    done = rng.random((T, E)) < 0.1
    trunc = (rng.random((T, E)) < 0.05) & ~done
    gamma = 0.99
    want = P.batch_q_lambda(r, gamma * (1.0 - (done | trunc)), q, lam)
    t = lambda x: torch.tensor(x, device="cuda")
    got = ops.q_lambda(t(q), t(r), t(done.astype(np.uint8)), t(trunc.astype(np.uint8)), gamma, lam)
    np.testing.assert_allclose(f64(got), want, rtol=1e-5, atol=1e-5)
    disc = (np.float32(gamma) * (1.0 - (done | trunc))).astype(np.float32)
    got2 = ops.lambda_returns(t(r), t(disc), t(q), lam)
    np.testing.assert_allclose(f64(got2), want, rtol=1e-5, atol=1e-5)
    # the generic face with A = 1 is batch_lambda_returns itself, batch-major through multistep
    from stoix_b200.utils.multistep import batch_lambda_returns, batch_q_lambda

    v = q.max(-1)
    np.testing.assert_allclose(f64(batch_lambda_returns(t(r.T.copy()), t(disc.T.copy()), t(v.T.copy()), lam)).T,
                               P.batch_lambda_returns(r, disc, v, lam), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(f64(batch_q_lambda(t(r), t(disc), t(q), lam, time_major=True)), want, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("delta", [0.0, 0.75])
def test_q_loss_grads(delta):
    rng = np.random.default_rng(7)
    B, mb, A = 4000, 1500, 7
    action = rng.integers(0, A, size=B).astype(np.int32)
    targets = rng.normal(size=B).astype(np.float32) * 2
    idx = rng.permutation(B)[:mb].astype(np.int32)
    q = rng.normal(size=(mb, A)).astype(np.float32)
    q[0, action[idx[0]]] = targets[idx[0]]                              # td = 0
    if delta > 0:  # |td| = delta exactly (representable)
        targets[idx[1]] = np.float32(1.0)
        q[1, action[idx[1]]] = np.float32(1.0 - delta)
        targets[idx[2]] = np.float32(-1.0)
        q[2, action[idx[2]]] = np.float32(-1.0 + delta)
    t = lambda x: torch.tensor(x, device="cuda")
    dq, metrics = torch.full((mb, A), 9.0, device="cuda"), torch.zeros(2, device="cuda")
    ops.q_loss_grads(t(q), t(idx), t(action), t(targets), delta, dq, metrics, weight=0.5)
    loss, want = P.q_loss_and_dq(q.astype(np.float64), action[idx], targets[idx].astype(np.float64), delta)
    np.testing.assert_allclose(f64(dq), want, rtol=1e-6, atol=1e-12)
    assert f64(dq)[0].max() == 0 and f64(dq)[0].min() == 0
    if delta > 0:  # at the tie both branches give -td times the fp32 reciprocal of mb
        inv_m = np.float32(1.0) / np.float32(mb)
        assert dq[1, action[idx[1]]].item() == -np.float32(delta) * inv_m and dq[2, action[idx[2]]].item() == np.float32(delta) * inv_m
    np.testing.assert_allclose(metrics[0].item(), 0.5 * loss, rtol=1e-6)
    assert metrics[1].item() == 0.0
    with pytest.raises(ops.StxError, match="contiguous"):   # the kernels index rows densely: strided views are refused
        ops.q_loss_grads(t(q).t().contiguous().t(), t(idx), t(action), t(targets), delta, dq, metrics)
    dq2, m2 = torch.zeros_like(dq), torch.zeros(2, device="cuda")
    ops.q_loss_grads(t(q), t(idx), t(action), t(targets), delta, dq2, m2, weight=0.5)
    assert torch.equal(dq, dq2) and torch.equal(metrics, m2)


@pytest.mark.parametrize("clip,decay", [(1e30, False), (0.5, False), (0.5, True)])
def test_clip_radam_steps_against_fp64(clip, decay):
    rng = np.random.default_rng(11)
    segs = [(0, 1001, 3e-3, clip), (1004, 517, 1e-3, clip * 2)]
    n = 1524
    dev = torch.device("cuda")
    spu, num_updates = 4, 12
    plan = ops.AdamPlan(segs, dev, b1=0.9, b2=0.999, eps=1e-8, decay=decay, steps_per_update=spu, num_updates=num_updates, rule="radam")
    p = torch.tensor(rng.normal(size=n).astype(np.float32), device=dev)
    mu, nu = torch.zeros_like(p), torch.zeros_like(p)
    pad0 = f64(p)[1001:1004].copy()
    b1, b2, eps = (float(np.float32(x)) for x in (0.9, 0.999, 1e-8))
    for step in range(45):
        g = torch.tensor((rng.normal(size=n) * 0.1).astype(np.float32), device=dev)
        p0, mu0, nu0, cnt = f64(p), f64(mu), f64(nu), plan.counts.cpu().numpy().copy()
        ops.clip_adam_step(plan, p, g, mu, nu)
        for s, (off, c, lr0, mg) in enumerate(segs):
            sl = slice(off, off + c)
            st = P.RadamState(mu0[sl].copy(), nu0[sl].copy(), int(cnt[2 * s]))
            lr = lr0 * (1.0 - (int(cnt[2 * s + 1]) // spu) / num_updates) if decay else lr0
            want = P.clip_radam_step(p0[sl], f64(g)[sl], st, lr, mg, b1, b2, eps)
            np.testing.assert_allclose(f64(p)[sl], want, rtol=2e-6, atol=lr0 * 2e-5, err_msg=f"step {step} segment {s}")
            np.testing.assert_allclose(f64(mu)[sl], st.mu, rtol=1e-5, atol=1e-9)
            np.testing.assert_allclose(f64(nu)[sl], st.nu, rtol=1e-5, atol=1e-12)
        assert int(plan.counts[0]) == step + 1
    assert (f64(p)[1001:1004] == pad0).all()   # the floats between the segments are untouched


def _learner(env_name, E, T, nmb, epochs, ln, extra=()):
    from stoix_b200 import random as srandom
    from stoix_b200.config import compose
    from stoix_b200.systems.q_learning import ff_pqn
    from stoix_b200.utils import make_env
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    ov = [f"env={env_name}", f"arch.total_num_envs={E}", f"system.rollout_length={T}", f"system.num_minibatches={nmb}",
          f"system.epochs={epochs}", f"arch.total_timesteps={E * T * 40}", "arch.num_evaluation=1", "logger.use_console=False",
          f"network.actor_network.pre_torso.use_layer_norm={ln}"] + list(extra)
    cfg = compose("default_ff_pqn", ov, config_dir="default/anakin")
    cfg.num_devices, cfg.rank = 1, 0
    cfg = check_total_timesteps(cfg, quiet=True)
    env, eval_env = make_env.make(cfg)
    keys = srandom.split(srandom.PRNGKey(3), 2)
    learn, eval_net, state = ff_pqn.learner_setup(env, (keys[0], keys[1]), cfg)
    return cfg, learn, eval_net, state, eval_env


@pytest.mark.parametrize("ln", [False, True])
@pytest.mark.parametrize("huber", [0.0, 1.0])
def test_three_updates_eager_and_graph_match_the_oracle(ln, huber):
    E, T, nmb, epochs = 64, 4, 4, 2
    extra = ["env.kwargs.obs_dim=8", "env.kwargs.num_actions=4", "network.actor_network.pre_torso.layer_sizes=[32,32]",
             f"system.huber_loss_parameter={huber}", "system.decay_learning_rates=True", "system.q_lr=1e-2"]
    cfg, learn, _, state, _ = _learner("synthetic/box", E, T, nmb, epochs, ln, extra)
    cfg.arch.num_updates_per_eval = 1
    spec = state.params.spec
    sizes = list(spec.sizes)
    h = P.PqnHyper(epochs, nmb, float(cfg.system.gamma), float(cfg.system.q_lambda), huber, float(cfg.system.q_lr),
                   float(cfg.system.max_grad_norm), num_updates=int(cfg.arch.num_updates), decay=True)
    params = O.MLPParams.from_flat(f64(state.params.flat), sizes, "silu", ln)
    st = P.RadamState(np.zeros(spec.param_count), np.zeros(spec.param_count))
    eps_sched = lambda k: P.epsilon_at(1.0, float(cfg.system.training_epsilon), float(cfg.arch.num_updates) * 0.5, True, k)
    for k in range(3):
        pre = O.MLPParams.from_flat(f64(state.params.flat), sizes, "silu", ln)   # the rollout's parameters (updated in place by learn)
        out = learn(state)
        torch.cuda.synchronize()
        sh = learn.built["shards"][0]
        assert (learn.built["graph"] is not None) == (k >= 1)
        obs, nxt = f64(sh.obs[:T]), f64(sh.next_obs)
        # every step drew from Q(obs[t]) of the rollout's parameters with the shard's seed, call t + (updates so far) * T
        q_roll, _ = O.mlp_forward(pre, obs.reshape(T * E, -1))
        np.testing.assert_allclose(f64(sh.q[:T]).reshape(T * E, -1), q_roll, rtol=1e-5, atol=1e-5)
        for t in range(T):
            want = P.epsilon_greedy(sh.q[t].cpu().numpy(), eps_sched(k), int(state.key[0]), t + k * T)
            np.testing.assert_array_equal(sh.action[t].cpu().numpy(), want, err_msg=f"update {k} step {t}")
        tg = P.targets_literal(params, obs, nxt, f64(sh.reward), sh.done.cpu().numpy(), sh.truncated.cpu().numpy(), h.gamma, h.q_lambda)
        np.testing.assert_allclose(f64(sh.targets), tg, rtol=1e-4, atol=1e-5)
        params = P.pqn_update(params, st, obs, sh.action.cpu().numpy(), tg, [p.cpu().numpy() for p in sh.perms], h, sizes)
        np.testing.assert_allclose(f64(out.learner_state.params.flat), params.flat(), rtol=1e-4, atol=2e-6, err_msg=f"update {k}")
        state = out.learner_state
        assert (f64(sh.epsilon) == eps_sched(k)).all()   # the device epsilon of this update, recorded for the episode metrics
        assert (sh.update_no.cpu().numpy() == k).all()
    assert out.train_metrics["q_loss"].shape == (1, epochs, nmb)
    assert set(out.episode_metrics) >= {"epsilon", "update_no", "episode_return"}


@pytest.mark.parametrize("ln", [False, True])
@pytest.mark.parametrize("huber", [0.0, 0.5])
def test_minibatch_grads_teacher_forced(ln, huber):
    """ff_pqn.minibatch_grads, the learner's gradient of one minibatch, on given data: two shards (weight 1/2 each, the first
    overwrites a dirty arena) against the fp64 oracle's mean of mlp_backward(q_loss_and_dq), 1e-5 norm-wise; bit-identical on repeat."""
    from stoix_b200.systems.q_learning import ff_pqn

    rng = np.random.default_rng(5)
    D, A, B, mb = 12, 6, 2048, 384
    spec = ops.MlpSpec((D, 64, 64, A), activation="silu", use_layer_norm=ln)
    sizes = list(spec.sizes)
    flat = (rng.normal(size=spec.param_count) * 0.2).astype(np.float32)
    net = O.MLPParams.from_flat(flat.astype(np.float64), sizes, "silu", ln)
    if ln:  # LayerNorm scales near 1
        for i in range(len(sizes) - 2):
            net.b[i] = net.b[i] + 1.0
        flat = net.flat().astype(np.float32)
        net = O.MLPParams.from_flat(flat.astype(np.float64), sizes, "silu", ln)
    t = lambda x, dt=None: torch.tensor(x, device="cuda", dtype=dt)
    shards, want, loss = [], np.zeros(spec.param_count), 0.0
    for u in range(2):
        obs = rng.normal(size=(B, D)).astype(np.float32)
        action = rng.integers(0, A, size=B).astype(np.int32)
        targets = (rng.normal(size=B) * 3).astype(np.float32)
        idx = rng.permutation(B)[:mb].astype(np.int32)
        shards.append((t(obs), t(idx), t(action), t(targets)))
        q, acts = O.mlp_forward(net, obs[idx].astype(np.float64))
        l, dq = P.q_loss_and_dq(q, action[idx], targets[idx].astype(np.float64), huber)
        want += 0.5 * O.mlp_backward(net, acts, dq).flat()
        loss += 0.5 * l
    params = t(flat)
    ws = ops.mlp_train_workspace(spec, mb, "cuda")
    q_mb, dq_mb = torch.empty(mb, A, device="cuda"), torch.empty(mb, A, device="cuda")
    got = []
    for _ in range(2):
        grads, metric = torch.full((spec.param_count,), 7.0, device="cuda"), torch.zeros(1, device="cuda")
        ff_pqn.minibatch_grads(spec, params, shards, huber, grads, metric, ws, q_mb, dq_mb)
        got.append((grads, metric))
    torch.cuda.synchronize()
    assert torch.equal(got[0][0], got[1][0]) and torch.equal(got[0][1], got[1][1])
    g = f64(got[0][0])
    assert np.linalg.norm(g - want) <= 1e-5 * np.linalg.norm(want), np.linalg.norm(g - want) / np.linalg.norm(want)
    np.testing.assert_allclose(got[0][1].item(), loss, rtol=1e-5)
    # a gradient off by a constant factor (a lost 1/mb or 1/U) is far outside the bound
    assert np.linalg.norm(2 * g - want) > 0.5 * np.linalg.norm(want)


def test_graph_replays_draw_fresh_actions_and_shuffles_and_shards_differ():
    E, T = 64, 4
    cfg, learn, _, state, _ = _learner("synthetic/box", E, T, 4, 2, True, ["env.kwargs.obs_dim=8", "arch.update_batch_size=2",
                                                                           "network.actor_network.pre_torso.layer_sizes=[32,32]"])
    cfg.arch.num_updates_per_eval = 1
    seen = []
    for _ in range(3):
        state = learn(state).learner_state
        torch.cuda.synchronize()
        shards = learn.built["shards"]
        seen.append((shards[0].action.clone(), shards[0].perms.clone()))
        assert not torch.equal(shards[0].perms, shards[1].perms) and not torch.equal(shards[0].obs, shards[1].obs)
    assert not torch.equal(seen[1][0], seen[2][0]) and not torch.equal(seen[1][1], seen[2][1])


def test_bf16_is_refused():
    with pytest.raises(ValueError, match="bf16"):
        _learner("synthetic/box", 64, 4, 4, 2, False, ["arch.precision=bf16"])


def test_cartpole_learns():
    """PQN with LayerNorm on CartPole, 48 updates of the 1e6-step schedule (1024 envs, T = 8, 4 x 16), evaluated greedily every 8
    updates.  A uniform policy returns about 22.  Greedy PQN returns swing widely between evaluations (500 at one, 150 at the next),
    so the test reads the best evaluation and the training episodes of the last 8 updates.  Measured on an H100 80GB HBM3 with this
    seed: evaluations 193, 151, 236, 500, 307, 345; training return 127.6.  Bars: 250 and 80."""
    from stoix_b200 import random as srandom
    from stoix_b200.evaluator import get_distribution_act_fn, get_ff_evaluator_fn

    cfg, learn, eval_net, state, eval_env = _learner("gymnax/cartpole", 1024, 8, 16, 4, True, ["arch.total_timesteps=1e6"])
    cfg.arch.num_updates_per_eval = 8
    evaluator = get_ff_evaluator_fn(eval_env, get_distribution_act_fn(cfg, eval_net.apply), cfg)
    evals = []
    for k in range(6):
        out = learn(state)
        state = out.learner_state
        evals.append(float(evaluator(state.params, srandom.PRNGKey(k))["episode_return"].mean()))
    em = out.episode_metrics
    train_return = float(em["episode_return"][em["is_terminal_step"]].mean())
    print(f"[pqn cartpole] greedy evaluations {[round(r, 1) for r in evals]}, training return {train_return:.1f}")
    assert max(evals) > 250.0 and train_return > 80.0


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
from tests import pqn_oracle as P
from stoix_b200 import random as srandom
from stoix_b200.config import compose
from stoix_b200.systems.q_learning import ff_pqn
from stoix_b200.utils import make_env
from stoix_b200.utils.total_timestep_checker import check_total_timesteps
E, T, nmb, epochs, n_upd = 64, 4, 4, 2, 3
cfg = compose("default_ff_pqn", ["env=synthetic/box", f"arch.total_num_envs={E * world}", f"system.rollout_length={T}",
                                 f"system.num_minibatches={nmb}", f"system.epochs={epochs}", f"arch.total_timesteps={E * world * T * n_upd}",
                                 "arch.num_evaluation=1", "logger.use_console=False", "env.kwargs.obs_dim=8", "env.kwargs.num_actions=4",
                                 "network.actor_network.pre_torso.layer_sizes=[32,32]", "network.actor_network.pre_torso.use_layer_norm=True",
                                 "system.q_lr=1e-2"], config_dir="default/anakin")
cfg.num_devices, cfg.rank = world, rank
cfg = check_total_timesteps(cfg, quiet=True)
assert cfg.arch.num_envs == E and cfg.arch.num_updates == n_upd
env, _ = make_env.make(cfg)
keys = srandom.split(srandom.PRNGKey(cfg.arch.seed), 2)
learn, _, state = ff_pqn.learner_setup(env, (keys[0], keys[1]), cfg)
cfg.arch.num_updates_per_eval = 1
f64 = lambda t: t.detach().double().cpu().numpy()
sizes = list(state.params.spec.sizes)
h = P.PqnHyper(epochs, nmb, float(cfg.system.gamma), float(cfg.system.q_lambda), 0.0, float(cfg.system.q_lr), float(cfg.system.max_grad_norm),
               num_updates=n_upd)

def grad_sync(g):   # pmean over "device": SUM over the ranks, then 1/world
    t = torch.from_numpy(np.ascontiguousarray(g, np.float64))
    dist.all_reduce(t, op=dist.ReduceOp.SUM, group=cpu_group)
    return t.numpy() / world

ok, why, worst = True, "", 0.0
for upd in range(n_upd):   # eager, graph capture, graph replay
    params = O.MLPParams.from_flat(f64(state.params.flat), sizes, "silu", True)   # every update checked on its own
    st = P.RadamState(f64(state.opt_states.mu)[: params.flat().size], f64(state.opt_states.nu)[: params.flat().size], upd * epochs * nmb)
    out = learn(state); state = out.learner_state
    torch.cuda.synchronize()
    sh = learn.built["shards"][0]
    obs = f64(sh.obs[:T])
    tg = P.targets_literal(params, obs, f64(sh.next_obs), f64(sh.reward), sh.done.cpu().numpy(), sh.truncated.cpu().numpy(), h.gamma, h.q_lambda)
    want = P.pqn_update(params, st, obs, sh.action.cpu().numpy(), tg, [p.cpu().numpy() for p in sh.perms], h, sizes, grad_sync=grad_sync).flat()
    err = float(np.abs(f64(state.params.flat)[: want.size] - want).max() / max(np.abs(want).max(), 1e-30))
    worst = max(worst, err)
    if not np.allclose(f64(state.params.flat)[: want.size], want, rtol=1e-4, atol=2e-6):
        ok, why = False, f"update {upd}: max relative parameter error {err:.3e}"
arena = state.params.arena
gathered = [torch.empty_like(arena) for _ in range(world)]
dist.all_gather(gathered, arena)
obs_sum = learn.built["shards"][0].obs[:T].sum()
sums = [torch.empty_like(obs_sum) for _ in range(world)]
dist.all_gather(sums, obs_sum)
loss = out.train_metrics["q_loss"].reshape(-1)
losses = [torch.empty_like(loss) for _ in range(world)]
dist.all_gather(losses, loss)
flags = torch.tensor([1.0 if ok else 0.0], device="cuda")
dist.all_reduce(flags, op=dist.ReduceOp.MIN)
if rank == 0:
    print(json.dumps({"oracle_ok_all_ranks": bool(flags.item() == 1.0), "why": why, "worst": worst,
                      "params_identical_across_ranks": all(torch.equal(gathered[0], g) for g in gathered),
                      "metrics_identical_across_ranks": all(torch.equal(losses[0], l) for l in losses),
                      "shards_differ": len({float(s) for s in sums}) == world, "counts": state.params.arena_counts.cpu().tolist()}))
dist.barrier(); torch.cuda.synchronize(); sys.stdout.flush(); os._exit(0)  # NCCL teardown can hang at exit here
'''


def test_two_rank_update_matches_oracle(tmp_path):
    """Two torchrun ranks, three whole updates (eager, capture, replay) with the NCCL all-reduce inside the captured step: each rank
    replays its own trajectory through the oracle with the gradient exchange as a gloo all-reduce (SUM, then 1/world), parameters
    rtol 1e-4 atol 2e-6 per update; replicas and the averaged q_loss metrics bit-identical across the ranks."""
    import json
    import os
    import subprocess
    import sys

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (NCCL refuses two ranks on one device)")
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29517", str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=240, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    res = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    print(res)
    assert res["oracle_ok_all_ranks"], res
    assert res["params_identical_across_ranks"] and res["metrics_identical_across_ranks"] and res["shards_differ"], res
    assert res["counts"] == [3 * 2 * 4] * 2, res
