"""The Anakin experiment driver (stoix_b200/systems/anakin.py) on the CPU: run_experiment with a fake learner, evaluators, logger and
checkpointer, get_final_step_metrics, and the shard / rank seed formulas."""
from types import SimpleNamespace

import pytest
import torch

from stoix_b200 import random as srandom
from stoix_b200.systems import anakin
from stoix_b200.utils.logger import LogEvent


class _Clock:
    """time.time() that advances by one second per call: every learn() and evaluation takes exactly 1 s."""

    def __init__(self):
        self.now = 0.0

    def time(self):
        self.now += 1.0
        return self.now


class _Logger:
    def __init__(self, config):
        self.events = []

    def log_config(self, config):
        pass

    def log(self, metrics, t, t_eval, event):
        self.events.append((event, t, t_eval, dict(metrics)))

    def stop(self):
        pass


class _Checkpointer:
    saved = []

    def __init__(self, **kwargs):
        pass

    def save(self, timestep, unreplicated_learner_state, episode_return):
        _Checkpointer.saved.append((timestep, unreplicated_learner_state.params.actor_params, episode_return))


def _state(i, running_statistics=None):
    """Learner state after i learn() calls: its policy tree is flat = [i, i]; `online` is a second tree, flat = [10 i, 10 i]."""
    tree = lambda v: SimpleNamespace(flat=torch.full((2,), float(v)), spec=f"spec{i}", flat_bf16=None)
    st = SimpleNamespace(params=SimpleNamespace(actor_params=tree(i), online=tree(10 * i)))
    if running_statistics is not None:
        st.running_statistics = running_statistics
    return st


def _run(monkeypatch, config_name, overrides, returns, finished, policy=None, running_statistics=None):
    """Run anakin.run_experiment with fakes.  Evaluation i returns episode_return = returns[i]; learn() call i reports a finished
    episode iff finished[i].  Returns (result, record) where record holds what the fakes saw."""
    from stoix_b200.config import compose

    logger = {}
    rec = {"learn": 0, "eval": [], "abs": [], "setup_config": None}
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(anakin, "time", _Clock())
    monkeypatch.setattr(anakin.environments, "make", lambda config: ("env", "eval_env"))
    monkeypatch.setattr(anakin, "StoixLogger", lambda config: logger.setdefault("it", _Logger(config)))
    monkeypatch.setattr(anakin, "Checkpointer", _Checkpointer)
    _Checkpointer.saved = []

    def learn(state):
        i = rec["learn"]
        rec["learn"] += 1
        term = torch.zeros(1, 1, 2, 3, dtype=torch.bool)
        term[0, 0, 1, 2] = finished[i]
        em = {"episode_return": torch.full((1, 1, 2, 3), 7.0 + i), "episode_length": torch.ones(1, 1, 2, 3, dtype=torch.int32),
              "is_terminal_step": term}
        return SimpleNamespace(learner_state=_state(i + 1, running_statistics), episode_metrics=em, train_metrics={"loss": torch.ones(2)})

    def setup(env, keys, config):
        assert env == "env"
        rec["setup_config"], rec["keys"] = config, keys
        return learn, "network", _state(0, running_statistics)

    def make_evaluators(eval_env, key_e, network, config):
        assert (eval_env, network) == ("eval_env", "network")

        def evaluator(params, key, **kw):
            rec["eval"].append((params, kw))
            r = returns[len(rec["eval"]) - 1]
            return {"episode_return": torch.tensor([r, r]), "episode_length": torch.tensor([3, 4])}

        def absolute(params, key, **kw):
            rec["abs"].append((params, kw))
            return {"episode_return": torch.tensor([-1.0, -3.0]), "episode_length": torch.tensor([5, 5])}

        return evaluator, absolute

    base = ["env=synthetic/box", "arch.total_num_envs=8", "system.rollout_length=4", "system.epochs=3", f"arch.num_evaluation={len(returns)}",
            f"arch.total_timesteps={8 * 4 * 2 * len(returns)}", "arch.absolute_metric=True", "logger.checkpointing.save_model=True"]
    kw = {} if policy is None else {"policy": policy}
    result = anakin.run_experiment(compose(config_name, base + overrides, config_dir="default/anakin"), setup, net_keys=2,
                                   make_evaluators=make_evaluators, best_tree=lambda net, tree, flat: ("best", tree.spec, flat.clone()), **kw)
    rec["events"] = logger["it"].events
    return result, rec


@pytest.mark.parametrize("config_name,extra,opt_steps", [("default_ff_ppo", ["system.num_minibatches=2"], 3 * 2),
                                                         ("default_ff_dqn", [], 3)])
def test_run_experiment_loop(monkeypatch, config_name, extra, opt_steps):
    returns, finished = [1.0, 3.0, 3.0, 2.0], [True, False, True, True]
    result, rec = _run(monkeypatch, config_name, extra, returns, finished)
    config = rec["setup_config"]
    assert (config.system.get("num_minibatches", None) is None) == (config_name == "default_ff_dqn")
    n = len(returns)
    assert rec["learn"] == n
    key, key_e, *net = srandom.split(srandom.PRNGKey(config.arch.seed), 4)
    assert rec["keys"] == (key, *net)
    upe = int(config.arch.num_updates_per_eval)
    steps_per_rollout = upe * int(config.system.rollout_length) * int(config.arch.update_batch_size) * int(config.arch.num_envs)
    by_event = lambda ev: [e for e in rec["events"] if e[0] == ev]
    assert [e[1] for e in by_event(LogEvent.MISC)] == [steps_per_rollout * (i + 1) for i in range(n)]
    assert [e[3]["timestep"] for e in by_event(LogEvent.MISC)] == [steps_per_rollout * (i + 1) for i in range(n)]
    act = by_event(LogEvent.ACT)
    assert [e[2] for e in act] == [i for i in range(n) if finished[i]]
    for e in act:
        assert e[3]["episode_return"].tolist() == [7.0 + e[2]]
        assert float(e[3]["steps_per_second"]) == steps_per_rollout
    train = by_event(LogEvent.TRAIN)
    assert len(train) == n and all(float(e[3]["steps_per_second"]) == upe * opt_steps for e in train)
    assert [e[3]["episode_return"].tolist() for e in by_event(LogEvent.EVAL)] == [[r, r] for r in returns]
    # evaluation i sees the parameters after learn() call i
    assert [p.flat[0].item() for p, _ in rec["eval"]] == [1.0, 2.0, 3.0, 4.0]
    # best parameters: the last evaluation with the highest return (ties go to the later one); the absolute evaluator gets its tree,
    # built on the final state's layout
    (tag, spec, flat), kw = rec["abs"][0]
    assert (tag, spec, flat.tolist()) == ("best", f"spec{n}", [3.0, 3.0])
    assert [e[1] for e in by_event(LogEvent.ABSOLUTE)] == [steps_per_rollout * n]
    assert [c[0] for c in _Checkpointer.saved] == [steps_per_rollout * (i + 1) for i in range(n)]
    assert [c[1].flat[0].item() for c in _Checkpointer.saved] == [1.0, 2.0, 3.0, 4.0]
    assert [c[2] for c in _Checkpointer.saved] == returns
    assert result == -2.0   # mean eval_metric of the last evaluation, the absolute one


def test_run_experiment_without_absolute_metric_returns_the_last_evaluation(monkeypatch):
    result, rec = _run(monkeypatch, "default_ff_ppo", ["arch.absolute_metric=False"], [1.0, 5.0], [True, True])
    assert rec["abs"] == [] and result == 5.0


def test_policy_is_what_is_evaluated_tracked_and_checkpointed(monkeypatch):
    _, rec = _run(monkeypatch, "default_ff_dqn", [], [2.0, 1.0], [True, True], policy=lambda s: s.params.online)
    assert [p.flat[0].item() for p, _ in rec["eval"]] == [10.0, 20.0]
    assert [c[1].flat[0].item() for c in _Checkpointer.saved] == [10.0, 20.0]
    assert rec["abs"][0][0][2].tolist() == [10.0, 10.0]


@pytest.mark.parametrize("with_stats", [False, True])
def test_running_statistics_reach_the_evaluators_only_when_present(monkeypatch, with_stats):
    rs = object() if with_stats else None
    _, rec = _run(monkeypatch, "default_ff_ppo", [], [1.0, 2.0], [True, True], running_statistics=rs)
    want = {"running_statistics": rs} if with_stats else {}
    assert all(kw == want for _, kw in rec["eval"] + rec["abs"])
    assert all(kw.get("running_statistics") is rs for _, kw in rec["eval"] + rec["abs"])


def test_get_final_step_metrics():
    term = torch.tensor([[False, True], [False, True]])
    metrics = {"episode_return": torch.tensor([[1.0, 2.0], [3.0, 4.0]]), "episode_length": torch.tensor([[5, 6], [7, 8]]), "is_terminal_step": term}
    out, has = anakin.get_final_step_metrics(metrics)
    assert has and set(out) == {"episode_return", "episode_length"}
    assert out["episode_return"].tolist() == [2.0, 4.0] and out["episode_length"].tolist() == [6, 8]
    out, has = anakin.get_final_step_metrics({**metrics, "is_terminal_step": torch.zeros_like(term)})
    assert not has and out["episode_return"].numel() == 0


class _Env:
    def __init__(self):
        self.seed, self.resets = None, []

    def reset(self, keys):
        self.resets.append((self.seed, keys))
        return f"state{len(self.resets)}", f"ts{len(self.resets)}"


@pytest.mark.parametrize("rank", [0, 3])
def test_reset_shards_seeds_each_rank_and_shard(rank):
    from stoix_b200.config import compose

    config = compose("default_ff_ppo", ["arch.update_batch_size=3", "arch.seed=5"], config_dir="default/anakin")
    config.arch.num_envs = 4
    shard_keys = srandom.split(123, 4)
    env = _Env()
    states, timesteps = anakin.reset_shards(env, shard_keys, config, rank)
    assert states == ["state1", "state2", "state3"] and timesteps == ["ts1", "ts2", "ts3"]
    assert env.resets == [((5 + 7919 * rank + 15485863 * u) & ((1 << 63) - 1), srandom.split(shard_keys[u], 4)) for u in range(3)]
    assert rank != 3 or env.resets[2][0] == 5 + 23757 + 30971726


@pytest.mark.parametrize("n,world_size", [(2, 1), (2, 4), (3, 2)])
def test_rank_seeds_split_per_rank_and_mask_62_bits(n, world_size):
    key = srandom.PRNGKey(9)
    step_key = srandom.split(key, n * world_size)
    for rank in range(world_size):
        seeds = anakin.rank_seeds(key, n, rank, world_size)
        assert seeds == tuple(step_key[n * rank + i] & ((1 << 62) - 1) for i in range(n))
        assert all(0 <= s < (1 << 62) for s in seeds)
    assert len({s for r in range(world_size) for s in anakin.rank_seeds(key, n, r, world_size)}) == n * world_size


def _compose(name, overrides=()):
    from stoix_b200.config import compose

    return compose(name, list(overrides), config_dir="default/anakin")


def test_learn_builds_once_seeds_the_carry_and_collects_every_update():
    from stoix_b200.envs.base import TimeStep

    T, E, D, U, n_upd = 3, 2, 4, 2, 3
    config = _compose("default_ff_pqn", ["arch.cuda_graph=False"])
    config.arch.num_updates_per_eval = n_upd
    built, rec = {}, {"builds": 0, "calls": 0, "first_rows": {}}

    def build(state):
        rec["builds"] += 1
        shards = [anakin.Trajectory(T, E, D, "cpu") for _ in range(U)]
        for sh in shards:
            sh.epsilon = torch.zeros(T, E)
        built.update(shards=shards, metrics=torch.zeros(2, 5), graph=None, eager_done=False)

    def step(state):
        k = rec["calls"]
        rec["calls"] += 1
        for u, sh in enumerate(built["shards"]):
            sh.carry_in()
            if k == 0:
                rec["first_rows"][u] = sh.obs[0].clone()
            v = 100 * k + 10 * u
            sh.obs[1:].fill_(v)
            sh.episode_return.fill_(v + 1)
            sh.episode_length.fill_(v + 2)
            sh.is_terminal_step.fill_((k + u) % 2)
            sh.epsilon.fill_(v + 3)
        built["metrics"].fill_(k)

    state = SimpleNamespace(timestep=[TimeStep(None, None, None, torch.full((E, D), -1.0 - u), {}) for u in range(U)])
    timestep, ep, train = anakin.learn(built, build, step, state, config, extra_fields=("epsilon",))
    assert rec["builds"] == 1 and built["eager_done"] and built["graph"] is None
    # the carry row T starts from the learner state's observation and is the first row of the first rollout
    assert all(torch.equal(rec["first_rows"][u], torch.full((E, D), -1.0 - u)) for u in range(U))
    assert set(ep) == {"episode_return", "episode_length", "is_terminal_step", "epsilon"}
    assert {k: (tuple(v.shape), v.dtype) for k, v in ep.items()} == {
        "episode_return": ((n_upd, U, T, E), torch.float32), "episode_length": ((n_upd, U, T, E), torch.int32),
        "is_terminal_step": ((n_upd, U, T, E), torch.bool), "epsilon": ((n_upd, U, T, E), torch.float32)}
    for k in range(n_upd):
        for u in range(U):
            v = 100 * k + 10 * u
            assert (ep["episode_return"][k, u] == v + 1).all() and (ep["episode_length"][k, u] == v + 2).all()
            assert (ep["is_terminal_step"][k, u] == bool((k + u) % 2)).all() and (ep["epsilon"][k, u] == v + 3).all()
    assert train.shape == (n_upd, 2, 5) and [float(train[k].unique()) for k in range(n_upd)] == [0.0, 1.0, 2.0]
    # the next learn() starts from row T of the last rollout
    for u, ts in enumerate(timestep):
        assert ts.observation.data_ptr() == built["shards"][u].obs[T].data_ptr() and (ts.observation == 100 * (n_upd - 1) + 10 * u).all()
    # a second call reuses the buffers and carries on from that row
    anakin.learn(built, build, step, SimpleNamespace(timestep=timestep), config)
    assert rec["builds"] == 1 and rec["calls"] == 2 * n_upd


@pytest.mark.parametrize("segments", [[(0, 5)], [(0, 5), (8, 7)], [(0, 5), (8, 16), (24, 1)]])
def test_arena_state_views_and_counts_layout(segments):
    from stoix_b200 import optim

    arena = torch.arange(32, dtype=torch.float32)
    tree = SimpleNamespace()
    states = optim.arena_state(tree, arena, segments)
    assert tree.arena is arena and len(states) == len(segments)
    for name in ("arena_mu", "arena_nu"):
        t = getattr(tree, name)
        assert t.shape == arena.shape and t.dtype == torch.float32 and not t.any() and t.data_ptr() != arena.data_ptr()
    counts = tree.arena_counts
    assert counts.dtype == torch.int32 and counts.tolist() == [0] * (2 * len(segments))
    for i, ((off, n), st) in enumerate(zip(segments, states)):
        # {count, schedule count} of segment i are counts[2i], counts[2i + 1]; mu / nu are views of the arenas
        assert st.count.data_ptr() == counts[2 * i:].data_ptr() and st.count.shape == (1,)
        assert st.sched_count.data_ptr() == counts[2 * i + 1:].data_ptr() and st.sched_count.shape == (1,)
        assert st.mu.data_ptr() == tree.arena_mu[off:].data_ptr() and st.mu.shape == (n,)
        assert st.nu.data_ptr() == tree.arena_nu[off:].data_ptr() and st.nu.shape == (n,)


def test_replay_buffers_split_the_totals_and_seed_each_shard():
    key = srandom.PRNGKey(11)
    config = _compose("default_ff_dqn", ["arch.update_batch_size=2", "system.total_buffer_size=1200", "system.total_batch_size=96"])
    made = anakin.replay_buffers(config, key, 1, 3, lambda size, batch, seed: (size, batch, seed))
    assert (config.system.buffer_size, config.system.batch_size) == (200, 16)
    # seed of shard u on rank r: split(key, n_devices * U)[r * U + u]
    assert made == [(200, 16, 7285328837743276888), (200, 16, 14567865290730263530)]
    assert [m[2] for m in made] == srandom.split(key, 6)[2:4]
    for bad in (["system.total_buffer_size=1201"], ["system.total_batch_size=97"]):
        with pytest.raises(AssertionError):
            anakin.replay_buffers(_compose("default_ff_dqn", bad), key, 0, 3, lambda *a: a)


class _Plan:
    def __init__(self, segments, device, **kwargs):
        self.segments, self.device, self.kwargs, self.counts = segments, device, kwargs, None


@pytest.mark.parametrize("decay", [True, False])
@pytest.mark.parametrize("system", ["ff_ppo", "rec_ppo", "ff_sac"])
def test_adam_plan_takes_decay_and_its_constants_from_the_schedule(monkeypatch, system, decay):
    """The plan arguments PPO, rec_ppo and SAC passed before: decay = system.decay_learning_rates, steps_per_update = epochs *
    num_minibatches (epochs for SAC), num_updates = arch.num_updates.  Without decay the kernel reads neither constant."""
    from stoix_b200 import ops
    from stoix_b200 import optim as optax
    from stoix_b200.utils.training import make_learning_rate

    monkeypatch.setattr(ops, "AdamPlan", _Plan)
    config = _compose(f"default_{system}", [f"system.decay_learning_rates={decay}", "system.epochs=3"])
    config.arch.num_updates = 70
    nmb = int(config.system.get("num_minibatches", 1))
    lrs = (config.system.actor_lr, config.system.q_lr, config.system.alpha_lr) if system == "ff_sac" else (config.system.actor_lr, config.system.critic_lr)
    opts = [optax.chain(optax.clip_by_global_norm(config.system.max_grad_norm),
                        optax.adam(make_learning_rate(lr, config, 3, None if system == "ff_sac" else nmb), eps=1e-5)) for lr in lrs]
    counts = torch.zeros(2 * len(opts), dtype=torch.int32)
    plan = optax.adam_plan([(8 * i, 5 + i, o) for i, o in enumerate(opts)], "cpu", counts)
    assert plan.counts is counts and plan.device == "cpu"
    assert plan.segments == [(8 * i, 5 + i, float(lr), float(config.system.max_grad_norm)) for i, lr in enumerate(lrs)]
    kw = plan.kwargs
    assert (kw["b1"], kw["b2"], kw["eps"], kw["decay"]) == (0.9, 0.999, 1e-5, decay)
    assert "rule" not in kw
    if decay:
        assert (kw["steps_per_update"], kw["num_updates"]) == (3 * nmb, 70)
    else:
        assert kw["steps_per_update"] > 0 and kw["num_updates"] > 0


def test_adam_plan_carries_the_radam_rule(monkeypatch):
    from stoix_b200 import ops
    from stoix_b200 import optim as optax

    monkeypatch.setattr(ops, "AdamPlan", _Plan)
    opt = optax.chain(optax.clip_by_global_norm(0.5), optax.radam(5e-4, eps_root=1e-9, threshold=4.0))
    plan = optax.adam_plan([(0, 10, opt)], "cpu", None)
    assert plan.segments == [(0, 10, 5e-4, 0.5)]
    assert {k: plan.kwargs[k] for k in ("rule", "eps_root", "threshold", "decay")} == {"rule": "radam", "eps_root": 1e-9, "threshold": 4.0,
                                                                                        "decay": False}
