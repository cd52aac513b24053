"""Driver for `ncu --set full`: ONE launch of every kernel of the hot path at the benchmark shapes (BASELINE config 2:
E=4096, T=128, D=64, A=8, mb=32768), after a warm-up launch of each.  Summarise the report with
scripts/ncu_summary.py.

    ncu --set full --clock-control none --import-source on --nvtx --nvtx-include "measure/" -o out/all python scripts/profile_all.py
"""
import sys

import torch

sys.path.insert(0, ".")
from stoix_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
E, T, D, A, mb = 4096, 128, 64, 8, 32768
B = T * E
g = torch.Generator(device=dev).manual_seed(0)
sa, sc = ops.MlpSpec((D, 256, 256, A)), ops.MlpSpec((D, 256, 256, 1))
_, coff, total = ops.arena_offsets(sa, sc)
arena = torch.randn(total, device=dev, generator=g) * 0.05
shadow = ops.cast_bf16(arena)
mu, nu = torch.zeros_like(arena), torch.zeros_like(arena)
obs = torch.randn(T + 1, E, D, device=dev, generator=g).to(torch.bfloat16)
next_obs = torch.zeros(T, E, D, device=dev, dtype=torch.bfloat16)
obs32 = torch.randn(T, E, D, device=dev, generator=g)
z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev)
action, log_prob, value, boot, reward = z(T, E, dt=torch.int32), z(T, E), z(T, E), z(T, E), torch.randn(T, E, device=dev, generator=g)
done = (torch.rand(T, E, device=dev, generator=g) < 0.005).to(torch.uint8)
trunc = z(T, E, dt=torch.uint8)
ep_ret, ep_len, is_term = z(T, E), z(T, E, dt=torch.int32), z(T, E, dt=torch.uint8)
run_ret, run_len = z(E), z(E, dt=torch.int32)
adv, tgt = z(T, E), z(T, E)
logits = z(E, A)
perm = torch.zeros(B, dtype=torch.int32, device=dev)
grads, metrics = z(total), z(8)
ws = ops.ppo_workspace(sa, sc, mb, ops.STX_PREC_BF16, dev)
plan = ops.AdamPlan([(0, sa.param_count, 3e-4, 0.5), (coff, sc.param_count, 3e-4, 0.5)], dev, steps_per_update=64, num_updates=100)
ctr = torch.zeros(1, dtype=torch.int64, device=dev)
rs_mean, rs_std, rs_sv, rs_cnt = z(D), torch.ones(D, device=dev), z(D), torch.zeros(1, dtype=torch.int64, device=dev)
norm_out = torch.empty(T, E, D, device=dev, dtype=torch.bfloat16)


def all_ops():
    ops.tc_rollout_synth(sa, arena[:coff], shadow[:coff], obs, next_obs, action, log_prob, reward, done, trunc, ep_ret, ep_len, is_term,
                         run_ret, run_len, 1, 0, ctr, 0.005, 0.002, 2, 0, ctr)
    ops.mlp_forward(sc, arena[coff:], obs[:T].view(B, D), precision=ops.STX_PREC_BF16, params_bf16=shadow[coff:], out=value.view(B, 1))
    ops.mlp_forward(sa, arena[:coff], obs[0], precision=ops.STX_PREC_BF16, params_bf16=shadow[:coff], out=logits)
    ops.categorical(logits, None, 3, 0, out=(action[0], log_prob[0]))
    ops.synth_env_step(E, D, 5, 0, 0.005, 0.002, action[0], obs[1], next_obs[0], reward[0], done[0], trunc[0], run_ret, run_len, ep_ret[0],
                       ep_len[0], is_term[0])
    _, _, stats = ops.gae_ppo(reward, value, boot, done, trunc, 0.99, 0.95, 1.0, 1, out=(adv, tgt))
    ops.make_permutation(B, 7, 0, out=perm)
    batch = ops.PpoBatch(obs[:T].view(B, D), action.view(B), log_prob.view(B), value.view(B), adv.view(B), tgt.view(B), stats, perm)
    ops.ppo_minibatch_grads(sa, sc, arena, batch, 0, mb, 0.2, 0.01, 0.5, True, grads, metrics, ws, ops.STX_PREC_BF16, 1.0, shadow, overwrite=True,
                            adam_scratch=plan.scratch)
    ops.clip_adam_step(plan, arena, grads, mu, nu, params_bf16=shadow, prenorm=True)
    ops.clip_adam_step(plan, arena, grads, mu, nu, params_bf16=shadow, prenorm=False)
    sums = ops.running_stats_accumulate(obs32.view(-1, D), rs_mean)
    ops.running_stats_finalize(sums, rs_cnt, rs_mean, rs_sv, rs_std, 5e-4, 5e4)
    ops.obs_normalize(obs32, rs_mean, rs_std, out=norm_out)
    ops.cast_bf16(arena, out=shadow)


all_ops()
torch.cuda.synchronize()
torch.cuda.nvtx.range_push("measure")
all_ops()
torch.cuda.synchronize()
torch.cuda.nvtx.range_pop()
