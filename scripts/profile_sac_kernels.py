"""Driver for `ncu --set full`: ONE launch of every kernel of the ff_sac update epoch (and the Sebulba / fp32 path's GEMMs) at the
BASELINE configs[3] shapes (obs 17, act 6, batch 256 and 4096, actor MLP[256x4] silu, twin-Q MLP[256x4] LayerNorm silu, replay
ring 1e6), after a warm-up launch of each.  Summarise with scripts/ncu_summary.py.

    ncu --set full --clock-control none --nvtx --nvtx-include "measure/" -o out/sac python scripts/profile_sac_kernels.py [batch]
"""
import sys

import torch

sys.path.insert(0, ".")
from stoix_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
D, A, CAP = 17, 6, 1_000_000
g = torch.Generator(device=dev).manual_seed(0)
sa = ops.MlpSpec((D, 256, 256, 256, 256, 2 * A), activation="silu")
sq = ops.MlpSpec((D + A, 256, 256, 256, 256, 1), activation="silu", use_layer_norm=True)
pa = torch.randn(sa.param_count, device=dev, generator=g) * 0.05
pq = torch.randn(sq.param_count, device=dev, generator=g) * 0.05
pq_t = pq.clone()
ga, gq = torch.zeros_like(pa), torch.zeros_like(pq)
z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev)
ring = ops.ReplayRing(CAP, D, A, dev)
ring.obs.normal_(generator=g), ring.next_obs.normal_(generator=g), ring.action.uniform_(-1, 1, generator=g), ring.reward.normal_(generator=g)
ring.state.copy_(torch.tensor([0, CAP], device=dev))
E, T = 1024, 1
r_obs, r_nobs, r_act = torch.randn(T, E, D, device=dev, generator=g), torch.randn(T, E, D, device=dev, generator=g), z(T, E, A)
r_rew, r_done = z(T, E), z(T, E, dt=torch.uint8)
xq_old, xq_new, xq_next = z(B, D + A), z(B, D + A), z(B, D + A)
b_rew, b_done, b_idx = z(B), z(B, dt=torch.uint8), z(B, dt=torch.int32)
ws_a, ws_q = ops.mlp_train_workspace(sa, B, dev), ops.mlp_train_workspace(sq, B, dev)
head, d_head, q1, q2, dq1, dq2, d_in = z(B, 2 * A), z(B, 2 * A), z(B, 1), z(B, 1), z(B, 1), z(B, 1), z(B, D + A)
log_alpha, metrics, g_alpha = z(1), z(8), z(1)
ctr = torch.zeros(1, dtype=torch.int64, device=dev)
act_out = z(E, 2 * A)


def all_ops():
    ops.replay_add(ring, r_obs, r_act, r_rew, r_done, r_nobs)
    ops.replay_sample(ring, B, 7, xq_old, b_rew, b_done, xq_new=xq_new, xq_next=xq_next, dev_counter=ctr, idx_out=b_idx)
    ops.mlp_forward_train(sa, pa, xq_new, ws_a, out=head)                      # panel / 64x64 FWD GEMMs (silu epilogue)
    _, logp, eps = ops.tanh_normal_sample(head, -1.0, 1.0, seed=3, dev_counter=ctr, action_out=xq_new[:, D:])
    ops.mlp_forward_train(sq, pq, xq_new, ws_q, out=q1)                        # FWD GEMMs + ln_apply_kernel
    ops.sac_actor_seed(q1, q1, logp, log_alpha, dq1, dq2, metrics=metrics)
    ops.mlp_backward(sq, pq, xq_new, dq1, ws_q, net_grad=None, d_input=d_in)  # DX GEMMs + ln_backward_kernel
    ops.tanh_normal_backward(head, eps, -1.0, 1.0, log_alpha, 1.0 / B, d_in[:, D:], out=d_head)
    ops.mlp_backward(sa, pa, xq_new, d_head, ws_a, net_grad=ga)               # DW + DX GEMMs + reduce_partials
    ops.mlp_forward_train(sq, pq, xq_old, ws_q, out=q1)
    ops.sac_q_loss(q1, q1, q2, q2, logp, b_rew, b_done, log_alpha, 0.99, dq1, dq2, metrics=metrics)
    ops.mlp_backward(sq, pq, xq_old, dq1, ws_q, net_grad=gq)                  # DW (LayerNorm torso) + scale / bias reductions
    ops.sac_alpha_grad(logp, log_alpha, -6.0, True, g_alpha, metrics=metrics)
    ops.polyak_update(pq_t, pq, 0.005)
    ops.mlp_forward(sa, pa, r_obs[0], out=act_out)                             # rollout actor forward, 1024 envs (inference form)


all_ops()
torch.cuda.synchronize()
torch.cuda.nvtx.range_push("measure")
all_ops()
torch.cuda.synchronize()
torch.cuda.nvtx.range_pop()
