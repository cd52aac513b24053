"""Drop-in for the hot functions of stoix/utils/loss.py (forward values).

The training step does not call these (the fused K3 kernel evaluates the same arithmetic together
with its gradient); they keep `stoix.utils.loss` call sites working on CUDA tensors.
"""
from __future__ import annotations

from typing import Tuple

import torch

from .. import ops


def _flat(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.float32).reshape(-1).contiguous()


def ppo_clip_loss(pi_log_prob_t: torch.Tensor, b_pi_log_prob_t: torch.Tensor, gae_t: torch.Tensor, epsilon: float) -> torch.Tensor:
    """stoix/utils/loss.py:17-32: -mean(min(ratio*A, clip(ratio, 1-eps, 1+eps)*A))."""
    return ops.ppo_clip_loss_value(_flat(pi_log_prob_t), _flat(b_pi_log_prob_t), _flat(gae_t), epsilon)


def ppo_penalty_loss(pi_log_prob_t: torch.Tensor, b_pi_log_prob_t: torch.Tensor, gae_t: torch.Tensor, beta: float, pi, b_pi
                     ) -> Tuple[torch.Tensor, torch.Tensor]:
    """stoix/utils/loss.py:35-47: (-mean(ratio*A - beta*kl), kl) with kl = mean(b_pi.kl_divergence(pi)), the KL of the
    behaviour policy from the current one.  `pi` / `b_pi` are the distributions of stoix_b200.networks.heads."""
    kl_rows = _flat(b_pi.kl_divergence(pi))
    return ops.ppo_penalty_loss_value(_flat(pi_log_prob_t), _flat(b_pi_log_prob_t), _flat(gae_t), kl_rows, beta)


def dpo_loss(pi_log_prob_t: torch.Tensor, b_pi_log_prob_t: torch.Tensor, gae_t: torch.Tensor, alpha: float, beta: float) -> torch.Tensor:
    """stoix/utils/loss.py:50-65: -mean(ratio*A - drift), drift = relu(x1 - alpha tanh(x1/alpha)) for A >= 0 and
    relu(x2 - beta tanh(x2/beta)) for A < 0, x1 = (ratio - 1) A, x2 = log(ratio) A."""
    return ops.dpo_loss_value(_flat(pi_log_prob_t), _flat(b_pi_log_prob_t), _flat(gae_t), alpha, beta)


def clipped_value_loss(pred_value_t: torch.Tensor, behavior_value_t: torch.Tensor, targets_t: torch.Tensor, epsilon: float) -> torch.Tensor:
    """stoix/utils/loss.py:68-78: 0.5*mean(max((v-tgt)^2, (v_clip-tgt)^2))."""
    return ops.clipped_value_loss_value(_flat(pred_value_t), _flat(behavior_value_t), _flat(targets_t), epsilon)


def _q_rows(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.float32).contiguous()


def _q_face(rule: str, q_tm1, a_tm1, r_t, d_t, q_t, q_aux, hyper) -> torch.Tensor:
    q_tm1 = _q_rows(q_tm1)
    A = int(q_tm1.shape[-1])
    if a_tm1.numel() and (int(a_tm1.min()) < 0 or int(a_tm1.max()) >= A):   # the kernel indexes row m at column a unchecked
        raise ops.StxError(f"{rule}: a_tm1 must lie in [0, {A}), got [{int(a_tm1.min())}, {int(a_tm1.max())}]")
    metrics = torch.zeros(1, dtype=torch.float32, device=q_tm1.device)
    ops.q_td_loss_grads(rule, q_tm1, _q_rows(q_t), a_tm1.to(torch.int32).reshape(-1).contiguous(), _flat(r_t), hyper, torch.empty_like(q_tm1),
                        metrics, discount=_flat(d_t), q_aux=None if q_aux is None else _q_rows(q_aux), scratch_key="q_td_face")
    return metrics[0]


def q_learning(q_tm1: torch.Tensor, a_tm1: torch.Tensor, r_t: torch.Tensor, d_t: torch.Tensor, q_t: torch.Tensor,
               huber_loss_parameter: float) -> torch.Tensor:
    """stoix/utils/loss.py:106-124: mean(l2 / Huber(r_t + d_t max_a q_t - q_tm1[a_tm1]))."""
    return _q_face("q_learning", q_tm1, a_tm1, r_t, d_t, q_t, None, ops.q_td_hyper(huber_delta=huber_loss_parameter))


def double_q_learning(q_tm1: torch.Tensor, q_t_value: torch.Tensor, a_tm1: torch.Tensor, r_t: torch.Tensor, d_t: torch.Tensor,
                      q_t_selector: torch.Tensor, huber_loss_parameter: float) -> torch.Tensor:
    """stoix/utils/loss.py:127-146: mean(l2 / Huber(r_t + d_t q_t_value[argmax q_t_selector] - q_tm1[a_tm1]))."""
    return _q_face("double_q_learning", q_tm1, a_tm1, r_t, d_t, q_t_value, q_t_selector, ops.q_td_hyper(huber_delta=huber_loss_parameter))


def munchausen_q_learning(q_tm1: torch.Tensor, q_tm1_target: torch.Tensor, a_tm1: torch.Tensor, r_t: torch.Tensor, d_t: torch.Tensor,
                          q_t_target: torch.Tensor, entropy_temperature: float, munchausen_coefficient: float, clip_value_min: float,
                          huber_loss_parameter: float) -> torch.Tensor:
    """stoix/utils/loss.py:190-223: the target r_t + alpha clip(tau log_softmax(q_tm1_target / tau)[a], clip_value_min, 0)
    + d_t tau logsumexp(q_t_target / tau), then mean(l2 / Huber(target - q_tm1[a_tm1]))."""
    h = ops.q_td_hyper(huber_delta=huber_loss_parameter, entropy_temperature=entropy_temperature, munchausen_coefficient=munchausen_coefficient,
                       clip_value_min=clip_value_min)
    return _q_face("munchausen_q_learning", q_tm1, a_tm1, r_t, d_t, q_t_target, q_tm1_target, h)


def _check_actions(who: str, a_tm1: torch.Tensor, A: int) -> torch.Tensor:
    if a_tm1.numel() and (int(a_tm1.min()) < 0 or int(a_tm1.max()) >= A):   # the kernels index row m at action a unchecked
        raise ops.StxError(f"{who}: a_tm1 must lie in [0, {A}), got [{int(a_tm1.min())}, {int(a_tm1.max())}]")
    return a_tm1.to(torch.int32).reshape(-1).contiguous()


def categorical_double_q_learning(q_logits_tm1: torch.Tensor, q_atoms_tm1: torch.Tensor, a_tm1: torch.Tensor, r_t: torch.Tensor, d_t: torch.Tensor,
                                  q_logits_t: torch.Tensor, q_atoms_t: torch.Tensor, q_t_selector: torch.Tensor) -> torch.Tensor:
    """stoix/utils/loss.py:81-103: per row, the cross-entropy of log_softmax(q_logits_tm1[a_tm1]) against
    rlax.categorical_l2_project(r_t + d_t q_atoms_t, softmax(q_logits_t[argmax q_t_selector]), q_atoms_tm1).  Logits (M, A, N),
    atoms (M, N), q_t_selector (M, A); returns the (M) vector."""
    M, A, N = q_logits_tm1.shape
    rows = lambda x: x.to(torch.float32).reshape(M, A * N).contiguous()
    a = _check_actions("categorical_double_q_learning", a_tm1, A)
    out = torch.empty(M, dtype=torch.float32, device=q_logits_tm1.device)
    metrics = torch.zeros(1, dtype=torch.float32, device=q_logits_tm1.device)
    ops.categorical_q_loss_grads(rows(q_logits_tm1), rows(q_logits_t), _q_rows(q_t_selector), _q_rows(q_atoms_tm1), _q_rows(q_atoms_t), a, _flat(r_t),
                                 ops.dist_q_hyper(), torch.empty(M, A * N, dtype=torch.float32, device=out.device), metrics, discount=_flat(d_t),
                                 loss_rows=out, scratch_key="c51_face")
    return out


def quantile_q_learning(dist_q_tm1: torch.Tensor, tau_q_tm1: torch.Tensor, a_tm1: torch.Tensor, r_t: torch.Tensor, d_t: torch.Tensor,
                        dist_q_t_selector: torch.Tensor, dist_q_t: torch.Tensor, huber_param: float = 0.0) -> torch.Tensor:
    """stoix/utils/loss.py:271-314: mean over rows of quantile_regression_loss(dist_q_tm1[:, :, a_tm1], tau_q_tm1, r_t + d_t
    dist_q_t[:, :, a*], huber_param), a* = argmax_a mean_i dist_q_t_selector[:, i, a].  Distributions (M, N, A) as the reference
    takes them (after its swapaxes), tau_q_tm1 (M, N); returns the scalar mean."""
    M, N, A = dist_q_tm1.shape
    rows = lambda x: x.to(torch.float32).transpose(1, 2).reshape(M, A * N).contiguous()   # to the head layout (M, A N)
    a = _check_actions("quantile_q_learning", a_tm1, A)
    metrics = torch.zeros(1, dtype=torch.float32, device=dist_q_tm1.device)
    ops.quantile_q_loss_grads(rows(dist_q_tm1), rows(dist_q_t), _q_rows(tau_q_tm1), a, _flat(r_t), ops.dist_q_hyper(huber_delta=huber_param),
                              torch.empty(M, A * N, dtype=torch.float32, device=metrics.device), metrics, A, q_sel=rows(dist_q_t_selector),
                              discount=_flat(d_t), scratch_key="qr_face")
    return metrics[0]
