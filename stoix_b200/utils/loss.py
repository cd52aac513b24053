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
