"""Drop-in for the hot functions of stoix/utils/multistep.py.

`batch_truncated_generalized_advantage_estimation` keeps the reference signature and semantics
(stoix/utils/multistep.py:14-145) but runs as one CUDA launch (stx_gae_generic_f32, K2 in DESIGN.md)
instead of a T-iteration lax.scan; `batch_lambda_returns` (:314-408) and `batch_q_lambda` (:533-569) run on
the same scan (stx_lambda_returns_f32).  Inputs are CUDA torch tensors; there is no CPU path.
"""
from __future__ import annotations

from typing import Optional, Tuple, Union

import torch

from .. import ops

Array = torch.Tensor


def _is_float(x: Array) -> bool:
    return isinstance(x, torch.Tensor) and x.is_floating_point()


def batch_truncated_generalized_advantage_estimation(
    r_t: Array,
    discount_t: Array,
    lambda_: Union[Array, float],
    values: Optional[Array] = None,
    v_tm1: Optional[Array] = None,
    v_t: Optional[Array] = None,
    truncation_t: Optional[Array] = None,
    stop_target_gradients: bool = False,
    time_major: bool = False,
    standardize_advantages: bool = False,
) -> Tuple[Array, Array]:
    """Truncated GAE for batched sequences; argument meaning exactly as multistep.py:26-74.

    Returns (advantages, target_values) with the layout of `r_t` ([B, T], or [T, B] if time_major).
    `stop_target_gradients` is accepted for signature compatibility: the outputs never carry
    gradients (the kernels are not autograd-traced), which is what ff_ppo relies on.
    """
    del stop_target_gradients
    # multistep.py:77-92 -- the same argument validation, as assertions.
    if values is None:
        assert _is_float(v_tm1) and _is_float(v_t), "either `values` or both v_tm1 and v_t are required"
    else:
        assert _is_float(values) and values.ndim == 2, "`values` must be a rank-2 float tensor"
        if time_major:
            v_tm1, v_t = values[:-1], values[1:]
        else:
            v_tm1, v_t = values[:, :-1], values[:, 1:]
    for name, x in (("r_t", r_t), ("discount_t", discount_t), ("v_tm1", v_tm1), ("v_t", v_t)):
        assert _is_float(x) and x.ndim == 2, f"{name} must be a rank-2 float tensor"
    assert r_t.shape == v_tm1.shape == v_t.shape, "r_t, v_tm1 and v_t must have equal shapes"
    if truncation_t is not None:
        assert truncation_t.ndim == 2 and truncation_t.shape == discount_t.shape

    def prep(x: Optional[Array]) -> Optional[Array]:
        if x is None:
            return None
        x = x.to(torch.float32)
        return (x if time_major else x.t()).contiguous()  # multistep.py:107-113

    lam = lambda_
    if isinstance(lambda_, torch.Tensor) and lambda_.ndim > 0:  # multistep.py:97
        lam = prep(lambda_.expand_as(discount_t))
    adv, tgt, _ = ops.gae_generic(
        prep(r_t), prep(discount_t), lam, prep(v_tm1), prep(v_t), prep(truncation_t),
        standardize=2 if standardize_advantages else 0,
    )
    if not time_major:  # multistep.py:134-136
        adv, tgt = adv.t().contiguous(), tgt.t().contiguous()
    return adv, tgt


def batch_lambda_returns(
    r_t: Array,
    discount_t: Array,
    v_t: Array,
    lambda_: Union[Array, float] = 1.0,
    stop_target_gradients: bool = False,
    time_major: bool = False,
) -> Array:
    """Multistep lambda returns G_t = r_t + d_t [(1 - lambda_t) v_t + lambda_t G_{t+1}] from G_T = v_t[-1] (multistep.py:314-408):
    [B, T] inputs, or [T, B] if time_major; lambda_ a scalar or an array of the inputs' shape.  The outputs carry no gradients."""
    return _lambda_returns(r_t, discount_t, v_t, lambda_, time_major, q_values=False)


def batch_q_lambda(
    r_t: Array,
    discount_t: Array,
    q_t: Array,
    lambda_: Union[Array, float],
    stop_target_gradients: bool = True,
    time_major: bool = False,
) -> Array:
    """Peng's / Watkins' Q(lambda) targets (multistep.py:533-569): batch_lambda_returns with v_t = max_a q_t, q_t of shape [B, T, A]
    (or [T, B, A] if time_major).  The max over actions is taken inside the scan's load."""
    return _lambda_returns(r_t, discount_t, q_t, lambda_, time_major, q_values=True)


def _lambda_returns(r_t, discount_t, v_t, lambda_, time_major: bool, q_values: bool) -> Array:
    for name, x in (("r_t", r_t), ("discount_t", discount_t)):
        assert _is_float(x) and x.ndim == 2, f"{name} must be a rank-2 float tensor"
    assert _is_float(v_t) and v_t.ndim == (3 if q_values else 2), f"{'q_t' if q_values else 'v_t'} must be a rank-{3 if q_values else 2} float tensor"
    assert r_t.shape == discount_t.shape == v_t.shape[:2], "r_t, discount_t and the values must share their leading shape"

    def prep(x: Array) -> Array:
        x = x.to(torch.float32)
        return (x if time_major else x.transpose(0, 1)).contiguous()

    lam = lambda_
    if isinstance(lambda_, torch.Tensor) and lambda_.ndim > 0:
        lam = prep(lambda_.expand_as(discount_t))
    out = ops.lambda_returns(prep(r_t), prep(discount_t), prep(v_t), lam)
    return out if time_major else out.t().contiguous()
