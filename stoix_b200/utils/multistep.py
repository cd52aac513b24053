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


def batch_n_step_bootstrapped_returns(
    r_t: Array,
    discount_t: Array,
    v_t: Array,
    n: int,
    lambda_t: float = 1.0,
    stop_target_gradients: bool = True,
) -> Array:
    """Strided n-step bootstrapped returns of batch-major [B, T] sequences (multistep.py:148-210), one CUDA launch
    (stx_n_step_returns_f32) in the reference's operation order: the bootstrap values shifted by n and padded with v_t[:, -1], then
    G = r + d ((1 - lambda) v + lambda G) from step t + n - 1 down to t, the padded steps reading r = 0, d = 1, lambda = 1.

    Only a scalar lambda_t is implemented; an array raises.  `stop_target_gradients` is accepted for signature compatibility (the
    outputs never carry gradients)."""
    if getattr(lambda_t, "ndim", 0) > 0 or isinstance(lambda_t, (list, tuple)):
        raise ValueError("batch_n_step_bootstrapped_returns: only a scalar lambda_t is implemented (the V-MPO systems pass none); "
                         f"got an array of shape {tuple(getattr(lambda_t, 'shape', (len(lambda_t),)))}")
    lam = float(lambda_t)
    tm = lambda x: x.to(torch.float32).transpose(0, 1).contiguous()
    targets, _ = ops.n_step_returns(tm(r_t), tm(discount_t), tm(v_t), int(n), lam)
    return targets.transpose(0, 1).contiguous()


def batch_general_off_policy_returns_from_q_and_v(
    q_t: Array,
    v_t: Array,
    r_t: Array,
    discount_t: Array,
    c_t: Array,
    stop_target_gradients: bool = False,
) -> Array:
    """G_t = r_t + d_t (v_t - c_t q_t + c_t G_{t+1}) from G_{K-1} = r + d v (multistep.py:210-267), [B, K] inputs (q_t, c_t [B, K-1]),
    in one launch of stx_retrace_f32 with the weights c_t as given.  The outputs carry no gradients."""
    del stop_target_gradients
    tm = lambda x: x.to(torch.float32).transpose(0, 1).contiguous()
    out = ops.retrace(tm(q_t), tm(v_t), tm(r_t), tm(discount_t), None, 1.0, c_t=tm(c_t))
    return out.transpose(0, 1).contiguous()


def batch_retrace_continuous(
    q_tm1: Array,
    q_t: Array,
    v_t: Array,
    r_t: Array,
    discount_t: Array,
    log_rhos: Array,
    lambda_: float,
    stop_target_gradients: bool = True,
) -> Array:
    """Retrace error target - q_tm1 (multistep.py:270-311), [B, K] inputs (q_t, log_rhos [B, K-1]); one launch of stx_retrace_f32
    computes the targets.  Only a scalar lambda_ is implemented."""
    del stop_target_gradients
    tm = lambda x: x.to(torch.float32).transpose(0, 1).contiguous()
    target = ops.retrace(tm(q_t), tm(v_t), tm(r_t), tm(discount_t), tm(log_rhos), float(lambda_))
    return target.transpose(0, 1) - q_tm1
