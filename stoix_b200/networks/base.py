"""FeedForwardActor / FeedForwardCritic -- the `.init(key, x)` / `.apply(params, obs)` interface of
stoix/networks/base.py:18-59 over the fused CUDA MLP.

Parameters are a nested dict with the flax tree names of the reference
(`{'params': {'torso': {'Dense_0': {'kernel','bias'}, ...}, 'action_head': {'Dense_0': ...}}}`,
SURVEY.md A.2); every leaf is a VIEW into one flat fp32 arena (`tree.flat`), which is what the
kernels, the optimiser and the gradient all-reduce operate on."""
from __future__ import annotations

from typing import Any, Dict, Optional

import numpy as np
import torch

from .. import ops
from .inputs import ArrayInput


class ParamTree(dict):
    """Nested dict of views + the flat arena they alias (`flat`) and the network shape (`spec`)."""

    flat: torch.Tensor
    spec: ops.MlpSpec
    flat_bf16: Optional[torch.Tensor] = None


def _orthogonal(gen: torch.Generator, n_in: int, n_out: int, scale: float) -> torch.Tensor:
    """flax.linen.initializers.orthogonal(scale): scale * Q from the QR of a normal matrix."""
    rows, cols = max(n_in, n_out), min(n_in, n_out)
    a = torch.randn(rows, cols, generator=gen, dtype=torch.float64)
    q, r = torch.linalg.qr(a)
    q = q * torch.sign(torch.diagonal(r))
    if n_in < n_out:
        q = q.t()
    return (scale * q).to(torch.float32)


def _lecun_normal(gen: torch.Generator, n_in: int, n_out: int, scale: float) -> torch.Tensor:
    """flax.linen.initializers.lecun_normal() = variance_scaling(scale, "fan_in", "truncated_normal"): a normal truncated to
    [-2, 2] standard deviations, scaled to variance scale / fan_in (std sqrt(scale / n_in) / 0.8796..., the std of the unit
    normal truncated there).  Out-of-range draws are redrawn."""
    a = torch.randn(n_in, n_out, generator=gen, dtype=torch.float64)
    bad = a.abs() > 2.0
    while bool(bad.any()):
        a[bad] = torch.randn(int(bad.sum()), generator=gen, dtype=torch.float64)
        bad = a.abs() > 2.0
    return (a * (np.sqrt(scale / n_in) / 0.87962566103423978)).to(torch.float32)


_KERNEL_INITS = {"orthogonal": _orthogonal, "lecun_normal": _lecun_normal}


def build_param_tree(spec: ops.MlpSpec, flat: torch.Tensor, head_name: str, flat_bf16=None) -> ParamTree:
    sl = spec.layer_slices()
    n = spec.n_layers
    torso: Dict[str, Any] = {}
    for i in range(n - 1):
        torso[f"Dense_{i}"] = {"kernel": flat[sl[i][0]].view(spec.sizes[i], spec.sizes[i + 1]), "bias": flat[sl[i][1]]}
    head = {"Dense_0": {"kernel": flat[sl[n - 1][0]].view(spec.sizes[n - 1], spec.sizes[n]), "bias": flat[sl[n - 1][1]]}}
    for i, b in enumerate(spec.ln_bias_slices()):  # LayerNorm torsos: Dense_i has no bias; LayerNorm_i/{scale, bias} (flax auto-names)
        if b is not None:
            torso[f"LayerNorm_{i}"] = {"scale": torso[f"Dense_{i}"].pop("bias"), "bias": flat[b]}
    tree = ParamTree({"params": {"torso": torso, head_name: head}})
    tree.flat = flat[: spec.param_count]
    tree.spec = spec
    tree.flat_bf16 = flat_bf16
    return tree


class _FeedForward:
    head_name = "head"

    def __init__(self, head, torso, input_layer=None):
        self.head = head
        self.torso = torso
        self.input_layer = input_layer if input_layer is not None else ArrayInput()
        self.precision = ops.STX_PREC_F32

    def spec_for(self, obs_dim: int) -> ops.MlpSpec:
        return ops.MlpSpec(tuple([int(obs_dim), *self.torso.layer_sizes, int(self.head.out_dim)]), activation=self.torso.activation,
                           use_layer_norm=self.torso.use_layer_norm)

    def init(self, key, x: torch.Tensor, flat: Optional[torch.Tensor] = None) -> ParamTree:
        """Initialise parameters (orthogonal kernels, zero biases -- torso.py:18, heads.py:32,130).
        `key`: int seed or key tensor; `x`: example observation (leading batch dim).  If `flat` is
        given the parameters are created inside that arena slice (used by learner_setup to lay actor
        and critic out in one arena)."""
        from .heads import _seed_to_int

        spec = self.spec_for(x.shape[-1])
        device = x.device
        gen = torch.Generator().manual_seed(_seed_to_int(key) % (2**63))
        host = torch.zeros(spec.param_count, dtype=torch.float32)
        sl = spec.layer_slices()
        for i in range(spec.n_layers):
            scale = self.torso.kernel_init_scale if i < spec.n_layers - 1 else self.head.kernel_init_scale
            blocks = getattr(self.head, "kernel_blocks", None) if i == spec.n_layers - 1 else None
            if blocks:  # several Dense heads side by side (NormalAffineTanhDistributionHead): independent orthogonal blocks
                host[sl[i][0]] = torch.cat([_orthogonal(gen, spec.sizes[i], int(b), scale) for b in blocks], dim=1).reshape(-1)
            else:   # the head's kernel_init_kind (orthogonal unless the head names another, as the distributional Q heads do)
                kind = getattr(self.head, "kernel_init_kind", "orthogonal") if i == spec.n_layers - 1 else "orthogonal"
                host[sl[i][0]] = _KERNEL_INITS[kind](gen, spec.sizes[i], spec.sizes[i + 1], scale).reshape(-1)
            if spec.has_ln(i):
                host[sl[i][1]] = 1.0  # LayerNorm scale = ones, bias = zeros (flax defaults)
        if flat is None:
            flat = torch.zeros(spec.param_count, dtype=torch.float32, device=device)
        flat[: spec.param_count].copy_(host)
        return build_param_tree(spec, flat, self.head_name)

    def _forward(self, params: ParamTree, observation: torch.Tensor, *extra) -> torch.Tensor:
        obs = self.input_layer(observation, *extra)
        lead = obs.shape[:-1]
        x = obs.reshape(-1, obs.shape[-1])
        want = torch.bfloat16 if self.precision == ops.STX_PREC_BF16 else torch.float32
        if x.dtype != want:  # e.g. fp32 (normalised) observations into the bf16 kernels (cold paths: evaluator, user calls)
            x = ops.cast_bf16(x.contiguous()) if (want == torch.bfloat16 and x.dtype == torch.float32) else x.to(want)
        if not x.is_contiguous():
            x = x.contiguous()
        out = ops.mlp_forward(params.spec, params.flat, x, precision=self.precision, params_bf16=params.flat_bf16)
        return out.view(*lead, params.spec.sizes[-1])


class FeedForwardActor(_FeedForward):
    """stoix/networks/base.py:18-36: input_layer -> torso -> action_head."""

    head_name = "action_head"

    def __init__(self, action_head, torso, input_layer=None):
        super().__init__(action_head, torso, input_layer)
        self.action_head = action_head

    def apply(self, params: ParamTree, observation: torch.Tensor, input_kwargs: Optional[Dict[str, Any]] = None,
              torso_kwargs: Optional[Dict[str, Any]] = None, head_kwargs: Optional[Dict[str, Any]] = None):
        """base.py:26-36.  head_kwargs reach the head's distribution (e.g. {"epsilon": e} for DiscreteQNetworkHead); the input layer and
        the MLP torso take no keyword arguments, so input_kwargs / torso_kwargs must be empty."""
        if input_kwargs or torso_kwargs:
            raise TypeError("FeedForwardActor.apply: the input layer and the MLP torso take no keyword arguments")
        out = self._forward(params, observation)
        return self.action_head.distribution(out, **head_kwargs) if head_kwargs else self.action_head.distribution(out)

    __call__ = apply


class FeedForwardCritic(_FeedForward):
    """stoix/networks/base.py:39-59: input_layer -> torso -> critic_head, squeezed."""

    head_name = "critic_head"

    def __init__(self, critic_head, torso, input_layer=None):
        super().__init__(critic_head, torso, input_layer)
        self.critic_head = critic_head

    def apply(self, params: ParamTree, observation: torch.Tensor) -> torch.Tensor:
        return self._forward(params, observation).squeeze(-1)

    __call__ = apply


class FeedForwardQ(_FeedForward):
    """One continuous Q network = CompositeNetwork([EmbeddingActionInput, MLPTorso, ScalarCriticHead]) of the reference
    (stoix/networks/base.py:88-101 as built at stoix/systems/sac/ff_sac.py:357-366): apply(params, observation, action) -> (rows,)."""

    head_name = "critic_head"

    def __init__(self, critic_head, torso, input_layer=None):
        from .inputs import EmbeddingActionInput

        super().__init__(critic_head, torso, input_layer if input_layer is not None else EmbeddingActionInput())

    def apply(self, params: ParamTree, observation: torch.Tensor, action: torch.Tensor) -> torch.Tensor:
        return self._forward(params, observation, action).squeeze(-1)

    __call__ = apply


class MultiNetwork:
    """stoix/networks/base.py:104-121: applies several networks to the same input and stacks the outputs on a new last axis;
    parameters = a list with one ParamTree per member."""

    def __init__(self, networks):
        self.networks = list(networks)

    def init(self, keys, x_and_a, flats=None):
        from ..random import split

        ks = split(keys, len(self.networks)) if not isinstance(keys, (list, tuple)) else list(keys)
        return [n.init(k, x_and_a, flat=None if flats is None else flats[i]) for i, (n, k) in enumerate(zip(self.networks, ks))]

    def apply(self, params, *network_input) -> torch.Tensor:
        return torch.stack([n.apply(p, *network_input) for n, p in zip(self.networks, params)], dim=-1)

    __call__ = apply


def __getattr__(name):   # stoix.networks.base.{ScannedRNN, RecurrentActor, RecurrentCritic} (base.py:124-222) live in recurrent.py
    if name in ("ScannedRNN", "RecurrentActor", "RecurrentCritic"):
        from stoix_b200.networks import recurrent

        return getattr(recurrent, name)
    raise AttributeError(name)
