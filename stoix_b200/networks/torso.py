"""MLPTorso -- constructor-compatible with stoix/networks/torso.py:12-33.

A torso here is a *description* (layer sizes, activation); the arithmetic runs in the fused CUDA MLP
kernels, so the object carries no tensors of its own."""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from .utils import parse_activation_fn


class MLPTorso:
    def __init__(self, layer_sizes: Sequence[int], activation: str = "relu", use_layer_norm: bool = False,
                 kernel_init: Optional[float] = None, activate_final: bool = True):
        if not activate_final:
            raise NotImplementedError("MLPTorso(activate_final=False) is not built (every PPO network config activates the last torso layer)")
        self.layer_sizes = tuple(int(s) for s in layer_sizes)
        self.activation = parse_activation_fn(activation)
        self.use_layer_norm = bool(use_layer_norm)   # Dense(use_bias=False) -> LayerNorm -> activation (torso.py:26-32)
        self.activate_final = True
        # orthogonal(sqrt(2)) is the reference default (torso.py:18)
        self.kernel_init_scale = float(np.sqrt(2.0)) if kernel_init is None else float(kernel_init)


class NoisyMLPTorso:
    """NoisyMLPTorso (stoix/networks/torso.py:36-57): NoisyLinear layers (stoix_b200.networks.dueling) instead of Dense.  As in the
    reference, its layers do not take kernel_init: every NoisyLinear kernel is lecun_normal."""

    def __init__(self, layer_sizes: Sequence[int], activation: str = "relu", use_layer_norm: bool = False, kernel_init: Optional[float] = None,
                 activate_final: bool = True, sigma_zero: float = 0.5):
        if not activate_final:
            raise NotImplementedError("NoisyMLPTorso(activate_final=False) is not built (the Rainbow network activates every torso layer)")
        self.layer_sizes = tuple(int(s) for s in layer_sizes)
        self.activation = parse_activation_fn(activation)
        self.use_layer_norm = bool(use_layer_norm)
        self.activate_final = True
        self.sigma_zero = float(sigma_zero)
