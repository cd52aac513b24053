"""Activation lookup (stoix/networks/utils.py:7-25).  A torso here is a description, so the parser returns the NAME; the
fp32 CUDA path implements relu, tanh, silu / swish, elu, gelu (flax default: tanh approximation), sigmoid, softplus and
identity / none (csrc/stx_simt_gemm.cuh); the bf16 tensor-core (wgmma) kernels implement relu.  The remaining names of the reference's
table are not elementwise torso activations (normalise, softmax, log_softmax) or unused (log_sigmoid) and raise."""

_SUPPORTED = {"relu", "tanh", "silu", "swish", "elu", "gelu", "sigmoid", "softplus", "identity", "none"}
_KNOWN = _SUPPORTED | {"normalise", "softmax", "log_softmax", "log_sigmoid"}


def parse_activation_fn(activation_fn_name: str) -> str:
    if activation_fn_name not in _KNOWN:
        raise KeyError(activation_fn_name)
    if activation_fn_name not in _SUPPORTED:
        raise NotImplementedError(f"activation '{activation_fn_name}' has no kernel implementation in this build")
    return activation_fn_name
