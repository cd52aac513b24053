"""Torch-tensor wrappers over the C ABI (include/stx.h).

PyTorch is plumbing here: it owns device memory and streams; every function below validates its
tensors and enqueues ONE call of libstoixb200 on the current CUDA stream.  No function has a CPU or
eager-PyTorch fallback -- a non-CUDA tensor raises StxError.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import STX_PREC_BF16, STX_PREC_F32, StxError

_scratch: Dict[Tuple, torch.Tensor] = {}
_retired: List[torch.Tensor] = []  # outgrown scratch tensors: a captured CUDA graph may still hold their raw pointers


def _need_cuda(*ts: Optional[torch.Tensor]) -> torch.device:
    dev = None
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda:
            raise StxError("stoix_b200 ops run only on CUDA tensors (no CPU fallback exists)")
        if not t.is_contiguous():
            raise StxError("stoix_b200 ops need contiguous tensors")
        dev = t.device
    return dev


def _p(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _zeros_scratch(key: Tuple, nbytes: int, device) -> torch.Tensor:
    """Zero-initialised scratch that persists (kernels restore their counters after use).

    A scratch that has been handed out is NEVER returned to the allocator: a captured update-step graph holds
    its raw pointer, so when a later (larger) request outgrows it the old tensor is retired, not freed --
    replays keep writing into memory nobody else owns.  Callers with their own life cycle (learner, evaluator)
    pass distinct keys so that they do not share workspaces in the first place."""
    full = key + (str(device),)
    t = _scratch.get(full)
    if t is None or t.numel() < nbytes:
        if t is not None:
            _retired.append(t)
        t = torch.zeros(max(int(nbytes), 256), dtype=torch.uint8, device=device)
        _scratch[full] = t
    return t


@dataclass(frozen=True)
class MlpSpec:
    """Layer widths of one network: sizes[0] = input dim, sizes[-1] = head width; torso activation and LayerNorm switch
    (stoix/networks/torso.py:12-33).  Arena layout per layer: W (in x out), then b (out) -- or, for LayerNorm torso
    layers, LayerNorm scale (out) and LayerNorm bias (out), the Dense having no bias (torso.py:26)."""

    sizes: Tuple[int, ...]
    activation: str = "relu"
    use_layer_norm: bool = False

    @property
    def n_layers(self) -> int:
        return len(self.sizes) - 1

    def has_ln(self, i: int) -> bool:
        return self.use_layer_norm and i < self.n_layers - 1

    @property
    def param_count(self) -> int:
        return sum(self.sizes[i] * self.sizes[i + 1] + (2 if self.has_ln(i) else 1) * self.sizes[i + 1] for i in range(self.n_layers))

    def layer_slices(self) -> List[Tuple[slice, slice]]:
        """(kernel slice, bias slice) per layer; for LayerNorm torso layers the second slice is the LayerNorm SCALE and
        `ln_bias_slices()[i]` the LayerNorm bias."""
        out, o = [], 0
        for i in range(self.n_layers):
            nw, nb = self.sizes[i] * self.sizes[i + 1], self.sizes[i + 1]
            out.append((slice(o, o + nw), slice(o + nw, o + nw + nb)))
            o += nw + (2 if self.has_ln(i) else 1) * nb
        return out

    def ln_bias_slices(self) -> List[Optional[slice]]:
        sl = self.layer_slices()
        return [slice(sl[i][1].stop, sl[i][1].stop + self.sizes[i + 1]) if self.has_ln(i) else None for i in range(self.n_layers)]

    def c_struct(self, params: torch.Tensor, params_bf16: Optional[torch.Tensor] = None) -> _lib.StxMlp:
        if self.n_layers < 1 or self.n_layers > _lib.STX_MAX_LAYERS:
            raise StxError(f"MLP with {self.n_layers} Dense layers unsupported (max {_lib.STX_MAX_LAYERS})")
        if params.dtype != torch.float32 or params.numel() < self.param_count:
            raise StxError("parameter arena must be float32 with at least param_count elements")
        m = self.shape_struct()
        m.params = params.data_ptr()
        m.params_bf16 = params_bf16.data_ptr() if params_bf16 is not None else None
        return m

    def shape_struct(self) -> _lib.StxMlp:
        if self.activation not in _lib.STX_ACTIVATIONS:
            raise StxError(f"activation '{self.activation}' has no kernel implementation")
        m = _lib.StxMlp()
        m.n_layers = self.n_layers
        for i, s in enumerate(self.sizes):
            m.sizes[i] = int(s)
        m.activation = _lib.STX_ACTIVATIONS[self.activation]
        m.use_layer_norm = int(bool(self.use_layer_norm))
        return m


def arena_offsets(actor: MlpSpec, critic: MlpSpec) -> Tuple[int, int, int]:
    """[actor | pad to 8 floats | critic | pad] -- mirrors stx_ppo_arena_offsets (8 floats keeps the bf16
    shadow of each network 16-byte aligned for TMA)."""
    coff = (actor.param_count + 7) // 8 * 8
    return 0, coff, coff + (critic.param_count + 7) // 8 * 8


# ------------------------------------------------------------------------------------------------
# K2 GAE
# ------------------------------------------------------------------------------------------------


def gae_ppo(reward, value, bootstrap_value, done, truncated, gamma, gae_lambda, reward_scale=1.0,
            standardize: int = 0, out=None):
    """ff_ppo.py:164-179 in one launch.  Inputs (T, E); done/truncated bool or uint8.
    Returns (advantages, targets, stats[2] or None)."""
    dev = _need_cuda(reward, value, bootstrap_value, done, truncated)
    T, E = reward.shape
    for t in (reward, value, bootstrap_value):
        if t.dtype != torch.float32 or t.shape != (T, E):
            raise StxError("gae_ppo: reward/value/bootstrap_value must be float32 (T, E)")
    done8 = done.view(torch.uint8) if done.dtype == torch.bool else done
    trunc8 = truncated.view(torch.uint8) if truncated.dtype == torch.bool else truncated
    if done8.dtype != torch.uint8 or trunc8.dtype != torch.uint8:
        raise StxError("gae_ppo: done/truncated must be bool or uint8")
    lib = _lib.load()
    adv, tgt = out if out is not None else (torch.empty_like(reward), torch.empty_like(reward))
    stats = torch.empty(2, dtype=torch.float32, device=dev) if standardize else None
    scratch = _zeros_scratch(("gae",), lib.stx_gae_scratch_bytes(T, E), dev)
    _lib.check(
        lib.stx_gae_ppo_f32(_p(reward), _p(value), _p(bootstrap_value), _p(done8), _p(trunc8), T, E,
                            float(gamma), float(gae_lambda), float(reward_scale), int(standardize),
                            _p(adv), _p(tgt), _p(stats), _p(scratch), _stream()),
        "stx_gae_ppo_f32",
    )
    return adv, tgt, stats


def gae_generic(r_t, discount_t, lambda_, v_tm1, v_t, truncation_t=None, standardize: int = 0):
    """Time-major generic face of multistep.py:14-145 (float discount / lambda / truncation arrays)."""
    dev = _need_cuda(r_t, discount_t, v_tm1, v_t, truncation_t)
    T, E = r_t.shape
    lam_t = None
    lam = 0.0
    if isinstance(lambda_, torch.Tensor) and lambda_.ndim > 0:
        lam_t = lambda_.to(torch.float32).expand(T, E).contiguous()
        _need_cuda(lam_t)
    else:
        lam = float(lambda_)
    lib = _lib.load()
    adv, tgt = torch.empty_like(r_t), torch.empty_like(r_t)
    stats = torch.empty(2, dtype=torch.float32, device=dev) if standardize else None
    scratch = _zeros_scratch(("gae",), lib.stx_gae_scratch_bytes(T, E), dev)
    _lib.check(
        lib.stx_gae_generic_f32(_p(r_t), _p(discount_t), _p(lam_t), lam, _p(v_tm1), _p(v_t),
                                _p(truncation_t), T, E, int(standardize), _p(adv), _p(tgt), _p(stats),
                                _p(scratch), _stream()),
        "stx_gae_generic_f32",
    )
    return adv, tgt, stats


# ------------------------------------------------------------------------------------------------
# K1 forward / categorical
# ------------------------------------------------------------------------------------------------


def mlp_forward(spec: MlpSpec, params: torch.Tensor, x: torch.Tensor, row_idx: Optional[torch.Tensor] = None,
                precision: int = STX_PREC_F32, params_bf16: Optional[torch.Tensor] = None,
                out: Optional[torch.Tensor] = None, ws_key: str = "fwd") -> torch.Tensor:
    dev = _need_cuda(params, x, row_idx, params_bf16)
    want = torch.float32 if precision == STX_PREC_F32 else torch.bfloat16
    if x.dtype != want or x.ndim != 2 or x.shape[1] != spec.sizes[0]:
        raise StxError(f"mlp_forward: x must be {want} (M, {spec.sizes[0]}), got {x.dtype} {tuple(x.shape)}")
    M = int(row_idx.numel()) if row_idx is not None else int(x.shape[0])
    if row_idx is not None and row_idx.dtype != torch.int32:
        raise StxError("mlp_forward: row_idx must be int32")
    lib = _lib.load()
    m = spec.c_struct(params, params_bf16)
    if out is None:
        out = torch.empty((M, spec.sizes[-1]), dtype=torch.float32, device=dev)
    nbytes = lib.stx_mlp_forward_workspace_bytes(C.byref(m), M, precision)
    ws = _zeros_scratch((ws_key, precision), nbytes, dev)
    _lib.check(
        lib.stx_mlp_forward(C.byref(m), _p(x), x.stride(0), _p(row_idx), M, _p(out), precision, _p(ws),
                            ws.numel(), _stream()),
        "stx_mlp_forward",
    )
    return out


NUM_SMS = 132  # H100 SXM


def set_forward_cta_budget(n: int) -> None:
    """Cap the grid of the persistent bf16 forward kernel for the launches that follow (0 = all SMs).  Host-side switch,
    read at launch (and therefore baked into a captured graph): used to run the critic next to the rollout kernel."""
    _lib.load().stx_tc_set_forward_ctas(int(n))


def tc_debug_forward(spec: MlpSpec, params: torch.Tensor, params_bf16: torch.Tensor, x: torch.Tensor):
    """bf16 tensor-core forward returning (out, h1, h2) -- test hook."""
    dev = _need_cuda(params, params_bf16, x)
    M = x.shape[0]
    out = torch.empty((M, spec.sizes[-1]), dtype=torch.float32, device=dev)
    h1 = torch.empty((M, 256), dtype=torch.float32, device=dev)
    h2 = torch.empty((M, 256), dtype=torch.float32, device=dev)
    m = spec.c_struct(params, params_bf16)
    _lib.check(_lib.load().stx_tc_debug_forward(C.byref(m), _p(x), x.stride(0), M, _p(out), _p(h1), _p(h2), _stream()),
               "stx_tc_debug_forward")
    return out, h1, h2


def categorical(logits: torch.Tensor, action: Optional[torch.Tensor] = None, seed: int = 0, offset: int = 0,
                dev_counter: Optional[torch.Tensor] = None, want_entropy: bool = False, out=None):
    """Sample (action is None) or score (action given) a Categorical(logits).
    Returns (action int32, log_prob, entropy or None)."""
    dev = _need_cuda(logits, action, dev_counter)
    E, A = logits.shape
    sample = action is None
    if out is not None:
        action_o, logp = out
        if sample:
            action = action_o
    else:
        logp = torch.empty(E, dtype=torch.float32, device=dev)
    if action is None:
        action = torch.empty(E, dtype=torch.int32, device=dev)
    if action.dtype != torch.int32:
        raise StxError("categorical: action must be int32")
    ent = torch.empty(E, dtype=torch.float32, device=dev) if want_entropy else None
    lib = _lib.load()
    _lib.check(
        lib.stx_categorical(_p(logits), E, A, int(sample), int(seed) & (2**64 - 1), int(offset), _p(dev_counter),
                            _p(action), _p(logp), _p(ent), _stream()),
        "stx_categorical",
    )
    return action, logp, ent


# ------------------------------------------------------------------------------------------------
# K3 PPO minibatch gradients
# ------------------------------------------------------------------------------------------------


@dataclass
class PpoBatch:
    """Flat (T*E) views of the PPOTransition fields the update needs (ppo_types.py:9-20)."""

    obs: torch.Tensor
    action: torch.Tensor
    log_prob: torch.Tensor
    value: torch.Tensor
    advantages: torch.Tensor
    targets: torch.Tensor
    adv_stats: Optional[torch.Tensor] = None
    perm: Optional[torch.Tensor] = None

    def c_struct(self) -> _lib.StxPpoBatch:
        b = _lib.StxPpoBatch()
        b.obs = self.obs.data_ptr()
        b.action = self.action.data_ptr()
        b.log_prob = self.log_prob.data_ptr()
        b.value = self.value.data_ptr()
        b.advantages = self.advantages.data_ptr()
        b.targets = self.targets.data_ptr()
        b.adv_stats = self.adv_stats.data_ptr() if self.adv_stats is not None else None
        b.perm = self.perm.data_ptr() if self.perm is not None else None
        b.B = int(self.action.numel())
        return b


def _shape_only_struct(spec: MlpSpec) -> _lib.StxMlp:
    m = spec.shape_struct()
    m.params = 256  # never dereferenced by the *_bytes queries
    m.params_bf16 = None
    return m


def ppo_workspace(actor: MlpSpec, critic: MlpSpec, mb: int, precision: int, device) -> torch.Tensor:
    """Zero-filled workspace for ppo_minibatch_grads (its first 256 bytes must start as zero)."""
    a, c = _shape_only_struct(actor), _shape_only_struct(critic)
    nbytes = _lib.load().stx_ppo_workspace_bytes(C.byref(a), C.byref(c), int(mb), precision)
    return torch.zeros(int(nbytes), dtype=torch.uint8, device=device)


def _minibatch_structs(who: str, actor: MlpSpec, critic: MlpSpec, param_arena: torch.Tensor, batch: PpoBatch, grad_arena: torch.Tensor,
                       metrics: torch.Tensor, workspace: torch.Tensor, hyper: Tuple, *, obs_dtype: torch.dtype, fp32_only: str = "",
                       n_metrics: int = 6, categorical: bool = True, param_arena_bf16: Optional[torch.Tensor] = None,
                       arenas: Tuple[torch.Tensor, ...] = (), adam_scratch: Optional[torch.Tensor] = None):
    """The checks every PPO minibatch wrapper shares, and its StxMlp (actor, critic), StxPpoBatch and StxPpoHyper.  hyper =
    (clip_eps, ent_coef, vf_coef, standardize, overwrite); `arenas` must hold the whole arena too; a tanh-Normal batch
    (categorical=False) holds float (B, A) actions that go to the C entry through StxTanhNormalPpo instead."""
    _need_cuda(param_arena, batch.obs, batch.action, batch.log_prob, batch.value, batch.advantages, batch.targets, batch.adv_stats, batch.perm,
               grad_arena, metrics, workspace, param_arena_bf16, *arenas)
    if (categorical and batch.action.dtype != torch.int32) or (batch.perm is not None and batch.perm.dtype != torch.int32):
        raise StxError(f"{who}: action / perm must be int32" if categorical else f"{who}: perm must be int32")
    if batch.obs.dtype != obs_dtype:
        raise StxError(f"{who}: obs must be {obs_dtype}" + (f" ({fp32_only} runs on the fp32 path)" if fp32_only else ""))
    _, coff, total = arena_offsets(actor, critic)
    if min(t.numel() for t in (param_arena, grad_arena) + arenas) < total or metrics.numel() < n_metrics:
        raise StxError(f"{who}: arena too small or metrics below {n_metrics} floats")
    a = actor.c_struct(param_arena, param_arena_bf16)
    c = critic.c_struct(param_arena[coff:], param_arena_bf16[coff:] if param_arena_bf16 is not None else None)
    b = batch.c_struct()
    if not categorical:
        B = int(batch.log_prob.numel())
        if batch.action.shape != (B, actor.sizes[-1] // 2):
            raise StxError(f"{who}: action must be float32 ({B}, {actor.sizes[-1] // 2})")
        b.action, b.B = None, B
    clip_eps, ent_coef, vf_coef, standardize, overwrite = hyper
    h = _lib.StxPpoHyper(float(clip_eps), float(ent_coef), float(vf_coef), int(bool(standardize)), int(bool(overwrite)), 0,
                         adam_scratch.data_ptr() if adam_scratch is not None else None)
    return a, c, b, h


def ppo_minibatch_grads(actor: MlpSpec, critic: MlpSpec, param_arena: torch.Tensor, batch: PpoBatch,
                        mb_off: int, mb: int, clip_eps: float, ent_coef: float, vf_coef: float,
                        standardize: bool, grad_arena: torch.Tensor, metrics: torch.Tensor,
                        workspace: torch.Tensor, precision: int = STX_PREC_F32, grad_weight: float = 1.0,
                        param_arena_bf16: Optional[torch.Tensor] = None, overwrite: bool = False,
                        adam_scratch: Optional[torch.Tensor] = None) -> None:
    """Accumulate grad_weight * d(loss)/d(params) of minibatch [mb_off, mb_off+mb) into grad_arena and
    the six loss metrics into `metrics` (ff_ppo.py:184-247)."""
    a, c, b, h = _minibatch_structs("ppo_minibatch_grads", actor, critic, param_arena, batch, grad_arena, metrics, workspace,
                                    (clip_eps, ent_coef, vf_coef, standardize, overwrite),
                                    obs_dtype=torch.float32 if precision == STX_PREC_F32 else torch.bfloat16,
                                    param_arena_bf16=param_arena_bf16, adam_scratch=adam_scratch)
    _lib.check(
        _lib.load().stx_ppo_minibatch_grads(C.byref(a), C.byref(c), C.byref(b), int(mb_off), int(mb), C.byref(h), float(grad_weight),
                                            _p(grad_arena), _p(metrics), precision, _p(workspace), workspace.numel(), _stream()),
        "stx_ppo_minibatch_grads",
    )


def ppo_minibatch_update(actor: MlpSpec, critic: MlpSpec, param_arena: torch.Tensor, batch: PpoBatch,
                         mb_off: int, mb: int, clip_eps: float, ent_coef: float, vf_coef: float,
                         standardize: bool, grad_arena: torch.Tensor, metrics: torch.Tensor,
                         workspace: torch.Tensor, plan: "AdamPlan", mu: torch.Tensor, nu: torch.Tensor,
                         param_arena_bf16: torch.Tensor, grad_weight: float = 1.0, grad_scale: float = 1.0) -> None:
    """One whole optimiser step on minibatch [mb_off, mb_off+mb) (ff_ppo.py:184-284): gradients of both losses,
    clip_by_global_norm + Adam on both networks, bf16 shadow refresh; the gradient reduction and the optimiser share
    one launch (stx_ppo_minibatch_update).  bf16 path, one shard, one device; `plan` must hold exactly the two
    segments (actor arena, critic arena).  Same results as ppo_minibatch_grads(overwrite=True) + clip_adam_step."""
    a, c, b, h = _minibatch_structs("ppo_minibatch_update", actor, critic, param_arena, batch, grad_arena, metrics, workspace,
                                    (clip_eps, ent_coef, vf_coef, standardize, True), obs_dtype=torch.bfloat16,
                                    param_arena_bf16=param_arena_bf16, arenas=(mu, nu, param_arena_bf16))
    if plan.nseg != 2:
        raise StxError("ppo_minibatch_update: the optimiser plan must have the two segments (actor, critic)")
    plan.hyper.grad_scale = float(grad_scale)
    plan.hyper.prenorm = 0
    opt = _lib.StxFusedAdam(_p(param_arena), _p(mu), _p(nu), _p(plan.counts), _p(plan.segs), plan.nseg, 0, plan.hyper,
                            _p(param_arena_bf16), _p(plan.gnorm), _p(plan.scratch))
    _lib.check(
        _lib.load().stx_ppo_minibatch_update(C.byref(a), C.byref(c), C.byref(b), int(mb_off), int(mb), C.byref(h), float(grad_weight),
                                             _p(grad_arena), _p(metrics), _p(workspace), workspace.numel(), C.byref(opt), _stream()),
        "stx_ppo_minibatch_update",
    )


def _loss_value(fn_name: str, a, b, c, eps: float) -> torch.Tensor:
    dev = _need_cuda(a, b, c)
    if not (a.dtype == b.dtype == c.dtype == torch.float32) or not (a.numel() == b.numel() == c.numel()):
        raise StxError(f"{fn_name}: expected three float32 tensors of equal size")
    lib = _lib.load()
    out = torch.empty(1, dtype=torch.float32, device=dev)
    scratch = _zeros_scratch(("loss",), lib.stx_loss_scratch_bytes(), dev)
    _lib.check(getattr(lib, fn_name)(_p(a), _p(b), _p(c), a.numel(), float(eps), _p(out), _p(scratch), _stream()), fn_name)
    return out[0]


def ppo_clip_loss_value(pi_log_prob_t, b_pi_log_prob_t, gae_t, epsilon) -> torch.Tensor:
    return _loss_value("stx_ppo_clip_loss", pi_log_prob_t, b_pi_log_prob_t, gae_t, epsilon)


def clipped_value_loss_value(pred_value_t, behavior_value_t, targets_t, epsilon) -> torch.Tensor:
    return _loss_value("stx_clipped_value_loss", pred_value_t, behavior_value_t, targets_t, epsilon)


# ------------------------------------------------------------------------------------------------
# K4 clip + Adam
# ------------------------------------------------------------------------------------------------


ADAM_MAX_SEGS = 8  # kAdamMaxSegs of stx_adam.cu


class AdamPlan:
    """Device-resident segment table + scratch for stx_clip_adam_step.

    segments: (offset, count, init_lr, max_grad_norm) per optimiser, 1..8 of them, disjoint.  The kernels read a segment as
    float4 items from `offset` on, so an offset must be a multiple of 4 floats (include/stx.h); a table that breaks this is
    refused here, before anything is allocated, instead of becoming a misaligned vector access on the device.

    rule: "adam" (optax.scale_by_adam, stx_clip_adam_step) or "radam" (optax.scale_by_radam with eps_root and threshold,
    stx_clip_radam_step); clip_adam_step runs whichever the plan holds."""

    def __init__(self, segments: Sequence[Tuple[int, int, float, float]], device, b1=0.9, b2=0.999, eps=1e-5,
                 decay=True, steps_per_update=1, num_updates=1, rule: str = "adam", eps_root: float = 0.0, threshold: float = 5.0):
        import numpy as np

        segments = [tuple(s) for s in segments]
        if not 1 <= len(segments) <= ADAM_MAX_SEGS:
            raise StxError(f"AdamPlan: {len(segments)} segments (1..{ADAM_MAX_SEGS} supported)")
        for off, cnt, _, _ in segments:
            if int(off) != off or int(cnt) != cnt:
                raise StxError(f"AdamPlan: segment ({off}, {cnt}): offset and count must be integers")
            if off < 0 or off % 4:
                raise StxError(f"AdamPlan: segment offset {off} is not a non-negative multiple of 4 floats (float4 access)")
            if cnt < 1:
                raise StxError(f"AdamPlan: segment at offset {off} has count {cnt} (at least 1)")
        spans = sorted((int(off), int(off) + int(cnt)) for off, cnt, _, _ in segments)
        for (a0, a1), (b0, b1_) in zip(spans, spans[1:]):
            if b0 < a1:
                raise StxError(f"AdamPlan: segments [{a0}, {a1}) and [{b0}, {b1_}) overlap")
        self.end = spans[-1][1]  # the arenas must hold at least this many floats
        self.nseg = len(segments)
        arr = (_lib.StxAdamSeg * self.nseg)()
        for i, (off, cnt, lr, mgn) in enumerate(segments):
            arr[i] = _lib.StxAdamSeg(int(off), int(cnt), float(lr), float(mgn))
        raw = np.frombuffer(bytes(arr), dtype=np.uint8).copy()
        self.segs = torch.from_numpy(raw).to(device)
        self.counts = torch.zeros(2 * self.nseg, dtype=torch.int32, device=device)
        self.gnorm = torch.zeros(self.nseg, dtype=torch.float32, device=device)
        self.scratch = torch.zeros(int(_lib.load().stx_adam_scratch_bytes(self.nseg)), dtype=torch.uint8, device=device)
        self.hyper = _lib.StxAdamHyper(float(b1), float(b2), float(eps), 1.0, int(bool(decay)),
                                       int(steps_per_update), int(num_updates), 0)
        if rule not in ("adam", "radam"):
            raise StxError(f"AdamPlan: rule={rule!r}; expected 'adam' or 'radam'")
        if rule == "radam" and eps_root < 0:
            raise StxError(f"AdamPlan: eps_root={eps_root} must be >= 0")
        self.rule = rule
        self.radam = _lib.StxRadamHyper(self.hyper, float(eps_root), float(threshold)) if rule == "radam" else None


def _check_adam_arenas(who: str, plan: AdamPlan, params_bf16: Optional[torch.Tensor], **arenas: torch.Tensor) -> None:
    """The fp32 arenas (and the bf16 shadow) must be contiguous, of the right dtype and hold every segment of the plan."""
    named = list(arenas.items()) + ([("params_bf16", params_bf16)] if params_bf16 is not None else [])
    for name, t in named:
        want = torch.bfloat16 if name == "params_bf16" else torch.float32
        if t.dtype != want or not t.is_contiguous():
            raise StxError(f"{who}: {name} must be a contiguous {want} tensor (got {t.dtype}"
                           f"{'' if t.is_contiguous() else ', not contiguous'})")
        if t.numel() < plan.end:
            raise StxError(f"{who}: {name} holds {t.numel()} elements, the last optimiser segment ends at {plan.end}")


def clip_adam_step(plan: AdamPlan, params: torch.Tensor, grads: torch.Tensor, mu: torch.Tensor, nu: torch.Tensor,
                   grad_scale: float = 1.0, params_bf16: Optional[torch.Tensor] = None, prenorm: bool = False) -> None:
    _check_adam_arenas("clip_adam_step", plan, params_bf16, params=params, grads=grads, mu=mu, nu=nu)
    _need_cuda(params, grads, mu, nu, params_bf16)
    plan.hyper.grad_scale = float(grad_scale)
    plan.hyper.prenorm = int(bool(prenorm))
    lib = _lib.load()
    if plan.rule == "radam":
        if prenorm:
            raise StxError("clip_adam_step: prenorm is not available with the radam rule")
        plan.radam.adam = plan.hyper
        _lib.check(
            lib.stx_clip_radam_step(_p(params), _p(grads), _p(mu), _p(nu), _p(plan.counts), _p(plan.segs), plan.nseg,
                                    C.byref(plan.radam), _p(params_bf16), _p(plan.gnorm), _p(plan.scratch), _stream()),
            "stx_clip_radam_step",
        )
        return
    _lib.check(
        lib.stx_clip_adam_step(_p(params), _p(grads), _p(mu), _p(nu), _p(plan.counts), _p(plan.segs), plan.nseg,
                               C.byref(plan.hyper), _p(params_bf16), _p(plan.gnorm), _p(plan.scratch), _stream()),
        "stx_clip_adam_step",
    )


class PeerGradBuffers:
    """Two gradient arenas in symmetric (peer-mapped) memory + the pointer tables the fused all-reduce/optimiser
    kernel needs.  torch.distributed._symmetric_memory is plumbing here (allocation + rendezvous of peer
    pointers); the all-reduce itself is done by stx_allreduce_clip_adam_step with direct NVLink loads."""

    def __init__(self, total: int, device, group=None):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem

        group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        if self.world > 8:
            raise StxError("fused all-reduce supports up to 8 ranks (one NVSwitch domain)")
        self.bufs, self.handles = [], []
        for _ in range(2):
            t = symm_mem.empty(int(total), dtype=torch.float32, device=device)
            t.zero_()
            self.bufs.append(t)
            self.handles.append(symm_mem.rendezvous(t, group))
        h0 = self.handles[0]
        pad_words = int(h0.signal_pad_size) // 4
        self.slot = pad_words - 64  # far from the channels torch's own barriers use at the start of the pad
        pad = h0.get_signal_pad(self.rank, (pad_words,), torch.uint32) if hasattr(h0, "get_signal_pad") else None
        if pad is not None:
            pad[self.slot:self.slot + 16] = 0
        self.grad_ptrs = [(C.c_void_p * self.world)(*[int(p) for p in h.buffer_ptrs]) for h in self.handles]
        self.pad_ptrs = (C.c_void_p * self.world)(*[int(p) for p in h0.signal_pad_ptrs])
        self.gsum = torch.zeros(int(total), dtype=torch.float32, device=device)
        # two-shot form: the reduced gradient of every rank is written by its peers -> symmetric too (+ the norm table)
        self.total = int(total)
        self.gsum2 = symm_mem.empty(self.total + 128, dtype=torch.float32, device=device)
        self.gsum2.zero_()
        self.gsum2_handle = symm_mem.rendezvous(self.gsum2, group)
        self.gsum2_ptrs = (C.c_void_p * self.world)(*[int(p) for p in self.gsum2_handle.buffer_ptrs])
        # 1 = one-shot (default), 2 = two-shot: the second cross-GPU hand-shake of two-shot (fence.sys after the peer stores,
        # last-block norm, signal flight) can cost more than the (W-1) extra arenas of 0.67 MB it saves.
        self.mode = int(os.environ.get("STX_ALLREDUCE_MODE", "1"))
        if self.total % 4 != 0:
            self.mode = 1
        torch.cuda.synchronize()
        dist.barrier(group)


def allreduce_clip_adam_step(plan: AdamPlan, peers: PeerGradBuffers, which: int, params: torch.Tensor, mu: torch.Tensor,
                             nu: torch.Tensor, params_bf16: Optional[torch.Tensor] = None) -> None:
    """Fused mean all-reduce of gradient arena `which` (0/1, ping-pong) + clip + Adam on every rank."""
    if plan.rule != "adam":
        raise StxError("allreduce_clip_adam_step: the fused all-reduce kernels implement the adam rule only; use an NCCL all-reduce "
                       "followed by clip_adam_step")
    _check_adam_arenas("allreduce_clip_adam_step", plan, params_bf16, params=params, mu=mu, nu=nu)
    _need_cuda(params, mu, nu, params_bf16)
    plan.hyper.grad_scale = 1.0 / peers.world
    plan.hyper.prenorm = 0
    if peers.mode == 2:
        _lib.check(
            _lib.load().stx_allreduce2_clip_adam_step(_p(params), peers.grad_ptrs[which], peers.gsum2_ptrs, peers.total, peers.pad_ptrs, peers.world,
                                                      peers.rank, peers.slot, _p(mu), _p(nu), _p(plan.counts), _p(plan.segs), plan.nseg,
                                                      C.byref(plan.hyper), _p(params_bf16), _p(plan.gnorm), _p(plan.scratch), 0, _stream()),
            "stx_allreduce2_clip_adam_step",
        )
        return
    _lib.check(
        _lib.load().stx_allreduce_clip_adam_step(_p(params), peers.grad_ptrs[which], peers.pad_ptrs, peers.world, peers.rank, peers.slot,
                                                 _p(peers.gsum), _p(mu), _p(nu), _p(plan.counts), _p(plan.segs), plan.nseg,
                                                 C.byref(plan.hyper), _p(params_bf16), _p(plan.gnorm), _p(plan.scratch), _stream()),
        "stx_allreduce_clip_adam_step",
    )


# ------------------------------------------------------------------------------------------------
# shuffle / env / misc
# ------------------------------------------------------------------------------------------------


def make_permutation(n: int, seed: int, stream_id: int, device=None, dev_counter: Optional[torch.Tensor] = None,
                     out: Optional[torch.Tensor] = None) -> torch.Tensor:
    if out is None:
        out = torch.empty(n, dtype=torch.int32, device=device)
    _need_cuda(out, dev_counter)
    _lib.check(
        _lib.load().stx_make_permutation(_p(out), int(n), int(seed) & (2**64 - 1), int(stream_id), _p(dev_counter), _stream()),
        "stx_make_permutation",
    )
    return out


def counter_add(counter: torch.Tensor, inc: int) -> None:
    _need_cuda(counter)
    if counter.dtype != torch.int64:
        raise StxError("counter must be an int64 tensor (used as uint64)")
    _lib.check(_lib.load().stx_counter_add(_p(counter), int(inc), _stream()), "stx_counter_add")


def synth_env_step(E, D, seed, step, p_term, p_trunc, action, obs_out, next_obs, reward, done, truncated,
                   run_return, run_length, ep_return, ep_length, is_terminal, dev_counter=None) -> None:
    _need_cuda(action, obs_out, next_obs, reward, done, truncated, run_return, run_length, ep_return,
               ep_length, is_terminal, dev_counter)
    bf16 = obs_out.dtype == torch.bfloat16
    if next_obs.dtype != obs_out.dtype:
        raise StxError("synth_env_step: obs_out / next_obs dtype mismatch")
    _lib.check(
        _lib.load().stx_synth_env_step(int(E), int(D), int(seed) & (2**64 - 1), int(step), _p(dev_counter),
                                       float(p_term), float(p_trunc), _p(action), _p(obs_out), _p(next_obs),
                                       int(bf16), _p(reward), _p(done), _p(truncated), _p(run_return),
                                       _p(run_length), _p(ep_return), _p(ep_length), _p(is_terminal), _stream()),
        "stx_synth_env_step",
    )


def tc_rollout_synth(spec: MlpSpec, params, params_bf16, obs, next_obs, action, log_prob, reward, done, truncated, ep_return,
                     ep_length, is_terminal, run_return, run_length, env_seed, env_step, env_counter, p_term, p_trunc, cat_seed,
                     cat_offset, cat_counter) -> None:
    """Fused T-step rollout of the synthetic env (stx_tc_rollout_synth); buffers are the time-major trajectory."""
    _need_cuda(params, params_bf16, obs, next_obs, action, log_prob, reward, done, truncated, ep_return, ep_length, is_terminal,
               run_return, run_length, env_counter, cat_counter)
    if obs.dtype != torch.bfloat16 or next_obs.dtype != torch.bfloat16:
        raise StxError("tc_rollout_synth: observation buffers must be bfloat16")
    T, E = int(action.shape[0]), int(action.shape[1])
    m = spec.c_struct(params, params_bf16)
    _lib.check(
        _lib.load().stx_tc_rollout_synth(C.byref(m), _p(obs), _p(next_obs), _p(action), _p(log_prob), _p(reward), _p(done), _p(truncated),
                                         _p(ep_return), _p(ep_length), _p(is_terminal), _p(run_return), _p(run_length), T, E,
                                         int(env_seed) & (2**64 - 1), int(env_step), _p(env_counter), float(p_term), float(p_trunc),
                                         int(cat_seed) & (2**64 - 1), int(cat_offset), _p(cat_counter), _stream()),
        "stx_tc_rollout_synth",
    )


def cast_bf16(src: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _need_cuda(src)
    if out is None:
        out = torch.empty(src.shape, dtype=torch.bfloat16, device=src.device)
    _lib.check(_lib.load().stx_cast_f32_to_bf16(_p(src), _p(out), src.numel(), _stream()), "stx_cast_f32_to_bf16")
    return out


# ------------------------------------------------------------------------------------------------
# observation normalisation (stoix/utils/running_statistics.py)
# ------------------------------------------------------------------------------------------------


def running_stats_accumulate(x: torch.Tensor, mean: torch.Tensor, weights: Optional[torch.Tensor] = None,
                             out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """sums[2D+1] (float64) = [sum w (x - mean), sum w (x - mean)^2, sum w] over the rows of x (rows, D) float32."""
    dev = _need_cuda(x, mean, weights, out)
    D = int(mean.numel())
    if x.dtype != torch.float32 or mean.dtype != torch.float32 or x.numel() % D != 0:
        raise StxError("running_stats_accumulate: x must be float32 with a trailing feature dim equal to mean.numel()")
    rows = x.numel() // D
    if weights is not None and (weights.dtype != torch.float32 or weights.numel() != rows):
        raise StxError("running_stats_accumulate: weights must be float32 with one entry per batch row")
    lib = _lib.load()
    if out is None:
        out = torch.empty(2 * D + 1, dtype=torch.float64, device=dev)
    scratch = _zeros_scratch(("rstats", D), lib.stx_running_stats_scratch_bytes(D), dev)
    _lib.check(lib.stx_running_stats_accumulate(_p(x), _p(weights), rows, D, _p(mean), _p(out), _p(scratch), _stream()),
               "stx_running_stats_accumulate")
    return out


def running_stats_finalize(sums: torch.Tensor, count: torch.Tensor, mean: torch.Tensor, summed_variance: torch.Tensor,
                           std: torch.Tensor, std_min_value: float, std_max_value: float) -> None:
    """In-place Welford update of (count int64[1], mean, summed_variance, std float32[D]) from accumulated sums."""
    _need_cuda(sums, count, mean, summed_variance, std)
    D = int(mean.numel())
    if sums.dtype != torch.float64 or sums.numel() != 2 * D + 1 or count.dtype != torch.int64:
        raise StxError("running_stats_finalize: sums must be float64[2D+1], count int64[1]")
    _lib.check(_lib.load().stx_running_stats_finalize(_p(sums), D, _p(count), _p(mean), _p(summed_variance), _p(std),
                                                      float(std_min_value), float(std_max_value), _stream()),
               "stx_running_stats_finalize")


def obs_normalize(x: torch.Tensor, mean: torch.Tensor, std: torch.Tensor, out: Optional[torch.Tensor] = None,
                  out_dtype: torch.dtype = torch.float32, max_abs_value: Optional[float] = None) -> torch.Tensor:
    """(x - mean) / std over the trailing feature dim (running_statistics.py:348-363); out float32 or bfloat16."""
    dev = _need_cuda(x, mean, std, out)
    D = int(mean.numel())
    if x.dtype != torch.float32 or x.numel() % D != 0:
        raise StxError("obs_normalize: x must be float32 with a trailing feature dim equal to mean.numel()")
    if out is None:
        out = torch.empty(x.shape, dtype=out_dtype, device=dev)
    if out.dtype not in (torch.float32, torch.bfloat16) or out.numel() != x.numel():
        raise StxError("obs_normalize: out must be float32 or bfloat16 with x's element count")
    _lib.check(_lib.load().stx_obs_normalize(_p(x), x.numel() // D, D, _p(mean), _p(std),
                                             float(max_abs_value) if max_abs_value is not None else 0.0, _p(out),
                                             int(out.dtype == torch.bfloat16), _stream()), "stx_obs_normalize")
    return out


# ------------------------------------------------------------------------------------------------
# generic train-mode MLP (fp32) + ff_sac building blocks (stoix/systems/sac/ff_sac.py:149-321)
# ------------------------------------------------------------------------------------------------


def mlp_train_workspace(spec: MlpSpec, M: int, device) -> torch.Tensor:
    """Zero-filled workspace for mlp_forward_train / mlp_backward of a batch of M rows (one per pending backward)."""
    m = _shape_only_struct(spec)
    return torch.zeros(int(_lib.load().stx_mlp_train_workspace_bytes(C.byref(m), int(M))), dtype=torch.uint8, device=device)


def mlp_forward_train(spec: MlpSpec, params: torch.Tensor, x: torch.Tensor, ws: torch.Tensor, out: Optional[torch.Tensor] = None,
                      row_idx: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Forward that keeps the torso pre-activations (and LayerNorm statistics) in `ws` for mlp_backward.  x (rows, >= in_dim)
    float32, rows may be wider than the input dim (leading dimension x.stride(0)); row_idx (int32, M): batch row m = x[row_idx[m]]."""
    dev = _need_cuda(params, ws, out, row_idx)
    if not x.is_cuda or x.dtype != torch.float32 or x.ndim != 2 or x.stride(1) != 1 or x.shape[1] < spec.sizes[0]:
        raise StxError("mlp_forward_train: x must be a CUDA float32 matrix with unit column stride and >= in_dim columns")
    if row_idx is not None and row_idx.dtype != torch.int32:
        raise StxError("mlp_forward_train: row_idx must be int32")
    M = int(row_idx.numel()) if row_idx is not None else int(x.shape[0])
    if out is None:
        out = torch.empty((M, spec.sizes[-1]), dtype=torch.float32, device=dev)
    m = spec.c_struct(params)
    _lib.check(_lib.load().stx_mlp_forward_train(C.byref(m), _p(x), x.stride(0), _p(row_idx), M, _p(out), _p(ws), ws.numel(), _stream()),
               "stx_mlp_forward_train")
    return out


def mlp_backward(spec: MlpSpec, params: torch.Tensor, x: torch.Tensor, d_out: torch.Tensor, ws: torch.Tensor,
                 net_grad: Optional[torch.Tensor] = None, grad_weight: float = 1.0, overwrite: bool = True,
                 d_input: Optional[torch.Tensor] = None, row_idx: Optional[torch.Tensor] = None) -> None:
    """Backward of the forward that filled `ws`: parameter gradients into net_grad (layout of the parameter arena) and / or
    d(loss)/d(input) into d_input (M, in_dim) dense."""
    _need_cuda(params, d_out, ws, net_grad, d_input, row_idx)
    M = int(row_idx.numel()) if row_idx is not None else int(x.shape[0])
    if d_out.dtype != torch.float32 or d_out.numel() != M * spec.sizes[-1]:
        raise StxError("mlp_backward: d_out must be float32 (M, out_dim)")
    if d_input is not None and (d_input.dtype != torch.float32 or d_input.numel() != M * spec.sizes[0]):
        raise StxError("mlp_backward: d_input must be float32 (M, in_dim)")
    m = spec.c_struct(params)
    _lib.check(_lib.load().stx_mlp_backward(C.byref(m), _p(x), x.stride(0), _p(row_idx), M, _p(d_out), _p(ws), ws.numel(), float(grad_weight),
                                            _p(net_grad), int(bool(overwrite)), _p(d_input), _stream()), "stx_mlp_backward")


def tanh_normal_sample(head_out: torch.Tensor, minimum: float, maximum: float, min_scale: float = 1e-3, eps: Optional[torch.Tensor] = None,
                       seed: int = 0, offset: int = 0, dev_counter: Optional[torch.Tensor] = None, action_out: Optional[torch.Tensor] = None,
                       want_eps: bool = True):
    """NormalAffineTanhDistributionHead sample + log_prob (heads.py:44-65, distributions.py:19-79) on head_out (M, 2A).
    `action_out` may be a column block of a wider matrix (e.g. the Q networks' concat input).  Returns (action, log_prob, eps)."""
    dev = _need_cuda(head_out, eps, dev_counter)
    M, A2 = head_out.shape
    A = A2 // 2
    if action_out is None:
        action_out = torch.empty(M, A, dtype=torch.float32, device=dev)
    if action_out.stride(1) != 1 or action_out.shape != (M, A):
        raise StxError("tanh_normal_sample: action_out must be (M, A) with unit column stride")
    logp = torch.empty(M, dtype=torch.float32, device=dev)
    eps_out = torch.empty(M, A, dtype=torch.float32, device=dev) if (want_eps and eps is None) else None
    _lib.check(_lib.load().stx_tanh_normal_sample(_p(head_out), M, A, _p(eps), int(seed) & (2**64 - 1), int(offset), _p(dev_counter), float(minimum),
                                                  float(maximum), float(min_scale), _p(action_out), action_out.stride(0), _p(logp), _p(eps_out),
                                                  _stream()), "stx_tanh_normal_sample")
    return action_out, logp, (eps if eps is not None else eps_out)


def tanh_normal_backward(head_out: torch.Tensor, eps: torch.Tensor, minimum: float, maximum: float, log_alpha: Optional[torch.Tensor],
                         g_logp_scale: float, g_action: Optional[torch.Tensor], min_scale: float = 1e-3,
                         out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """d(loss)/d(head_out) for loss = g_logp_scale * exp(log_alpha) * sum log_prob + sum g_action * action (eps fixed)."""
    dev = _need_cuda(head_out, eps, log_alpha)
    M, A2 = head_out.shape
    if out is None:
        out = torch.empty(M, A2, dtype=torch.float32, device=dev)
    if g_action is not None and (g_action.stride(1) != 1 or g_action.shape != (M, A2 // 2)):
        raise StxError("tanh_normal_backward: g_action must be (M, A) with unit column stride")
    _lib.check(_lib.load().stx_tanh_normal_backward(_p(head_out), _p(eps), M, A2 // 2, float(minimum), float(maximum), float(min_scale), _p(log_alpha),
                                                    float(g_logp_scale), _p(g_action), g_action.stride(0) if g_action is not None else 0, _p(out),
                                                    _stream()), "stx_tanh_normal_backward")
    return out


def tanh_normal_log_prob(head_out: torch.Tensor, action: torch.Tensor, minimum: float, maximum: float, min_scale: float = 1e-3,
                         out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """log_prob of GIVEN actions (M, A) under the tanh-Normal head on head_out (M, 2A) (distributions.py:56-80, the inverse path
    with the clipped tails).  `action` may be a column block of a wider matrix (unit column stride)."""
    dev = _need_cuda(head_out, out)
    M, A2 = head_out.shape
    A = A2 // 2
    if not action.is_cuda or action.dtype != torch.float32 or action.shape != (M, A) or action.stride(1) != 1:
        raise StxError("tanh_normal_log_prob: action must be a CUDA float32 (M, A) matrix with unit column stride")
    if out is None:
        out = torch.empty(M, dtype=torch.float32, device=dev)
    _lib.check(_lib.load().stx_tanh_normal_log_prob(_p(head_out), M, A, _p(action), action.stride(0), float(minimum), float(maximum),
                                                    float(min_scale), _p(out), _stream()), "stx_tanh_normal_log_prob")
    return out


def tanh_normal_entropy(head_out: torch.Tensor, minimum: float, maximum: float, min_scale: float = 1e-3, eps: Optional[torch.Tensor] = None,
                        seed: int = 0, offset: int = 0, dev_counter: Optional[torch.Tensor] = None,
                        want_eps: bool = False) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """The seeded one-sample entropy estimate of the tanh-Normal head per row (distributions.py:85-88).  Returns (entropy, eps)."""
    dev = _need_cuda(head_out, eps, dev_counter)
    M, A2 = head_out.shape
    ent = torch.empty(M, dtype=torch.float32, device=dev)
    eps_out = torch.empty(M, A2 // 2, dtype=torch.float32, device=dev) if (want_eps and eps is None) else None
    _lib.check(_lib.load().stx_tanh_normal_entropy(_p(head_out), M, A2 // 2, _p(eps), int(seed) & (2**64 - 1), int(offset), _p(dev_counter),
                                                   float(minimum), float(maximum), float(min_scale), _p(ent), _p(eps_out), _stream()),
               "stx_tanh_normal_entropy")
    return ent, (eps if eps is not None else eps_out)


def _tanh_normal_ppo(action,minimum, maximum, min_scale, seed, offset, dev_counter, eps_in, eps_out) -> _lib.StxTanhNormalPpo:
    _need_cuda(action, eps_in, eps_out, dev_counter)
    for t, name in ((action, "action"), (eps_in, "eps_in"), (eps_out, "eps_out")):
        if t is not None and t.dtype != torch.float32:
            raise StxError(f"tanh-Normal PPO head: {name} must be float32")
    if dev_counter is not None and dev_counter.dtype != torch.int64:
        raise StxError("tanh-Normal PPO head: dev_counter must be an int64 tensor (used as uint64)")
    return _lib.StxTanhNormalPpo(_p(action), _p(eps_in), _p(eps_out), _p(dev_counter), int(seed) & (2**64 - 1), int(offset), float(minimum),
                                 float(maximum), float(min_scale), 0)


def _head_grads_io(who: str, head_out: torch.Tensor, idx: Optional[torch.Tensor], d_head_out: Optional[torch.Tensor],
                   metrics: Optional[torch.Tensor], n_metrics: int, scratch_key: str, *tensors: Optional[torch.Tensor]):
    """The checks and buffers the actor head-grad wrappers share: (d_head_out, metrics, scratch), allocating what is not given
    (metrics zeroed, 6 or 8 floats)."""
    dev = _need_cuda(head_out, idx, d_head_out, metrics, *tensors)
    if idx is not None and idx.dtype != torch.int32:
        raise StxError(f"{who}: idx must be int32")
    d_head_out = torch.empty(head_out.shape, dtype=torch.float32, device=dev) if d_head_out is None else d_head_out
    metrics = torch.zeros(6 if n_metrics <= 6 else 8, dtype=torch.float32, device=dev) if metrics is None else metrics
    if metrics.numel() < n_metrics:
        raise StxError(f"{who}: metrics must hold at least {n_metrics} floats")
    return d_head_out, metrics, _zeros_scratch((scratch_key,), _lib.load().stx_ppo_head_scratch_bytes(head_out.shape[0]), dev)


def ppo_tanh_normal_head_grads(head_out: torch.Tensor, idx: Optional[torch.Tensor], action: torch.Tensor, logp_old: torch.Tensor,
                               adv: torch.Tensor, adv_stats: Optional[torch.Tensor], clip_eps: float, ent_coef: float, minimum: float,
                               maximum: float, min_scale: float = 1e-3, seed: int = 0, offset: int = 0,
                               dev_counter: Optional[torch.Tensor] = None, eps_in: Optional[torch.Tensor] = None,
                               eps_out: Optional[torch.Tensor] = None, d_head_out: Optional[torch.Tensor] = None,
                               metrics: Optional[torch.Tensor] = None, weight: float = 1.0, row0: int = 0,
                               scratch_key: str = "ppo_tanh_normal_head") -> Tuple[torch.Tensor, torch.Tensor]:
    """The actor half of continuous PPO's _update_minibatch on head outputs computed elsewhere (stx_ppo_tanh_normal_head_grads):
    row m of head_out (mb, 2A) pairs with batch row idx[m] (or row0 + m) of action (B, A) / logp_old / adv.
    Returns (d_head_out, metrics[6]); metrics slots 0, 1, 3 = actor_loss, entropy, mean advantage."""
    who = "ppo_tanh_normal_head_grads"
    d_head_out, metrics, scratch = _head_grads_io(who, head_out, idx, d_head_out, metrics, 6, scratch_key, action, logp_old, adv, adv_stats)
    mb, A2 = head_out.shape
    if action.ndim != 2 or action.shape[1] != A2 // 2:
        raise StxError(f"{who}: action must be (B, A) with 2A = head_out.shape[1]")
    hd = _tanh_normal_ppo(action, minimum, maximum, min_scale, seed, offset, dev_counter, eps_in, eps_out)
    _lib.check(_lib.load().stx_ppo_tanh_normal_head_grads(_p(head_out), _p(idx), int(row0), C.byref(hd), _p(logp_old), _p(adv), _p(adv_stats), mb,
                                                          A2 // 2, float(clip_eps), float(ent_coef), _p(d_head_out), _p(metrics), float(weight),
                                                          _p(scratch), _stream()), "stx_ppo_tanh_normal_head_grads")
    return d_head_out, metrics


def ppo_continuous_minibatch_grads(actor: MlpSpec, critic: MlpSpec, param_arena: torch.Tensor, batch: PpoBatch, mb_off: int, mb: int,
                                   clip_eps: float, ent_coef: float, vf_coef: float, standardize: bool, grad_arena: torch.Tensor,
                                   metrics: torch.Tensor, workspace: torch.Tensor, minimum: float, maximum: float, min_scale: float = 1e-3,
                                   seed: int = 0, offset: int = 0, dev_counter: Optional[torch.Tensor] = None,
                                   eps_in: Optional[torch.Tensor] = None, eps_out: Optional[torch.Tensor] = None,
                                   precision: int = STX_PREC_F32, grad_weight: float = 1.0, overwrite: bool = False) -> None:
    """ppo_minibatch_grads for a tanh-Normal actor (ff_ppo_continuous.py:184-247): batch.action holds the float (B, A) actions.
    Entropy noise from Philox (seed, minibatch row, offset + *dev_counter) unless eps_in (mb, A) is given; eps_out records it."""
    a, c, b, h = _minibatch_structs("ppo_continuous_minibatch_grads", actor, critic, param_arena, batch, grad_arena, metrics, workspace,
                                    (clip_eps, ent_coef, vf_coef, standardize, overwrite), obs_dtype=torch.float32,
                                    fp32_only="the tanh-Normal head", categorical=False)
    hd = _tanh_normal_ppo(batch.action, minimum, maximum, min_scale, seed, offset, dev_counter, eps_in, eps_out)
    _lib.check(
        _lib.load().stx_ppo_continuous_minibatch_grads(C.byref(a), C.byref(c), C.byref(b), C.byref(hd), int(mb_off), int(mb), C.byref(h),
                                                       float(grad_weight), _p(grad_arena), _p(metrics), int(precision), _p(workspace),
                                                       workspace.numel(), _stream()),
        "stx_ppo_continuous_minibatch_grads",
    )


# ------------------------------------------------------------------------------------------------
# PPO variants: KL penalty (ff_ppo_penalty*, loss.py:35-47) and DPO (ff_dpo_continuous, loss.py:50-65)
# ------------------------------------------------------------------------------------------------

STX_PPO_KL_PENALTY, STX_PPO_DPO = _lib.STX_PPO_KL_PENALTY, _lib.STX_PPO_DPO
METRIC_SLOT_KL = 6  # metrics slot of kl_divergence (0 actor_loss, 1 entropy, 2 value_loss, 3-5 as on the clip path)


def _variant(kind: int, behaviour: Optional[torch.Tensor], kl_coef: float, dpo_alpha: float, dpo_beta: float) -> _lib.StxPpoVariant:
    _need_cuda(behaviour)
    if behaviour is not None and behaviour.dtype != torch.float32:
        raise StxError("PPO variant: behaviour head outputs must be float32")
    if kind == STX_PPO_KL_PENALTY and behaviour is None:
        raise StxError("PPO variant: the KL penalty needs the behaviour head outputs")
    return _lib.StxPpoVariant(_p(behaviour), int(kind), float(kl_coef), float(dpo_alpha), float(dpo_beta))


def categorical_kl(logits_p: torch.Tensor, logits_q: torch.Tensor) -> torch.Tensor:
    """KL(Categorical(logits_p) || Categorical(logits_q)) per row of (M, A) logits."""
    dev = _need_cuda(logits_p, logits_q)
    if logits_p.shape != logits_q.shape or logits_p.dtype != torch.float32 or logits_q.dtype != torch.float32 or logits_p.ndim != 2:
        raise StxError("categorical_kl: expected two float32 (M, A) logit matrices of the same shape")
    out = torch.empty(logits_p.shape[0], dtype=torch.float32, device=dev)
    _lib.check(_lib.load().stx_categorical_kl(_p(logits_p), _p(logits_q), logits_p.shape[0], logits_p.shape[1], _p(out), _stream()),
               "stx_categorical_kl")
    return out


def tanh_normal_kl(head_p: torch.Tensor, head_q: torch.Tensor, min_scale: float = 1e-3) -> torch.Tensor:
    """KL(p || q) per row of two tanh-Normal heads (M, 2A) with the same bounds: the KL of the base Normals summed over the dims."""
    dev = _need_cuda(head_p, head_q)
    if head_p.shape != head_q.shape or head_p.dtype != torch.float32 or head_q.dtype != torch.float32 or head_p.ndim != 2 or head_p.shape[1] % 2:
        raise StxError("tanh_normal_kl: expected two float32 (M, 2A) head outputs of the same shape")
    out = torch.empty(head_p.shape[0], dtype=torch.float32, device=dev)
    _lib.check(_lib.load().stx_tanh_normal_kl(_p(head_p), _p(head_q), head_p.shape[0], head_p.shape[1] // 2, float(min_scale), _p(out), _stream()),
               "stx_tanh_normal_kl")
    return out


def _flat_f32(*ts: torch.Tensor, what: str) -> None:
    _need_cuda(*ts)
    if any(t.dtype != torch.float32 for t in ts) or len({t.numel() for t in ts}) != 1:
        raise StxError(f"{what}: expected float32 tensors of equal size")


def ppo_penalty_loss_value(pi_log_prob_t, b_pi_log_prob_t, gae_t, kl, beta: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """(-mean(ratio A) + beta mean(kl), mean(kl)) of ppo_penalty_loss (loss.py:35-47) from per-row KL values."""
    _flat_f32(pi_log_prob_t, b_pi_log_prob_t, gae_t, kl, what="ppo_penalty_loss_value")
    lib = _lib.load()
    out = torch.empty(2, dtype=torch.float32, device=gae_t.device)
    scratch = _zeros_scratch(("loss",), lib.stx_loss_scratch_bytes(), gae_t.device)
    _lib.check(lib.stx_ppo_penalty_loss(_p(pi_log_prob_t), _p(b_pi_log_prob_t), _p(gae_t), _p(kl), gae_t.numel(), float(beta), _p(out), _p(scratch),
                                        _stream()), "stx_ppo_penalty_loss")
    return out[0], out[1]


def dpo_loss_value(pi_log_prob_t, b_pi_log_prob_t, gae_t, alpha: float, beta: float) -> torch.Tensor:
    """-mean(ratio A - drift) of dpo_loss (loss.py:50-65)."""
    _flat_f32(pi_log_prob_t, b_pi_log_prob_t, gae_t, what="dpo_loss_value")
    lib = _lib.load()
    out = torch.empty(1, dtype=torch.float32, device=gae_t.device)
    scratch = _zeros_scratch(("loss",), lib.stx_loss_scratch_bytes(), gae_t.device)
    _lib.check(lib.stx_dpo_loss(_p(pi_log_prob_t), _p(b_pi_log_prob_t), _p(gae_t), gae_t.numel(), float(alpha), float(beta), _p(out), _p(scratch),
                                _stream()), "stx_dpo_loss")
    return out[0]


def ppo_penalty_head_grads(logits: torch.Tensor, idx: Optional[torch.Tensor], behaviour: torch.Tensor, action: torch.Tensor, logp_old: torch.Tensor,
                           adv: torch.Tensor, adv_stats: Optional[torch.Tensor], kl_coef: float, ent_coef: float,
                           d_logits: Optional[torch.Tensor] = None, metrics: Optional[torch.Tensor] = None, weight: float = 1.0, row0: int = 0,
                           scratch_key: str = "ppo_penalty_head") -> Tuple[torch.Tensor, torch.Tensor]:
    """The actor half of ff_ppo_penalty's _update_minibatch on logits (mb, A) computed elsewhere: row m pairs with batch row idx[m]
    (or row0 + m) of behaviour (B, A) / action / logp_old / adv.  Returns (d_logits, metrics[8]); slots 0, 1, 6 = actor_loss,
    entropy, kl_divergence."""
    who = "ppo_penalty_head_grads"
    d_logits, metrics, scratch = _head_grads_io(who, logits, idx, d_logits, metrics, 7, scratch_key, behaviour, action, logp_old, adv, adv_stats)
    mb, A = logits.shape
    if action.dtype != torch.int32:
        raise StxError(f"{who}: action must be int32")
    if behaviour.ndim != 2 or behaviour.shape[1] != A:
        raise StxError(f"{who}: behaviour must be (B, A) with A = logits.shape[1]")
    v = _variant(STX_PPO_KL_PENALTY, behaviour, kl_coef, 0.0, 0.0)
    _lib.check(_lib.load().stx_ppo_penalty_head_grads(_p(logits), _p(idx), int(row0), C.byref(v), _p(action), _p(logp_old), _p(adv), _p(adv_stats),
                                                      mb, A, float(ent_coef), _p(d_logits), _p(metrics), float(weight), _p(scratch), _stream()),
               "stx_ppo_penalty_head_grads")
    return d_logits, metrics


def ppo_variant_tanh_normal_head_grads(head_out: torch.Tensor, idx: Optional[torch.Tensor], kind: int, action: torch.Tensor, logp_old: torch.Tensor,
                                       adv: torch.Tensor, adv_stats: Optional[torch.Tensor], ent_coef: float, minimum: float, maximum: float,
                                       min_scale: float = 1e-3, behaviour: Optional[torch.Tensor] = None, kl_coef: float = 0.0,
                                       dpo_alpha: float = 2.0, dpo_beta: float = 0.6, seed: int = 0, offset: int = 0,
                                       dev_counter: Optional[torch.Tensor] = None, eps_in: Optional[torch.Tensor] = None,
                                       eps_out: Optional[torch.Tensor] = None, d_head_out: Optional[torch.Tensor] = None,
                                       metrics: Optional[torch.Tensor] = None, weight: float = 1.0, row0: int = 0,
                                       scratch_key: str = "ppo_variant_head") -> Tuple[torch.Tensor, torch.Tensor]:
    """The actor half of ff_ppo_penalty_continuous / ff_dpo_continuous (kind STX_PPO_KL_PENALTY / STX_PPO_DPO) on head outputs
    (mb, 2A) computed elsewhere; entropy noise as ppo_tanh_normal_head_grads.  Returns (d_head_out, metrics[8])."""
    who = "ppo_variant_tanh_normal_head_grads"
    d_head_out, metrics, scratch = _head_grads_io(who, head_out, idx, d_head_out, metrics, 7, scratch_key, action, logp_old, adv, adv_stats)
    mb, A2 = head_out.shape
    if action.ndim != 2 or action.shape[1] != A2 // 2 or (behaviour is not None and (behaviour.ndim != 2 or behaviour.shape[1] != A2)):
        raise StxError(f"{who}: action must be (B, A) and behaviour (B, 2A) with 2A = head_out.shape[1]")
    hd = _tanh_normal_ppo(action, minimum, maximum, min_scale, seed, offset, dev_counter, eps_in, eps_out)
    v = _variant(kind, behaviour, kl_coef, dpo_alpha, dpo_beta)
    _lib.check(_lib.load().stx_ppo_variant_tanh_normal_head_grads(_p(head_out), _p(idx), int(row0), C.byref(hd), C.byref(v), _p(logp_old), _p(adv),
                                                                  _p(adv_stats), mb, A2 // 2, float(ent_coef), _p(d_head_out), _p(metrics),
                                                                  float(weight), _p(scratch), _stream()), "stx_ppo_variant_tanh_normal_head_grads")
    return d_head_out, metrics


def ppo_penalty_minibatch_grads(actor: MlpSpec, critic: MlpSpec, param_arena: torch.Tensor, batch: PpoBatch, mb_off: int, mb: int,
                                behaviour: torch.Tensor, kl_coef: float, clip_eps: float, ent_coef: float, vf_coef: float, standardize: bool,
                                grad_arena: torch.Tensor, metrics: torch.Tensor, workspace: torch.Tensor, precision: int = STX_PREC_F32,
                                grad_weight: float = 1.0, overwrite: bool = False) -> None:
    """ppo_minibatch_grads with ff_ppo_penalty's actor loss (ff_ppo_penalty.py:149-210): behaviour (B, A) holds the behaviour
    policy's logits per batch row; clip_eps clips only the value loss."""
    who = "ppo_penalty_minibatch_grads"
    a, c, b, h = _minibatch_structs(who, actor, critic, param_arena, batch, grad_arena, metrics, workspace,
                                    (clip_eps, ent_coef, vf_coef, standardize, overwrite), obs_dtype=torch.float32,
                                    fp32_only="the KL-penalty loss", n_metrics=7)
    if behaviour.shape != (batch.action.numel(), actor.sizes[-1]):
        raise StxError(f"{who}: behaviour must be ({batch.action.numel()}, {actor.sizes[-1]})")
    v = _variant(STX_PPO_KL_PENALTY, behaviour, kl_coef, 0.0, 0.0)
    _lib.check(_lib.load().stx_ppo_penalty_minibatch_grads(C.byref(a), C.byref(c), C.byref(b), C.byref(v), int(mb_off), int(mb), C.byref(h),
                                                           float(grad_weight), _p(grad_arena), _p(metrics), int(precision), _p(workspace),
                                                           workspace.numel(), _stream()), "stx_ppo_penalty_minibatch_grads")


def ppo_variant_continuous_minibatch_grads(actor: MlpSpec, critic: MlpSpec, param_arena: torch.Tensor, batch: PpoBatch, mb_off: int, mb: int,
                                           kind: int, clip_eps: float, ent_coef: float, vf_coef: float, standardize: bool,
                                           grad_arena: torch.Tensor, metrics: torch.Tensor, workspace: torch.Tensor, minimum: float,
                                           maximum: float, min_scale: float = 1e-3, behaviour: Optional[torch.Tensor] = None,
                                           kl_coef: float = 0.0, dpo_alpha: float = 2.0, dpo_beta: float = 0.6, seed: int = 0,
                                           offset: int = 0, dev_counter: Optional[torch.Tensor] = None,
                                           eps_in: Optional[torch.Tensor] = None, eps_out: Optional[torch.Tensor] = None,
                                           precision: int = STX_PREC_F32, grad_weight: float = 1.0, overwrite: bool = False) -> None:
    """ppo_continuous_minibatch_grads with the actor loss of ff_ppo_penalty_continuous (kind STX_PPO_KL_PENALTY, behaviour (B, 2A)
    head outputs) or ff_dpo_continuous (kind STX_PPO_DPO); entropy noise as in ppo_continuous_minibatch_grads."""
    who = "ppo_variant_continuous_minibatch_grads"
    a, c, b, h = _minibatch_structs(who, actor, critic, param_arena, batch, grad_arena, metrics, workspace,
                                    (clip_eps, ent_coef, vf_coef, standardize, overwrite), obs_dtype=torch.float32,
                                    fp32_only="the KL-penalty and DPO losses", n_metrics=7, categorical=False)
    if behaviour is not None and behaviour.shape != (b.B, actor.sizes[-1]):
        raise StxError(f"{who}: behaviour must be ({b.B}, {actor.sizes[-1]})")
    hd = _tanh_normal_ppo(batch.action, minimum, maximum, min_scale, seed, offset, dev_counter, eps_in, eps_out)
    v = _variant(kind, behaviour, kl_coef, dpo_alpha, dpo_beta)
    _lib.check(_lib.load().stx_ppo_variant_continuous_minibatch_grads(C.byref(a), C.byref(c), C.byref(b), C.byref(hd), C.byref(v), int(mb_off),
                                                                      int(mb), C.byref(h), float(grad_weight), _p(grad_arena), _p(metrics),
                                                                      int(precision), _p(workspace), workspace.numel(), _stream()),
               "stx_ppo_variant_continuous_minibatch_grads")


def sac_actor_seed(q1, q2, log_prob, log_alpha, dq1, dq2, metrics=None, weight: float = 1.0) -> None:
    _need_cuda(q1, q2, log_prob, log_alpha, dq1, dq2, metrics)
    _lib.check(_lib.load().stx_sac_actor_seed(_p(q1), _p(q2), _p(log_prob), _p(log_alpha), q1.numel(), _p(dq1), _p(dq2), _p(metrics), float(weight),
                                              _stream()), "stx_sac_actor_seed")


def sac_q_loss(q1, q2, next_q1, next_q2, next_log_prob, reward, done, log_alpha, gamma: float, dq1, dq2, metrics=None, weight: float = 1.0) -> None:
    _need_cuda(q1, q2, next_q1, next_q2, next_log_prob, reward, done, log_alpha, dq1, dq2, metrics)
    d8 = done.view(torch.uint8) if done.dtype == torch.bool else done
    _lib.check(_lib.load().stx_sac_q_loss(_p(q1), _p(q2), _p(next_q1), _p(next_q2), _p(next_log_prob), _p(reward), _p(d8), _p(log_alpha), float(gamma),
                                          q1.numel(), _p(dq1), _p(dq2), _p(metrics), float(weight), _stream()), "stx_sac_q_loss")


def sac_alpha_grad(log_prob, log_alpha, target_entropy: float, autotune: bool, grad, grad_weight: float = 1.0, overwrite: bool = True,
                   metrics=None, weight: float = 1.0) -> None:
    _need_cuda(log_prob, log_alpha, grad, metrics)
    _lib.check(_lib.load().stx_sac_alpha_grad(_p(log_prob), _p(log_alpha), float(target_entropy), log_prob.numel(), int(bool(autotune)), _p(grad),
                                              float(grad_weight), int(bool(overwrite)), _p(metrics), float(weight), _stream()), "stx_sac_alpha_grad")


def polyak_update(target: torch.Tensor, online: torch.Tensor, tau: float) -> None:
    _need_cuda(target, online)
    _lib.check(_lib.load().stx_polyak_update(_p(target), _p(online), target.numel(), float(tau), _stream()), "stx_polyak_update")


def uniform_indices(M: int, range_dev: torch.Tensor, seed: int, offset: int = 0, dev_counter: Optional[torch.Tensor] = None,
                    out: Optional[torch.Tensor] = None) -> torch.Tensor:
    dev = _need_cuda(range_dev, dev_counter, out)
    if range_dev.dtype != torch.int64:
        raise StxError("uniform_indices: range must be an int64 device scalar")
    if out is None:
        out = torch.empty(int(M), dtype=torch.int32, device=dev)
    _lib.check(_lib.load().stx_uniform_indices(_p(out), int(M), int(seed) & (2**64 - 1), int(offset), _p(dev_counter), _p(range_dev), _stream()),
               "stx_uniform_indices")
    return out


def gather_rows(src: torch.Tensor, idx: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out[r, :C] = src[idx[r]] for float32 row-major src (N, C) / (N,), uint8 (N,); `out` may be a column block."""
    _need_cuda(src, idx)
    M = int(idx.numel())
    if src.dtype == torch.uint8 or src.dtype == torch.bool:
        s8, o8 = (src.view(torch.uint8) if src.dtype == torch.bool else src), (out.view(torch.uint8) if out.dtype == torch.bool else out)
        _lib.check(_lib.load().stx_gather_u8(_p(s8), _p(idx), M, _p(o8), _stream()), "stx_gather_u8")
        return out
    Cn = 1 if src.ndim == 1 else int(src.shape[1])
    ld = 1 if out.ndim == 1 else out.stride(0)
    _lib.check(_lib.load().stx_gather_rows_f32(_p(src), _p(idx), M, Cn, _p(out), int(ld), _stream()), "stx_gather_rows_f32")
    return out


class ReplayRing:
    """Device storage + StxReplay descriptor of the transition ring buffer (stx_replay_add / stx_replay_sample)."""

    def __init__(self, capacity: int, obs_dim: int, act_dim: int, device):
        self.capacity, self.obs_dim, self.act_dim = int(capacity), int(obs_dim), int(act_dim)
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.obs, self.next_obs = z(self.capacity, self.obs_dim), z(self.capacity, self.obs_dim)
        self.action, self.reward, self.done = z(self.capacity, self.act_dim), z(self.capacity), z(self.capacity, dt=torch.uint8)
        self.state = z(2, dt=torch.int64)   # {write position, valid items}
        self.c = _lib.StxReplay(_p(self.obs), _p(self.action), _p(self.reward), _p(self.done), _p(self.next_obs), _p(self.state), self.capacity,
                                self.obs_dim, self.act_dim)


def replay_add(rb: ReplayRing, obs, action, reward, done, next_obs) -> None:
    """Append the rows of a (T, E, ...) / (n, ...) batch of transitions (contiguous fp32; done uint8 / bool)."""
    _need_cuda(obs, action, reward, done, next_obs)
    n = int(reward.numel())
    for t, cols, name in ((obs, rb.obs_dim, "obs"), (next_obs, rb.obs_dim, "next_obs"), (action, rb.act_dim, "action"), (reward, 1, "reward")):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() != n * cols:
            raise StxError(f"replay_add: {name} must be contiguous float32 with {n} x {cols} elements")
    d8 = done.view(torch.uint8) if done.dtype == torch.bool else done
    if d8.dtype != torch.uint8 or not d8.is_contiguous() or d8.numel() != n:
        raise StxError("replay_add: done must be contiguous uint8 / bool")
    _lib.check(_lib.load().stx_replay_add(C.byref(rb.c), _p(obs), _p(action), _p(reward), _p(d8), _p(next_obs), n, _stream()), "stx_replay_add")


def replay_sample(rb: ReplayRing, M: int, seed: int, xq_old: torch.Tensor, reward: torch.Tensor, done: torch.Tensor, xq_new=None, xq_next=None,
                  offset: int = 0, dev_counter: Optional[torch.Tensor] = None, idx_in: Optional[torch.Tensor] = None,
                  idx_out: Optional[torch.Tensor] = None) -> None:
    """One launch: draw M indices (or take idx_in) and write (obs | action), (obs | .), (next_obs | .), reward, done."""
    _need_cuda(xq_old, xq_new, xq_next, reward, done, dev_counter, idx_in, idx_out)
    ld = xq_old.stride(0)
    for t in (xq_old, xq_new, xq_next):
        if t is not None and (t.dtype != torch.float32 or t.shape[0] != M or t.stride(0) != ld or t.stride(1) != 1):
            raise StxError("replay_sample: xq_* must be float32 (M, >= obs_dim + act_dim) with one common leading dimension")
    _lib.check(_lib.load().stx_replay_sample(C.byref(rb.c), int(M), int(seed) & (2**64 - 1), int(offset), _p(dev_counter), _p(idx_in), _p(xq_old),
                                             _p(xq_new), _p(xq_next), int(ld), _p(reward), _p(done), _p(idx_out), _stream()), "stx_replay_sample")


class DiscreteReplayRing:
    """Device storage + StxReplayDiscrete descriptor of the DQN family's transition ring (one int32 action per row;
    stx_replay_add_discrete / stx_replay_sample_discrete)."""

    def __init__(self, capacity: int, obs_dim: int, device):
        self.capacity, self.obs_dim = int(capacity), int(obs_dim)
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.obs, self.next_obs = z(self.capacity, self.obs_dim), z(self.capacity, self.obs_dim)
        self.action, self.reward, self.done = z(self.capacity, dt=torch.int32), z(self.capacity), z(self.capacity, dt=torch.uint8)
        self.state = z(2, dt=torch.int64)   # {write position, valid items}
        self.c = _lib.StxReplayDiscrete(_p(self.obs), _p(self.action), _p(self.reward), _p(self.done), _p(self.next_obs), _p(self.state),
                                        self.capacity, self.obs_dim, 0)


def _u8(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.uint8) if t.dtype == torch.bool else t


def replay_add_discrete(rb: DiscreteReplayRing, obs, action, reward, done, next_obs) -> None:
    """Append the rows of a (T, E, ...) / (n, ...) batch of transitions (contiguous; obs / next_obs / reward fp32, action int32,
    done uint8 / bool) in time-major order."""
    _need_cuda(obs, action, reward, done, next_obs)
    n = int(reward.numel())
    for t, cols, dt, name in ((obs, rb.obs_dim, torch.float32, "obs"), (next_obs, rb.obs_dim, torch.float32, "next_obs"),
                              (reward, 1, torch.float32, "reward"), (action, 1, torch.int32, "action"), (_u8(done), 1, torch.uint8, "done")):
        if t.dtype != dt or not t.is_contiguous() or t.numel() != n * cols:
            raise StxError(f"replay_add_discrete: {name} must be contiguous {dt} with {n} x {cols} elements")
    _lib.check(_lib.load().stx_replay_add_discrete(C.byref(rb.c), _p(obs), _p(action), _p(reward), _p(_u8(done)), _p(next_obs), n, _stream()),
               "stx_replay_add_discrete")


def replay_sample_discrete(rb: DiscreteReplayRing, M: int, seed: int, obs: torch.Tensor, next_obs: torch.Tensor, action: torch.Tensor,
                           reward: torch.Tensor, done: torch.Tensor, offset: int = 0, dev_counter: Optional[torch.Tensor] = None,
                           idx_in: Optional[torch.Tensor] = None, idx_out: Optional[torch.Tensor] = None) -> None:
    """One launch: draw M indices (or take idx_in) and write obs, next_obs (M, obs_dim), action, reward, done (M)."""
    _need_cuda(obs, next_obs, action, reward, done, dev_counter, idx_in, idx_out)
    M = int(M)
    for t, cols, dt, name in ((obs, rb.obs_dim, torch.float32, "obs"), (next_obs, rb.obs_dim, torch.float32, "next_obs"),
                              (reward, 1, torch.float32, "reward"), (action, 1, torch.int32, "action"), (_u8(done), 1, torch.uint8, "done")):
        if t.dtype != dt or not t.is_contiguous() or t.numel() != M * cols:
            raise StxError(f"replay_sample_discrete: {name} must be contiguous {dt} with {M} x {cols} elements")
    for t, name in ((idx_in, "idx_in"), (idx_out, "idx_out")):
        if t is not None and (t.dtype != torch.int32 or not t.is_contiguous() or t.numel() != M):
            raise StxError(f"replay_sample_discrete: {name} must be contiguous int32 (M)")
    _lib.check(_lib.load().stx_replay_sample_discrete(C.byref(rb.c), M, int(seed) & (2**64 - 1), int(offset), _p(dev_counter), _p(idx_in), _p(obs),
                                                      _p(next_obs), _p(action), _p(reward), _p(_u8(done)), _p(idx_out), _stream()),
               "stx_replay_sample_discrete")


# ------------------------------------------------------------------------------------------------
# recurrent PPO building blocks (stoix/networks/base.py:124-222, stoix/systems/ppo/anakin/rec_ppo.py)
# ------------------------------------------------------------------------------------------------


def gru_workspace(T: int, E: int, H: int, device) -> torch.Tensor:
    return torch.zeros(int(_lib.load().stx_gru_workspace_bytes(int(T), int(E), int(H))), dtype=torch.uint8, device=device)


def gru_sequence_forward(gi: torch.Tensor, reset: torch.Tensor, h0: torch.Tensor, w_h: torch.Tensor, b_hn: torch.Tensor, ws: torch.Tensor,
                         out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """ScannedRNN(gru) over (T, E): gi (T, E, 3H) input projections, reset (T, E) uint8 / bool, h0 (E, H) -> h_seq (T, E, H)."""
    dev = _need_cuda(gi, reset, h0, w_h, b_hn, ws, out)
    T, E, H3 = gi.shape
    H = H3 // 3
    r8 = reset.view(torch.uint8) if reset.dtype == torch.bool else reset
    for t_, shape, name in ((gi, (T, E, 3 * H), "gi"), (h0, (E, H), "h0"), (w_h, (H, 3 * H), "w_h"), (b_hn, (H,), "b_hn")):
        if t_.dtype != torch.float32 or tuple(t_.shape) != shape or not t_.is_contiguous():
            raise StxError(f"gru_sequence_forward: {name} must be contiguous float32 {shape}")
    if r8.dtype != torch.uint8 or tuple(r8.shape) != (T, E) or not r8.is_contiguous():
        raise StxError("gru_sequence_forward: reset must be contiguous uint8 / bool (T, E)")
    if out is None:
        out = torch.empty(T, E, H, dtype=torch.float32, device=dev)
    _lib.check(_lib.load().stx_gru_sequence_forward(_p(gi), _p(r8), _p(h0), _p(w_h), _p(b_hn), T, E, H, _p(out), _p(ws), ws.numel(), _stream()),
               "stx_gru_sequence_forward")
    return out


def gru_sequence_backward(d_h_seq: torch.Tensor, reset: torch.Tensor, w_h: torch.Tensor, ws: torch.Tensor, d_gi: torch.Tensor,
                          d_w_h: Optional[torch.Tensor] = None, d_b_hn: Optional[torch.Tensor] = None, grad_weight: float = 1.0,
                          overwrite: bool = True, d_h0: Optional[torch.Tensor] = None) -> None:
    _need_cuda(d_h_seq, reset, w_h, ws, d_gi, d_w_h, d_b_hn, d_h0)
    T, E, H = d_h_seq.shape
    r8 = reset.view(torch.uint8) if reset.dtype == torch.bool else reset
    if d_h_seq.dtype != torch.float32 or not d_h_seq.is_contiguous() or d_gi.dtype != torch.float32 or d_gi.numel() != T * E * 3 * H:
        raise StxError("gru_sequence_backward: d_h_seq (T, E, H) / d_gi (T, E, 3H) must be contiguous float32")
    _lib.check(_lib.load().stx_gru_sequence_backward(_p(d_h_seq), _p(r8), _p(w_h), T, E, H, _p(ws), ws.numel(), _p(d_gi), _p(d_w_h), _p(d_b_hn),
                                                     float(grad_weight), int(bool(overwrite)), _p(d_h0), _stream()), "stx_gru_sequence_backward")


def ppo_head_grads(logits: Optional[torch.Tensor], value: Optional[torch.Tensor], idx: Optional[torch.Tensor], action, logp_old, v_old, adv, targets,
                   adv_stats, clip_eps: float, ent_coef: float, vf_coef: float, d_logits, d_value, metrics: torch.Tensor, weight: float = 1.0,
                   row0: int = 0, scratch_key: str = "ppo_head") -> None:
    """PPO losses and their gradients w.r.t. network outputs computed elsewhere (see stx_ppo_head_grads)."""
    dev = _need_cuda(logits, value, idx, action, logp_old, v_old, adv, targets, adv_stats, d_logits, d_value, metrics)
    mb = int(logits.shape[0]) if logits is not None else int(value.numel())
    A = int(logits.shape[1]) if logits is not None else 0
    lib = _lib.load()
    scratch = _zeros_scratch((scratch_key,), lib.stx_ppo_head_scratch_bytes(mb), dev)   # one per concurrently running stream
    _lib.check(lib.stx_ppo_head_grads(_p(logits), _p(value), _p(idx), int(row0), _p(action), _p(logp_old), _p(v_old), _p(adv), _p(targets), _p(adv_stats),
                                      mb, A, float(clip_eps), float(ent_coef), float(vf_coef), _p(d_logits), _p(d_value), _p(metrics), float(weight),
                                      _p(scratch), _stream()), "stx_ppo_head_grads")


def lstm_workspace(T: int, E: int, H: int, device) -> torch.Tensor:
    return torch.zeros(int(_lib.load().stx_lstm_workspace_bytes(int(T), int(E), int(H))), dtype=torch.uint8, device=device)


def lstm_sequence_forward(gi: torch.Tensor, reset: torch.Tensor, carry0: torch.Tensor, w_h: torch.Tensor, ws: torch.Tensor,
                          out: Optional[torch.Tensor] = None, carry_last: Optional[torch.Tensor] = None) -> torch.Tensor:
    """ScannedRNN(lstm) over (T, E): gi (T, E, 4H), carry0 (E, 2H) = (c | h), w_h (H, 4H) -> h_seq (T, E, H); carry_last (E, 2H) optional."""
    dev = _need_cuda(gi, reset, carry0, w_h, ws, out, carry_last)
    T, E, H4 = gi.shape
    H = H4 // 4
    r8 = reset.view(torch.uint8) if reset.dtype == torch.bool else reset
    for t_, shape, name in ((gi, (T, E, 4 * H), "gi"), (carry0, (E, 2 * H), "carry0"), (w_h, (H, 4 * H), "w_h")):
        if t_.dtype != torch.float32 or tuple(t_.shape) != shape or not t_.is_contiguous():
            raise StxError(f"lstm_sequence_forward: {name} must be contiguous float32 {shape}")
    if r8.dtype != torch.uint8 or tuple(r8.shape) != (T, E) or not r8.is_contiguous():
        raise StxError("lstm_sequence_forward: reset must be contiguous uint8 / bool (T, E)")
    if out is None:
        out = torch.empty(T, E, H, dtype=torch.float32, device=dev)
    _lib.check(_lib.load().stx_lstm_sequence_forward(_p(gi), _p(r8), _p(carry0), _p(w_h), T, E, H, _p(out), _p(carry_last), _p(ws), ws.numel(), _stream()),
               "stx_lstm_sequence_forward")
    return out


def lstm_sequence_backward(d_h_seq: torch.Tensor, reset: torch.Tensor, w_h: torch.Tensor, ws: torch.Tensor, d_gi: torch.Tensor,
                           d_w_h: Optional[torch.Tensor] = None, grad_weight: float = 1.0, overwrite: bool = True,
                           d_carry0: Optional[torch.Tensor] = None) -> None:
    _need_cuda(d_h_seq, reset, w_h, ws, d_gi, d_w_h, d_carry0)
    T, E, H = d_h_seq.shape
    r8 = reset.view(torch.uint8) if reset.dtype == torch.bool else reset
    if d_h_seq.dtype != torch.float32 or not d_h_seq.is_contiguous() or d_gi.dtype != torch.float32 or d_gi.numel() != T * E * 4 * H:
        raise StxError("lstm_sequence_backward: d_h_seq (T, E, H) / d_gi (T, E, 4H) must be contiguous float32")
    _lib.check(_lib.load().stx_lstm_sequence_backward(_p(d_h_seq), _p(r8), _p(w_h), T, E, H, _p(ws), ws.numel(), _p(d_gi), _p(d_w_h), float(grad_weight),
                                                      int(bool(overwrite)), _p(d_carry0), _stream()), "stx_lstm_sequence_backward")


# ------------------------------------------------------------------------------------------------
# PQN: epsilon-greedy head, Q(lambda) targets, Q loss (stoix/systems/q_learning/ff_pqn.py)
# ------------------------------------------------------------------------------------------------


def epsilon_schedule_struct(init_value: float, end_value: float, transition_steps: float, steps_per_update: int = 1,
                            decay: bool = True) -> _lib.StxEpsilonSchedule:
    """The device-evaluated epsilon schedule of stx_epsilon_greedy; decay=False is the constant schedule at end_value."""
    return _lib.StxEpsilonSchedule(float(init_value), float(end_value), float(transition_steps), int(steps_per_update), int(bool(decay)), 0)


def epsilon_greedy(q: torch.Tensor, sched: _lib.StxEpsilonSchedule, seed: int = 0, offset: int = 0, dev_counter: Optional[torch.Tensor] = None,
                   count: Optional[torch.Tensor] = None, mode: bool = False, out: Optional[torch.Tensor] = None,
                   epsilon_out: Optional[torch.Tensor] = None, update_no_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """distrax.EpsilonGreedy(q, epsilon).sample (mode=False) or .mode() on q (E, A) float32; epsilon from `sched` at the optimiser
    count word `count` (int32, nullable: count 0).  Returns the int32 actions (E)."""
    dev = _need_cuda(q, dev_counter, count, out, epsilon_out, update_no_out)
    if q.dtype != torch.float32 or q.ndim != 2:
        raise StxError("epsilon_greedy: q must be float32 (E, A)")
    if count is not None and count.dtype != torch.int32:
        raise StxError("epsilon_greedy: count must be an int32 device word")
    E, A = q.shape
    if out is None:
        out = torch.empty(E, dtype=torch.int32, device=dev)
    if out.dtype != torch.int32 or out.numel() != E:
        raise StxError("epsilon_greedy: out must be int32 (E)")
    for name, t, dt in (("epsilon_out", epsilon_out, torch.float32), ("update_no_out", update_no_out, torch.int32)):
        if t is not None and (t.dtype != dt or t.numel() != E):
            raise StxError(f"epsilon_greedy: {name} must be {dt} (E)")
    _lib.check(_lib.load().stx_epsilon_greedy(_p(q), E, A, int(bool(mode)), int(seed) & (2**64 - 1), int(offset), _p(dev_counter), _p(count),
                                              C.byref(sched), _p(out), _p(epsilon_out), _p(update_no_out), _stream()), "stx_epsilon_greedy")
    return out


def q_lambda(q_t: torch.Tensor, reward: torch.Tensor, done: torch.Tensor, truncated: torch.Tensor, gamma: float, q_lambda_: float,
             out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Q(lambda) targets (T, E) of a time-major rollout: q_t (T, E, A) the successor rows' Q values, discount gamma (1 - (done | truncated))."""
    dev = _need_cuda(q_t, reward, done, truncated, out)
    T, E = reward.shape
    if q_t.dtype != torch.float32 or q_t.ndim != 3 or tuple(q_t.shape[:2]) != (T, E) or reward.dtype != torch.float32:
        raise StxError("q_lambda: q_t must be float32 (T, E, A) and reward float32 (T, E)")
    done8 = done.view(torch.uint8) if done.dtype == torch.bool else done
    trunc8 = truncated.view(torch.uint8) if truncated.dtype == torch.bool else truncated
    if done8.dtype != torch.uint8 or trunc8.dtype != torch.uint8 or done8.shape != (T, E) or trunc8.shape != (T, E):
        raise StxError("q_lambda: done / truncated must be bool or uint8 (T, E)")
    if out is None:
        out = torch.empty((T, E), dtype=torch.float32, device=dev)
    _lib.check(_lib.load().stx_q_lambda_f32(_p(q_t), int(q_t.shape[2]), _p(reward), _p(done8), _p(trunc8), T, E, float(gamma), float(q_lambda_),
                                            _p(out), _stream()), "stx_q_lambda_f32")
    return out


def lambda_returns(r_t: torch.Tensor, discount_t: torch.Tensor, v_t: torch.Tensor, lambda_) -> torch.Tensor:
    """Time-major lambda returns (T, E) with float discounts; v_t (T, E) or (T, E, A) (then max over A: Q(lambda)); lambda_ a scalar or a
    (T, E) tensor."""
    dev = _need_cuda(r_t, discount_t, v_t)
    T, E = r_t.shape
    A = 1 if v_t.ndim == 2 else int(v_t.shape[2])
    if tuple(v_t.shape[:2]) != (T, E) or discount_t.shape != (T, E) or any(x.dtype != torch.float32 for x in (r_t, discount_t, v_t)):
        raise StxError("lambda_returns: r_t, discount_t float32 (T, E); v_t float32 (T, E) or (T, E, A)")
    lam_t, lam = None, 0.0
    if isinstance(lambda_, torch.Tensor) and lambda_.ndim > 0:
        lam_t = lambda_.to(torch.float32).expand(T, E).contiguous()
        _need_cuda(lam_t)
    else:
        lam = float(lambda_)
    out = torch.empty((T, E), dtype=torch.float32, device=dev)
    _lib.check(_lib.load().stx_lambda_returns_f32(_p(r_t), _p(discount_t), _p(v_t), A, _p(lam_t), lam, T, E, _p(out), _stream()),
               "stx_lambda_returns_f32")
    return out


def q_loss_grads(q: torch.Tensor, idx: Optional[torch.Tensor], action: torch.Tensor, targets: torch.Tensor, huber_delta: float, d_q: torch.Tensor,
                 metrics: torch.Tensor, weight: float = 1.0, row0: int = 0, scratch_key: str = "q_loss") -> None:
    """_q_loss_fn (ff_pqn.py:139-162) on Q rows computed elsewhere: d mean(loss) / d q into d_q (mb, A), metrics[0] += weight * q_loss.
    Row m pairs with batch row idx[m] (or row0 + m) of action / targets."""
    dev = _need_cuda(q, idx, action, targets, d_q, metrics)
    if q.dtype != torch.float32 or q.ndim != 2 or d_q.dtype != torch.float32 or d_q.shape != q.shape:
        raise StxError("q_loss_grads: q and d_q must be float32 (mb, A)")
    if action.dtype != torch.int32 or targets.dtype != torch.float32 or (idx is not None and idx.dtype != torch.int32):
        raise StxError("q_loss_grads: action / idx int32, targets float32")
    mb, A = q.shape
    if idx is not None and idx.numel() != mb:
        raise StxError("q_loss_grads: idx must hold one row index per q row")
    lib = _lib.load()
    scratch = _zeros_scratch((scratch_key,), lib.stx_ppo_head_scratch_bytes(mb), dev)
    _lib.check(lib.stx_q_loss_grads(_p(q), _p(idx), int(row0), _p(action), _p(targets), mb, A, float(huber_delta), _p(d_q), _p(metrics),
                                    float(weight), _p(scratch), _stream()), "stx_q_loss_grads")


# ------------------------------------------------------------------------------------------------
# DQN family: one-step Q-learning losses (stoix/utils/loss.py:106-146, 190-223; stoix/systems/q_learning/ff_dqn_reg.py:165-176)
# ------------------------------------------------------------------------------------------------

Q_RULES = {"q_learning": 0, "double_q_learning": 1, "munchausen_q_learning": 2, "q_learning_reg": 3}   # STX_Q_* of stx.h


def q_td_hyper(gamma: float = 0.99, max_abs_reward: float = float("inf"), huber_delta: float = 0.0, entropy_temperature: float = 0.03,
               munchausen_coefficient: float = 0.9, clip_value_min: float = -1e3, regularizer_coeff: float = 0.0) -> _lib.StxQTdHyper:
    return _lib.StxQTdHyper(float(gamma), float(max_abs_reward), float(huber_delta), float(entropy_temperature), float(munchausen_coefficient),
                            float(clip_value_min), float(regularizer_coeff), 0)


def q_td_loss_grads(rule: str, q_tm1: torch.Tensor, q_t: torch.Tensor, action: torch.Tensor, reward: torch.Tensor, hyper: _lib.StxQTdHyper,
                    d_q: torch.Tensor, metrics: torch.Tensor, done: Optional[torch.Tensor] = None, discount: Optional[torch.Tensor] = None,
                    q_aux: Optional[torch.Tensor] = None, weight: float = 1.0, scratch_key: str = "q_td_loss") -> None:
    """The loss of `rule` (a key of Q_RULES) on Q rows computed elsewhere, all (M, A) contiguous fp32: d mean(loss) / d q_tm1 into d_q,
    metrics[0] += weight * loss.  q_aux: the DDQN selector Q(online, next_obs) / the MDQN Q(target, obs).  The discount is
    (1 - done) gamma from `done` (uint8 / bool), or `discount` (M) fp32 given directly."""
    dev = _need_cuda(q_tm1, q_t, q_aux, action, reward, done, discount, d_q, metrics)
    if rule not in Q_RULES:
        raise StxError(f"q_td_loss_grads: rule {rule!r} is not one of {sorted(Q_RULES)}")
    if q_tm1.dtype != torch.float32 or q_tm1.ndim != 2 or not q_tm1.is_contiguous():
        raise StxError("q_td_loss_grads: q_tm1 must be contiguous float32 (M, A)")
    M, A = q_tm1.shape
    for t, name in ((q_t, "q_t"), (q_aux, "q_aux"), (d_q, "d_q")):
        if t is not None and (t.dtype != torch.float32 or tuple(t.shape) != (M, A) or not t.is_contiguous()):
            raise StxError(f"q_td_loss_grads: {name} must be contiguous float32 ({M}, {A})")
    for t, dt, name in ((action, torch.int32, "action"), (reward, torch.float32, "reward"), (discount, torch.float32, "discount"),
                        (None if done is None else _u8(done), torch.uint8, "done")):
        if t is not None and (t.dtype != dt or t.numel() != M or not t.is_contiguous()):
            raise StxError(f"q_td_loss_grads: {name} must be contiguous {dt} (M)")
    lib = _lib.load()
    scratch = _zeros_scratch((scratch_key,), lib.stx_ppo_head_scratch_bytes(M), dev)
    _lib.check(lib.stx_q_td_loss_grads(Q_RULES[rule], _p(q_tm1), _p(q_t), _p(q_aux), _p(action), _p(reward), _p(None if done is None else _u8(done)),
                                       _p(discount), M, A, C.byref(hyper), _p(d_q), _p(metrics), float(weight), _p(scratch), _stream()),
               "stx_q_td_loss_grads")
