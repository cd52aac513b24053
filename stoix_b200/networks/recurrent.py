"""ScannedRNN, RecurrentActor, RecurrentCritic -- the faces of stoix/networks/base.py:124-222 over the GRU sequence kernels.

One flat fp32 arena per network: [pre-torso Dense layers | W_i (P x 3H, columns r|z|n) | b_i (3H) | W_h (H x 3H) | b_hn (H) |
post-torso Dense layers | head].  `spec_pre` = MLP(D, *pre_sizes, 3H) -- the input projections of the cell are its "head"
(Dense with bias, no activation) -- and `spec_post` = MLP(H, *post_sizes, out).  The parameter tree exposes flax's names
(params / pre_torso / ScannedRNN_0 / GRUCell_0 / {ir, iz, in, hr, hz, hn} / post_torso / head) as views into the arena.

With a DuelingQNetwork head (R2D2), `spec_post` = MLP(H, *post_sizes, *branch_sizes, A) runs the post-torso and the advantage
branch (MLPTorso_1, activate_final=False: its last Dense has no bias and is followed by a LayerNorm, MlpSpec.ln_final) as one chain,
and the value branch (MLPTorso_0) follows in the arena as `spec_value` = MLP(post_out, *branch_sizes, 1), in the same form.  That
branch ends in a LayerNorm over one element, whose output is exactly its bias: the network computes Q = v + (adv - mean adv) with
v = that bias (stx_dueling_q) and never runs the rest of the branch, whose gradient is exactly zero."""
from __future__ import annotations

from typing import Any, Dict, Optional, Tuple

import numpy as np
import torch

from stoix_b200 import ops
from .base import ParamTree, _orthogonal
from .inputs import ArrayInput


class ScannedRNN:
    """networks/base.py:124-159: description of the recurrent layer (the arithmetic is stx_{gru,lstm}_sequence_forward / _backward,
    run through RecLayout.sequence_forward / sequence_backward)."""

    def __init__(self, hidden_state_dim: int, cell_type: str = "gru"):
        cell_type = {"optimised_lstm": "lstm"}.get(str(cell_type), str(cell_type))   # OptimizedLSTMCell: same function as LSTMCell
        if cell_type not in ("gru", "lstm"):
            raise NotImplementedError(f"cell_type '{cell_type}' is not built: the CUDA sequence kernels implement flax's GRUCell "
                                      "(configs/network/rnn.yaml default) and LSTMCell")
        self.hidden_state_dim, self.cell_type = int(hidden_state_dim), cell_type
        self.gates = 3 if cell_type == "gru" else 4
        self.state_dim = self.hidden_state_dim * (1 if cell_type == "gru" else 2)   # lstm: the carry (c, h) as ONE tensor (c | h)

    def initialize_carry(self, batch_size: int, device=None) -> torch.Tensor:
        """Zeros, like every flax cell's default carry initialiser (base.py:154-159); lstm: (batch, 2H) = (c | h)."""
        return torch.zeros(int(batch_size), self.state_dim, dtype=torch.float32, device=device)


class RecLayout:
    """Offsets of the blocks of one recurrent network inside its flat arena."""

    def __init__(self, obs_dim: int, pre_sizes, H: int, post_sizes, out_dim: int, activation_pre: str, ln_pre: bool, activation_post: str, ln_post: bool,
                 cell_type: str = "gru", branch_sizes=None):
        self.H, self.cell_type = int(H), cell_type
        self.G = 3 if cell_type == "gru" else 4                   # gate blocks of W_i / W_h
        self.S = self.H if cell_type == "gru" else 2 * self.H     # carry width
        self.spec_pre = ops.MlpSpec((int(obs_dim), *[int(s) for s in pre_sizes], self.G * self.H), activation=activation_pre, use_layer_norm=ln_pre)
        self.dueling = branch_sizes is not None
        self.n_post_torso = len(post_sizes)
        branch = [int(s) for s in branch_sizes] if self.dueling else []
        self.spec_post = ops.MlpSpec((self.H, *[int(s) for s in post_sizes], *branch, int(out_dim)), activation=activation_post, use_layer_norm=ln_post,
                                     ln_final=self.dueling)
        self.off_pre = 0
        self.off_wh = self.spec_pre.param_count
        self.off_bhn = self.off_wh + self.H * self.G * self.H
        self.off_post = self.off_bhn + (self.H if cell_type == "gru" else 0)   # lstm: the hidden biases are the bias of W_i
        self.off_value = self.off_post + self.spec_post.param_count
        self.spec_value = None
        if self.dueling:
            post_out = int(post_sizes[-1]) if len(post_sizes) else self.H
            self.spec_value = ops.MlpSpec((post_out, *branch, 1), activation=activation_post, use_layer_norm=True, ln_final=True)
        self.param_count = self.off_value + (self.spec_value.param_count if self.dueling else 0)

    def value_bias(self, flat: torch.Tensor) -> torch.Tensor:
        """The (1,) view of the value branch's final LayerNorm bias: the value of every state."""
        sl = self.spec_value.ln_bias_slices()[-1]
        return flat[self.off_value + sl.start: self.off_value + sl.stop]

    def blocks(self, flat: torch.Tensor):
        """(pre arena, W_h (H, G*H), b_hn (H; empty for lstm), post arena) views."""
        H = self.H
        return (flat[self.off_pre: self.off_wh], flat[self.off_wh: self.off_bhn].view(H, self.G * H), flat[self.off_bhn: self.off_post],
                flat[self.off_post: self.param_count])

    def sequence_workspace(self, T: int, E: int, device) -> torch.Tensor:
        """Workspace of one (T, E) sequence of this cell: what its forward saves for the backward."""
        return (ops.lstm_workspace if self.cell_type == "lstm" else ops.gru_workspace)(T, E, self.H, device)

    def sequence_forward(self, p_flat: torch.Tensor, gi: torch.Tensor, reset: torch.Tensor, carry0: torch.Tensor, ws: torch.Tensor,
                         out: Optional[torch.Tensor] = None, carry_last: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The recurrence over gi (T, E, G*H) from carry0 (E, S) with the W_h (and b_hn) of the arena p_flat -> h_seq (T, E, H), into
        `out` when given.  carry_last (E, S), when given, gets the carry after the last step."""
        _, w_h, b_hn, _ = self.blocks(p_flat)
        if self.cell_type == "lstm":
            return ops.lstm_sequence_forward(gi, reset, carry0, w_h, ws, out=out, carry_last=carry_last)
        h_seq = ops.gru_sequence_forward(gi, reset, carry0, w_h, b_hn, ws, out=out)
        if carry_last is not None:   # the GRU's carry is its last output
            carry_last.copy_(h_seq[-1])
        return h_seq

    def sequence_backward(self, p_flat: torch.Tensor, g_flat: torch.Tensor, d_h: torch.Tensor, reset: torch.Tensor, ws: torch.Tensor, d_gi: torch.Tensor,
                          weight: float, overwrite: bool, d_carry0: Optional[torch.Tensor] = None) -> None:
        """Backward through time of the last sequence_forward on `ws`: d_h (T, E, H) -> d_gi (T, E, G*H), and weight * d(W_h) (and
        d(b_hn)) into the gradient arena g_flat (overwritten or added); d_carry0 (E, S) when given."""
        _, w_h, _, _ = self.blocks(p_flat)
        _, g_wh, g_bhn, _ = self.blocks(g_flat)
        if self.cell_type == "lstm":
            ops.lstm_sequence_backward(d_h, reset, w_h, ws, d_gi, d_w_h=g_wh, grad_weight=weight, overwrite=overwrite, d_carry0=d_carry0)
        else:
            ops.gru_sequence_backward(d_h, reset, w_h, ws, d_gi, d_w_h=g_wh, d_b_hn=g_bhn, grad_weight=weight, overwrite=overwrite, d_h0=d_carry0)


def _dense_tree(spec: ops.MlpSpec, flat: torch.Tensor, first: int, last: int) -> Dict[str, Any]:
    sl = spec.layer_slices()
    out: Dict[str, Any] = {}
    for i in range(first, last):
        out[f"Dense_{i - first}"] = {"kernel": flat[sl[i][0]].view(spec.sizes[i], spec.sizes[i + 1]), "bias": flat[sl[i][1]]}
    for i, b in enumerate(spec.ln_bias_slices()):
        if b is not None and first <= i < last:
            out[f"LayerNorm_{i - first}"] = {"scale": out[f"Dense_{i - first}"].pop("bias"), "bias": flat[b]}
    return out


class _Recurrent:
    head_name = "head"

    def __init__(self, head, post_torso, hidden_state_dim: int, cell_type: str, pre_torso, input_layer=None):
        self.head, self.post_torso, self.pre_torso = head, post_torso, pre_torso
        self.rnn = ScannedRNN(hidden_state_dim, cell_type)
        self.hidden_state_dim, self.cell_type = self.rnn.hidden_state_dim, self.rnn.cell_type
        self.input_layer = input_layer if input_layer is not None else ArrayInput()
        self._ws: Dict[Tuple[int, int], torch.Tensor] = {}

    def layout_for(self, obs_dim: int) -> RecLayout:
        return RecLayout(obs_dim, self.pre_torso.layer_sizes, self.hidden_state_dim, self.post_torso.layer_sizes, self.head.out_dim,
                         self.pre_torso.activation, self.pre_torso.use_layer_norm, self.post_torso.activation, self.post_torso.use_layer_norm,
                         self.cell_type, getattr(self.head, "branch_sizes", None))

    def build_tree(self, lay: RecLayout, flat: torch.Tensor) -> ParamTree:
        H = lay.H
        pre, w_h, b_hn, post = lay.blocks(flat)
        n_pre, n_post = lay.spec_pre.n_layers, lay.spec_post.n_layers
        sl = lay.spec_pre.layer_slices()
        w_i = pre[sl[n_pre - 1][0]].view(lay.spec_pre.sizes[n_pre - 1], lay.G * H)
        b_i = pre[sl[n_pre - 1][1]]
        blk = lambda m, g: m[..., g * H:(g + 1) * H]
        if lay.cell_type == "gru":
            cell_name = "GRUCell_0"
            cell = {"ir": {"kernel": blk(w_i, 0), "bias": blk(b_i, 0)}, "iz": {"kernel": blk(w_i, 1), "bias": blk(b_i, 1)},
                    "in": {"kernel": blk(w_i, 2), "bias": blk(b_i, 2)}, "hr": {"kernel": blk(w_h, 0)}, "hz": {"kernel": blk(w_h, 1)},
                    "hn": {"kernel": blk(w_h, 2), "bias": b_hn}}
        else:   # flax LSTMCell: input Denses without bias, hidden Denses with bias (stored as the bias of the fused input projection)
            cell_name = "LSTMCell_0"
            cell = {}
            for g, nm in enumerate("ifgo"):
                cell["i" + nm] = {"kernel": blk(w_i, g)}
                cell["h" + nm] = {"kernel": blk(w_h, g), "bias": blk(b_i, g)}
        if lay.dueling:   # DuelingQNetwork: MLPTorso_0 = value branch, MLPTorso_1 = advantage branch
            n_t, sv = lay.n_post_torso, lay.spec_value
            head = {"MLPTorso_0": _dense_tree(sv, flat[lay.off_value: lay.param_count], 0, sv.n_layers),
                    "MLPTorso_1": _dense_tree(lay.spec_post, post, n_t, n_post)}
        else:
            n_t, head = n_post - 1, _dense_tree(lay.spec_post, post, n_post - 1, n_post)
        tree = ParamTree({"params": {"pre_torso": _dense_tree(lay.spec_pre, pre, 0, n_pre - 1), "ScannedRNN_0": {cell_name: cell},
                                     "post_torso": _dense_tree(lay.spec_post, post, 0, n_t), self.head_name: head}})
        tree.flat, tree.layout, tree.spec, tree.flat_bf16 = flat[: lay.param_count], lay, lay.spec_post, None
        return tree

    def init(self, key, hstate: torch.Tensor, x, flat: Optional[torch.Tensor] = None) -> ParamTree:
        """`x` = (observation (T, E, D), done (T, E)) as the reference's init_x (rec_ppo.py:478-491).  Torso kernels orthogonal(sqrt 2),
        heads orthogonal(head scale), cell: input kernels lecun-normal, recurrent kernels orthogonal per gate, zero biases (flax)."""
        from .heads import _seed_to_int

        obs = x[0]
        lay = self.layout_for(obs.shape[-1])
        gen = torch.Generator().manual_seed(_seed_to_int(key) % (2**63))
        host = torch.zeros(lay.param_count, dtype=torch.float32)
        H = lay.H
        for spec, off, torso, is_post in ((lay.spec_pre, lay.off_pre, self.pre_torso, False), (lay.spec_post, lay.off_post, self.post_torso, True)):
            sl = spec.layer_slices()
            for i in range(spec.n_layers):
                last = i == spec.n_layers - 1
                w = host[off:][sl[i][0]]
                if last and not is_post:      # W_i: G Dense(features=H) with the default lecun_normal initialiser
                    w.copy_((torch.randn(spec.sizes[i], lay.G * H, generator=gen) / np.sqrt(spec.sizes[i])).reshape(-1))
                else:
                    scale = self.head.kernel_init_scale if last else torso.kernel_init_scale
                    w.copy_(_orthogonal(gen, spec.sizes[i], spec.sizes[i + 1], scale).reshape(-1))
                if spec.has_ln(i):
                    host[off:][sl[i][1]] = 1.0
        host[lay.off_wh: lay.off_bhn].copy_(torch.cat([_orthogonal(gen, H, H, 1.0) for _ in range(lay.G)], dim=1).reshape(-1))
        if lay.dueling:   # the value branch: orthogonal(kernel_init) kernels, LayerNorm scales 1, biases 0
            sv, sl = lay.spec_value, lay.spec_value.layer_slices()
            for i in range(sv.n_layers):
                host[lay.off_value:][sl[i][0]] = _orthogonal(gen, sv.sizes[i], sv.sizes[i + 1], self.head.kernel_init_scale).reshape(-1)
                host[lay.off_value:][sl[i][1]] = 1.0
        if flat is None:
            flat = torch.zeros(lay.param_count, dtype=torch.float32, device=obs.device)
        flat[: lay.param_count].copy_(host)
        return self.build_tree(lay, flat)

    def _forward(self, params: ParamTree, hstate: torch.Tensor, observation_done):
        """Inference form (rollout step, evaluator): pre-torso + input projections for all steps, the recurrence, post-torso + head."""
        observation, done = observation_done
        obs = self.input_layer(observation).float()
        T, E, D = obs.shape
        lay: RecLayout = params.layout
        pre, _, _, post = lay.blocks(params.flat)
        gi = ops.mlp_forward(lay.spec_pre, pre, obs.reshape(T * E, D).contiguous(), ws_key=("rec_pre", id(self)))
        ws = self._ws.get((T, E))
        if ws is None:
            ws = self._ws[(T, E)] = lay.sequence_workspace(T, E, obs.device)
        d8 = done.to(torch.uint8) if done.dtype not in (torch.uint8, torch.bool) else done
        last = torch.empty(E, lay.S, dtype=torch.float32, device=obs.device)
        h_seq = lay.sequence_forward(params.flat, gi.view(T, E, lay.G * lay.H), d8.contiguous(), hstate.contiguous(), ws, carry_last=last)
        out = ops.mlp_forward(lay.spec_post, post, h_seq.view(T * E, lay.H), ws_key=("rec_post", id(self)))
        if lay.dueling:
            out = ops.dueling_q(out, lay.value_bias(params.flat))
        return last, out.view(T, E, -1)


class RecurrentActor(_Recurrent):
    """networks/base.py:162-190: (policy_hidden_state, (observation, done)) -> (policy_hidden_state, distribution)."""

    head_name = "action_head"

    def __init__(self, action_head, post_torso, hidden_state_dim: int, cell_type: str, pre_torso, input_layer=None):
        super().__init__(action_head, post_torso, hidden_state_dim, cell_type, pre_torso, input_layer)
        self.action_head = action_head

    def apply(self, params: ParamTree, policy_hidden_state: torch.Tensor, observation_done):
        h, logits = self._forward(params, policy_hidden_state, observation_done)
        return h, self.action_head.distribution(logits)

    __call__ = apply


class RecurrentCritic(_Recurrent):
    """networks/base.py:193-222: (critic_hidden_state, (observation, done)) -> (critic_hidden_state, value (T, E))."""

    head_name = "critic_head"

    def __init__(self, critic_head, post_torso, hidden_state_dim: int, cell_type: str, pre_torso, input_layer=None):
        super().__init__(critic_head, post_torso, hidden_state_dim, cell_type, pre_torso, input_layer)
        self.critic_head = critic_head

    def apply(self, params: ParamTree, critic_hidden_state: torch.Tensor, observation_done):
        h, v = self._forward(params, critic_hidden_state, observation_done)
        return h, v.squeeze(-1)

    __call__ = apply
