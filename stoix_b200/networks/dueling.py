"""NoisyDistributionalDuelingQNetwork (stoix/networks/dueling.py:90-124) and the noisy feed-forward network Rainbow runs it in.

Every NoisyLinear (stoix/networks/layers.py:71-169) keeps mu and sigma in one flat fp32 arena, in the order and with the names of the
flax tree: `{'params': {'torso': {'NoisyLinear_k': ...}, 'action_head': {'NoisyMLPTorso_0': {'NoisyLinear_k': ...}, 'NoisyMLPTorso_1':
{...}, 'NoisyLinear_0': ..., 'NoisyLinear_1': ...}}}`, each layer `{kernel (in, out), bias (out), sigma_w (in, out), sigma_b (out)}`, laid
out in that order.  The optimiser, the target update, the all-reduce and checkpoints see only this arena.

A forward draws fresh factorised noise and writes the effective weights mu + sigma o eps into a dense StxMlp arena (stx_noisy_weights);
the fp32 MLP kernels run unchanged on it.  The whole network is one MLP chain:
  (D, *torso, 2 b_1, ..., 2 b_k, N + A N)
The value and advantage branches sit side by side: their first layers read the same torso output, so that layer is the two kernels
next to each other (columns [0, b_1) value, [b_1, 2 b_1) advantage); every later branch layer and the output layer are block
diagonal (value rows and columns first), the off-diagonal blocks zero and never written.  The output row is (v (N) | adv (A N)),
which stx_dueling_combine turns into the q_logits (A N) the C51 kernels read."""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import ops
from .base import ParamTree, _lecun_normal
from .heads import DistributionalDiscreteQNetwork, EpsilonGreedy, _seed_to_int
from .torso import NoisyMLPTorso
from .utils import parse_activation_fn


class DuelingQNetwork:
    """dueling.py:15-49: value MLPTorso((*layer_sizes, 1)) and advantage MLPTorso((*layer_sizes, A)) branches with activate_final=False,
    q = v + (adv - mean_a adv), returning EpsilonGreedy(q, epsilon).  A description: the recurrent Q network (networks/recurrent.py)
    runs it; only its use_layer_norm=True form is built, where the value branch's output is its final LayerNorm bias."""

    def __init__(self, action_dim: int, epsilon: float, layer_sizes: Sequence[int], activation: str = "relu", use_layer_norm: bool = False,
                 kernel_init: Optional[float] = None):
        self.action_dim, self.epsilon = int(action_dim), float(epsilon)
        self.branch_sizes = tuple(int(s) for s in layer_sizes)
        self.activation, self.use_layer_norm = parse_activation_fn(activation), bool(use_layer_norm)
        self.out_dim = self.action_dim
        self.kernel_init_scale = float(np.sqrt(2.0)) if kernel_init is None else float(kernel_init)   # dueling.py:23

    def distribution(self, q_values: torch.Tensor, epsilon: Optional[float] = None) -> EpsilonGreedy:
        return EpsilonGreedy(q_values, self.epsilon if epsilon is None else epsilon)


class NoisyDistributionalDuelingQNetwork(DistributionalDiscreteQNetwork):
    """dueling.py:90-124: value and advantage NoisyMLPTorso(layer_sizes) branches, NoisyLinear(N) and NoisyLinear(A N) heads,
    q_logits = v + adv - mean_a adv; apply returns (EpsilonGreedy(q), q_logits (M, A, N), atoms (M, N)) like the C51 head."""

    def __init__(self, action_dim: int, epsilon: float, layer_sizes: Sequence[int], sigma_zero: float, num_atoms: int = 51, vmin: float = 0.0,
                 vmax: float = 500.0, activation: str = "relu", use_layer_norm: bool = False, kernel_init: Optional[float] = None):
        super().__init__(action_dim, epsilon, num_atoms, vmin, vmax)
        # dueling.py:104-109 passes sigma_zero as the 4th positional argument of NoisyMLPTorso, whose 4th field is kernel_init
        # (torso.py:36-44), which NoisyLinear never reads: the two branches keep NoisyMLPTorso's default sigma_zero = 0.5.  Restated
        # as written; only the two output NoisyLinear layers take this sigma_zero.
        self.branch = NoisyMLPTorso(layer_sizes, activation, use_layer_norm, sigma_zero)
        self.layer_sizes, self.activation, self.use_layer_norm = self.branch.layer_sizes, self.branch.activation, self.branch.use_layer_norm
        self.sigma_zero = float(sigma_zero)
        self.out_dim = self.num_atoms + self.action_dim * self.num_atoms   # the (v | adv) row of the last MLP layer


class NoisyLayout:
    """Where each NoisyLinear of the network lives: its flax path, its floats in the parameter arena, its block of the effective
    StxMlp arena (`spec`) and its noise (f_in | f_out)."""

    def __init__(self, obs_dim: int, torso: NoisyMLPTorso, head: NoisyDistributionalDuelingQNetwork):
        N, A = head.num_atoms, head.action_dim
        t_sizes, b_sizes = list(torso.layer_sizes), list(head.layer_sizes)
        self.spec = ops.MlpSpec(tuple([int(obs_dim), *t_sizes, *(2 * b for b in b_sizes), N + A * N]), activation=torso.activation)
        sl = self.spec.layer_slices()
        m, k = len(t_sizes), len(b_sizes)
        t_out = t_sizes[-1] if t_sizes else int(obs_dim)
        # (path, in, out, eff_w, eff_b, ld, sigma_zero of the module that owns the layer) in parameter order
        rows: List[Tuple[Tuple[str, ...], int, int, int, int, int, float]] = []
        prev = int(obs_dim)
        for i, s in enumerate(t_sizes):
            rows.append((("torso", f"NoisyLinear_{i}"), prev, s, sl[i][0].start, sl[i][1].start, s, torso.sigma_zero))
            prev = s
        for h in range(2):   # NoisyMLPTorso_0 = value branch, NoisyMLPTorso_1 = advantage branch
            b_in = t_out
            for j, b in enumerate(b_sizes):
                ld, row_off = 2 * b, (0 if j == 0 else h * b_in)
                rows.append((("action_head", f"NoisyMLPTorso_{h}", f"NoisyLinear_{j}"), b_in, b, sl[m + j][0].start + row_off * ld + h * b,
                             sl[m + j][1].start + h * b, ld, head.branch.sigma_zero))
                b_in = b
        ld = N + A * N
        b_in = b_sizes[-1] if b_sizes else t_out
        for h, (cols, col_off) in enumerate(((N, 0), (A * N, N))):   # NoisyLinear_0 = value logits, NoisyLinear_1 = advantage logits
            row_off = h * b_in if k else 0
            rows.append((("action_head", f"NoisyLinear_{h}"), b_in, cols, sl[m + k][0].start + row_off * ld + col_off, sl[m + k][1].start + col_off, ld,
                         head.sigma_zero))
        if len(rows) > ops._lib.STX_NOISY_MAX_LAYERS:
            raise ValueError(f"the noisy dueling network has {len(rows)} NoisyLinear layers; at most {ops._lib.STX_NOISY_MAX_LAYERS} are supported")
        self.layers: List[Dict[str, Any]] = []
        p = q = 0
        for path, n_in, n_out, eff_w, eff_b, ld, sigma_zero in rows:
            self.layers.append(dict(path=path, in_=n_in, out=n_out, param=p, eff_w=eff_w, eff_b=eff_b, noise=q, ld=ld, sigma_zero=sigma_zero))
            p += 2 * n_in * n_out + 2 * n_out
            q += n_in + n_out
        self.param_count, self.noise_count, self.eff_count = p, q, self.spec.param_count
        self.net = ops.noisy_net_struct([(L["param"], L["eff_w"], L["eff_b"], L["noise"], L["in_"], L["out"], L["ld"]) for L in self.layers])
        self.sizes = (self.param_count, self.eff_count, self.noise_count)

    def tree(self, flat: torch.Tensor) -> ParamTree:
        """The flax-named views of a parameter arena."""
        root: Dict[str, Any] = {}
        for L in self.layers:
            n_in, n_out, o = L["in_"], L["out"], L["param"]
            W = n_in * n_out
            node = root
            for name in L["path"][:-1]:
                node = node.setdefault(name, {})
            node[L["path"][-1]] = {"kernel": flat[o:o + W].view(n_in, n_out), "bias": flat[o + W:o + W + n_out],
                                   "sigma_w": flat[o + W + n_out:o + 2 * W + n_out].view(n_in, n_out), "sigma_b": flat[o + 2 * W + n_out:o + 2 * W + 2 * n_out]}
        tree = ParamTree({"params": root})
        tree.flat = flat[: self.param_count]
        tree.spec = self.spec
        tree.layout = self
        return tree

    def weights(self, params: torch.Tensor, eff: torch.Tensor, noise: torch.Tensor, seed: int = 0, offset: int = 0,
                dev_counter: Optional[torch.Tensor] = None, draw: bool = True) -> None:
        ops.noisy_weights(self.net, params, eff, noise, seed, offset, dev_counter, draw, self.sizes)

    def fold(self, eff_grad: torch.Tensor, noise: torch.Tensor, grad: torch.Tensor, overwrite: bool = True) -> None:
        ops.noisy_fold(self.net, eff_grad, noise, grad, overwrite, self.sizes)

    def scratch(self, device) -> Tuple[torch.Tensor, torch.Tensor]:
        """A zero effective arena (its off-diagonal blocks stay zero) and a noise buffer."""
        return (torch.zeros(self.eff_count, dtype=torch.float32, device=device), torch.zeros(self.noise_count, dtype=torch.float32, device=device))


class NoisyFeedForwardActor:
    """FeedForwardActor(torso=NoisyMLPTorso, action_head=NoisyDistributionalDuelingQNetwork) (stoix/networks/base.py:18-36) with the
    noise passed at apply time: `apply(params, obs, seed, offset, dev_counter)` draws the noise of call offset + *dev_counter."""

    head_name = "action_head"

    def __init__(self, action_head: NoisyDistributionalDuelingQNetwork, torso: NoisyMLPTorso):
        self.action_head, self.torso = action_head, torso
        self._layouts: Dict[int, NoisyLayout] = {}
        self._scratch: Dict[Tuple[str, str], Tuple[torch.Tensor, torch.Tensor]] = {}

    def layout(self, obs_dim: int) -> NoisyLayout:
        if obs_dim not in self._layouts:
            self._layouts[obs_dim] = NoisyLayout(obs_dim, self.torso, self.action_head)
        return self._layouts[obs_dim]

    def spec_for(self, obs_dim: int) -> ops.MlpSpec:
        return self.layout(obs_dim).spec

    def init(self, key, x: torch.Tensor, flat: Optional[torch.Tensor] = None) -> ParamTree:
        """NoisyLinear init (layers.py:120-150): kernel lecun_normal, bias 0, sigma_w = sigma_b = sigma_zero / sqrt(fan_in) in fp32, with
        the sigma_zero of the module that owns the layer (the torso's, 0.5 for the dueling branches, the head's for its outputs)."""
        lay = self.layout(int(x.shape[-1]))
        gen = torch.Generator().manual_seed(_seed_to_int(key) % (2**63))
        host = torch.zeros(lay.param_count, dtype=torch.float32)
        for L in lay.layers:
            n_in, n_out, o = L["in_"], L["out"], L["param"]
            W = n_in * n_out
            sigma = float(np.float32(L["sigma_zero"]) / np.sqrt(np.float32(n_in)))
            host[o:o + W] = _lecun_normal(gen, n_in, n_out, 1.0).reshape(-1)
            host[o + W + n_out:o + 2 * W + 2 * n_out] = sigma
        if flat is None:
            flat = torch.zeros(lay.param_count, dtype=torch.float32, device=x.device)
        flat[: lay.param_count].copy_(host)
        return lay.tree(flat)

    def head_rows(self, params: ParamTree, x: torch.Tensor, seed: int = 0, offset: int = 0, dev_counter: Optional[torch.Tensor] = None,
                  ws_key: str = "noisy_apply") -> torch.Tensor:
        """(v | adv) rows (M, N + A N) of a fresh noise draw."""
        lay = params.layout
        key = (ws_key, str(x.device))
        if key not in self._scratch:
            self._scratch[key] = lay.scratch(x.device)
        eff, noise = self._scratch[key]
        lay.weights(params.flat, eff, noise, seed, offset, dev_counter)
        return ops.mlp_forward(lay.spec, eff, x, ws_key=ws_key)

    def apply(self, params: ParamTree, observation: torch.Tensor, seed=0, offset: int = 0, dev_counter: Optional[torch.Tensor] = None,
              epsilon: Optional[float] = None):
        h = self.action_head
        lead = observation.shape[:-1]
        x = observation.reshape(-1, observation.shape[-1]).float().contiguous()
        logits = ops.dueling_combine(self.head_rows(params, x, _seed_to_int(seed), offset, dev_counter), h.action_dim, h.num_atoms)
        pi, q_logits, atoms = h.distribution(logits, epsilon)
        if len(lead) != 1:
            pi = EpsilonGreedy(pi.preferences.view(*lead, h.action_dim), pi.epsilon)
        return pi, q_logits, atoms

    __call__ = apply
