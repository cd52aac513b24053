"""CategoricalHead / NormalAffineTanhDistributionHead / ScalarCriticHead -- constructor-compatible with
stoix/networks/heads.py:30-41, 44-65, 129-134, and the distribution objects the actor returns (tfd.Categorical's sample /
log_prob / entropy / mode as used at ff_ppo.py:100-101,199,205; the tanh-Normal's sample / log_prob / mode as used at
ff_sac.py:119-122,165-167); DiscreteQNetworkHead (heads.py:202-217) and its EpsilonGreedy (ff_pqn.py:79-82);
DistributionalDiscreteQNetwork and QuantileDiscreteQNetwork (heads.py:236-292)."""
from __future__ import annotations

from typing import Optional, Sequence, Union

import numpy as np
import torch

from .. import ops


class Categorical:
    """Categorical(logits) backed by stx_categorical."""

    def __init__(self, logits: torch.Tensor):
        self.logits = logits
        self._lead = tuple(logits.shape[:-1])                     # any leading shape, e.g. (T, E) from the recurrent networks
        self._flat = logits.reshape(-1, logits.shape[-1]).contiguous()

    def sample(self, seed=None, offset: int = 0, dev_counter: Optional[torch.Tensor] = None) -> torch.Tensor:
        """`seed` is an int or a PRNG key tensor (any integer tensor: its first two words are used)."""
        s = _seed_to_int(seed)
        a, lp, _ = ops.categorical(self._flat, None, s, offset, dev_counter)
        a, lp = a.view(self._lead), lp.view(self._lead)
        self._last = (a, lp)
        return a

    def log_prob(self, action: torch.Tensor) -> torch.Tensor:
        last = getattr(self, "_last", None)
        if last is not None and last[0] is action:
            return last[1]
        _, lp, _ = ops.categorical(self._flat, action.to(torch.int32).reshape(-1).contiguous())
        return lp.view(self._lead)

    def entropy(self) -> torch.Tensor:
        a = torch.zeros(self._flat.shape[0], dtype=torch.int32, device=self.logits.device)
        _, _, ent = ops.categorical(self._flat, a, want_entropy=True)
        return ent.view(self._lead)

    def kl_divergence(self, other: "Categorical") -> torch.Tensor:
        """KL(self || other) per row (tfd.Categorical.kl_divergence, as ppo_penalty_loss calls it, loss.py:44)."""
        if not isinstance(other, Categorical) or other._flat.shape != self._flat.shape:
            raise TypeError("Categorical.kl_divergence: `other` must be a Categorical over the same shape")
        return ops.categorical_kl(self._flat, other._flat).view(self._lead)

    def mode(self) -> torch.Tensor:
        return torch.argmax(self.logits, dim=-1).to(torch.int32)


def _seed_to_int(seed) -> int:
    if seed is None:
        return 0
    if isinstance(seed, torch.Tensor):
        w = seed.reshape(-1).to(torch.int64).cpu().tolist()
        return ((w[0] & 0xFFFFFFFF) << 32 | (w[-1] & 0xFFFFFFFF)) & (2**64 - 1)
    return int(seed) & (2**64 - 1)


class CategoricalHead:
    def __init__(self, action_dim: Union[int, Sequence[int]], kernel_init: Optional[float] = None):
        if not isinstance(action_dim, (int, np.integer)):
            raise NotImplementedError("factorised action_dim is outside the hot path of this build")
        self.action_dim = int(action_dim)
        self.out_dim = self.action_dim
        self.kernel_init_scale = 0.01 if kernel_init is None else float(kernel_init)  # heads.py:32

    def distribution(self, logits: torch.Tensor) -> Categorical:
        return Categorical(logits)


class ScalarCriticHead:
    def __init__(self, kernel_init: Optional[float] = None):
        self.out_dim = 1
        self.kernel_init_scale = 1.0 if kernel_init is None else float(kernel_init)  # heads.py:130


class AffineTanhNormal:
    """Independent(AffineTanhTransformedDistribution(Normal(loc, scale), minimum, maximum)) (stoix/networks/distributions.py:19-79)
    backed by stx_tanh_normal_sample.  `head_out` = (rows, 2A): loc | scale pre-activation."""

    def __init__(self, head_out: torch.Tensor, minimum: float, maximum: float, min_scale: float):
        self.head_out, self.minimum, self.maximum, self.min_scale = head_out, float(minimum), float(maximum), float(min_scale)
        self._last = None

    def sample(self, seed=None, offset: int = 0, dev_counter: Optional[torch.Tensor] = None) -> torch.Tensor:
        a, lp, eps = ops.tanh_normal_sample(self.head_out, self.minimum, self.maximum, self.min_scale, seed=_seed_to_int(seed), offset=offset,
                                            dev_counter=dev_counter)
        self._last = (a, lp, eps)
        return a

    def _rows(self) -> torch.Tensor:
        return self.head_out.reshape(-1, self.head_out.shape[-1]).contiguous()

    def log_prob(self, action: torch.Tensor) -> torch.Tensor:
        """log_prob of `action` (distributions.py:56-80).  The action this object has just sampled returns the value the sampler
        computed with it (ff_sac.py:165-167); any other action is scored by stx_tanh_normal_log_prob."""
        if self._last is not None and self._last[0] is action:
            return self._last[1]
        A = self.head_out.shape[-1] // 2
        a = action.to(torch.float32).reshape(-1, A).contiguous()
        return ops.tanh_normal_log_prob(self._rows(), a, self.minimum, self.maximum, self.min_scale).view(self.head_out.shape[:-1])

    def entropy(self, seed=None, offset: int = 0, dev_counter: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The reference's seeded one-sample estimate entropy(seed) (distributions.py:85-88) per row: Normal entropy plus the
        log-det-Jacobian of the Shift / Scale / Tanh chain at a Normal sample drawn with `seed`."""
        ent, _ = ops.tanh_normal_entropy(self._rows(), self.minimum, self.maximum, self.min_scale, seed=_seed_to_int(seed), offset=offset,
                                         dev_counter=dev_counter)
        return ent.view(self.head_out.shape[:-1])

    def kl_divergence(self, other: "AffineTanhNormal") -> torch.Tensor:
        """KL(self || other) per row.  Both transform their base Normal by the same affine-tanh bijector, and a KL is invariant
        under a shared bijection, so it is the KL of the base Normals summed over the action dimensions (the registration tfp
        applies to Independent / TransformedDistribution pairs, loss.py:44)."""
        if not isinstance(other, AffineTanhNormal) or other.head_out.shape != self.head_out.shape:
            raise TypeError("AffineTanhNormal.kl_divergence: `other` must be an AffineTanhNormal over the same shape")
        if (other.minimum, other.maximum, other.min_scale) != (self.minimum, self.maximum, self.min_scale):
            raise ValueError("AffineTanhNormal.kl_divergence: both distributions must share the bounds and min_scale")
        return ops.tanh_normal_kl(self._rows(), other._rows(), self.min_scale).view(self.head_out.shape[:-1])

    def mode(self) -> torch.Tensor:
        A = self.head_out.shape[-1] // 2
        s, sh = (self.maximum - self.minimum) / 2.0, (self.minimum + self.maximum) / 2.0
        return sh + s * torch.tanh(self.head_out[..., :A])


class EpsilonGreedy:
    """distrax.EpsilonGreedy(preferences=q, epsilon) backed by stx_epsilon_greedy: with probability 1 - epsilon a uniformly chosen
    maximal action, else a uniform action.  `sample` draws from Philox (seed, row, offset + *dev_counter); `mode` is the first
    argmax."""

    def __init__(self, preferences: torch.Tensor, epsilon: float):
        self.preferences = preferences
        self.epsilon = float(epsilon)
        self._lead = tuple(preferences.shape[:-1])
        self._flat = preferences.reshape(-1, preferences.shape[-1]).contiguous()

    def _sched(self):
        return ops.epsilon_schedule_struct(self.epsilon, self.epsilon, 0.0, decay=False)

    def sample(self, seed=None, offset: int = 0, dev_counter: Optional[torch.Tensor] = None) -> torch.Tensor:
        return ops.epsilon_greedy(self._flat, self._sched(), _seed_to_int(seed), offset, dev_counter).view(self._lead)

    def mode(self) -> torch.Tensor:
        return ops.epsilon_greedy(self._flat, self._sched(), mode=True).view(self._lead)


class DiscreteQNetworkHead:
    """heads.py:202-217: Dense(action_dim), orthogonal(1.0) kernel, returning EpsilonGreedy(q, epsilon); `epsilon` passed at apply
    time (head_kwargs) overrides the constructor's."""

    def __init__(self, action_dim: int, epsilon: float = 0.1, kernel_init: Optional[float] = None):
        self.action_dim = int(action_dim)
        self.epsilon = float(epsilon)
        self.out_dim = self.action_dim
        self.kernel_init_scale = 1.0 if kernel_init is None else float(kernel_init)

    def distribution(self, q_values: torch.Tensor, epsilon: Optional[float] = None) -> EpsilonGreedy:
        return EpsilonGreedy(q_values, self.epsilon if epsilon is None else epsilon)


class NormalAffineTanhDistributionHead:
    """heads.py:44-65: loc = Dense(A), scale = softplus(Dense(A)) + min_scale, both orthogonal(0.01); the two Dense layers are
    ONE (in x 2A) matrix in the arena: columns [0, A) = loc (flax `Dense_0`), [A, 2A) = scale (`Dense_1`)."""

    def __init__(self, action_dim: int, minimum: float, maximum: float, min_scale: float = 1e-3, kernel_init: Optional[float] = None):
        self.action_dim, self.minimum, self.maximum, self.min_scale = int(action_dim), float(minimum), float(maximum), float(min_scale)
        self.out_dim = 2 * self.action_dim
        self.kernel_init_scale = 0.01 if kernel_init is None else float(kernel_init)
        self.kernel_blocks = (self.action_dim, self.action_dim)   # initialised as two independent orthogonal matrices

    def distribution(self, head_out: torch.Tensor) -> AffineTanhNormal:
        return AffineTanhNormal(head_out, self.minimum, self.maximum, self.min_scale)


def linspace_f32(start: float, stop: float, num: int) -> np.ndarray:
    """jnp.linspace(start, stop, num) in float32 by JAX's formula: start (1 - s_i) + stop s_i with s_i = i / (num - 1), the last
    point exactly `stop`.  The C51 atoms: the kernels, the value faces and the oracle all read these values."""
    start, stop = np.float32(start), np.float32(stop)
    if num == 1:
        return np.array([start], np.float32)
    s = np.arange(num, dtype=np.float32) / np.float32(num - 1)
    out = (start * (np.float32(1) - s) + stop * s).astype(np.float32)
    out[-1] = stop
    return out


class DistributionalDiscreteQNetwork:
    """heads.py:236-258: Dense(action_dim num_atoms) with a lecun_normal kernel; apply returns (EpsilonGreedy(q), logits (M, A, N),
    atoms (M, N)), q = sum_i softmax(logits[a])_i atoms_i from stx_dist_q_values."""

    kernel_init_kind = "lecun_normal"

    def __init__(self, action_dim: int, epsilon: float = 0.1, num_atoms: int = 51, vmin: float = 0.0, vmax: float = 500.0):
        self.action_dim, self.epsilon, self.num_atoms = int(action_dim), float(epsilon), int(num_atoms)
        self.vmin, self.vmax = float(vmin), float(vmax)
        self.out_dim = self.action_dim * self.num_atoms
        self.kernel_init_scale = 1.0
        self.atoms_host = linspace_f32(self.vmin, self.vmax, self.num_atoms)
        self._atoms = {}

    def atoms(self, device) -> torch.Tensor:
        """The (N) atoms on `device`, built once per device."""
        key = str(device)
        if key not in self._atoms:
            self._atoms[key] = torch.tensor(self.atoms_host, device=device)
        return self._atoms[key]

    def distribution(self, logits: torch.Tensor, epsilon: Optional[float] = None):
        A, N = self.action_dim, self.num_atoms
        flat = logits.reshape(-1, A * N).contiguous()
        atoms = self.atoms(flat.device)
        q = ops.dist_q_values("categorical", flat, A, N, atoms)
        return (EpsilonGreedy(q, self.epsilon if epsilon is None else epsilon), flat.view(-1, A, N),
                atoms.expand(flat.shape[0], N))


class QuantileDiscreteQNetwork:
    """heads.py:275-292: Dense(action_dim num_quantiles) with a lecun_normal kernel; apply returns (EpsilonGreedy(q), q_dist (M, A, N)),
    q = mean_i q_dist[a, i] from stx_dist_q_values."""

    kernel_init_kind = "lecun_normal"

    def __init__(self, action_dim: int, epsilon: float = 0.1, num_quantiles: int = 200):
        self.action_dim, self.epsilon, self.num_quantiles = int(action_dim), float(epsilon), int(num_quantiles)
        self.out_dim = self.action_dim * self.num_quantiles
        self.kernel_init_scale = 1.0

    def distribution(self, out: torch.Tensor, epsilon: Optional[float] = None):
        A, N = self.action_dim, self.num_quantiles
        flat = out.reshape(-1, A * N).contiguous()
        q = ops.dist_q_values("quantile", flat, A, N)
        return EpsilonGreedy(q, self.epsilon if epsilon is None else epsilon), flat.view(-1, A, N)
