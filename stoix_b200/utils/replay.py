"""Transition replay buffer on the GPU -- the part of flashbax's item buffer the SAC systems use
(`fbx.make_item_buffer(max_length, min_length, sample_batch_size, add_batches=True, add_sequences=True)`,
stoix/systems/sac/ff_sac.py:449-456): `add` appends a (T, E, ...) batch of transitions to the ring (oldest overwritten),
`sample` draws `sample_batch_size` items uniformly WITH replacement from the valid part.  The write position and fill count
live in device memory (stx_replay_add / stx_replay_sample), so a whole update step -- rollout, add, sample, three losses,
optimiser -- is stream-ordered and can be captured into one CUDA graph."""
from __future__ import annotations

from typing import Optional

import torch

from stoix_b200 import ops


class TransitionBuffer:
    def __init__(self, max_length: int, min_length: int, sample_batch_size: int, obs_dim: int, act_dim: int, device, seed: int = 0):
        self.max_length, self.min_length, self.sample_batch_size = int(max_length), int(min_length), int(sample_batch_size)
        self.ring = ops.ReplayRing(self.max_length, obs_dim, act_dim, device)
        self.seed = int(seed) & ((1 << 62) - 1)
        self.counter = torch.zeros(1, dtype=torch.int64, device=device)   # sample calls so far (device-resident RNG stream position)
        self.added = 0                                                    # host mirror of the item count (can_sample)

    def add(self, transition) -> None:
        """transition: anything with .obs (T, E, D), .action (T, E, A), .reward, .done (T, E), .next_obs."""
        ops.replay_add(self.ring, transition.obs, transition.action, transition.reward, transition.done, transition.next_obs)
        self.added += int(transition.reward.numel())

    def can_sample(self) -> bool:
        return min(self.added, self.max_length) >= self.min_length

    def sample_into(self, xq_old, reward, done, xq_new=None, xq_next=None, idx_in: Optional[torch.Tensor] = None,
                    idx_out: Optional[torch.Tensor] = None) -> None:
        """Draw one batch and write it as the network inputs of one epoch (see stx_replay_sample); advances the stream position."""
        ops.replay_sample(self.ring, self.sample_batch_size, self.seed, xq_old, reward, done, xq_new=xq_new, xq_next=xq_next,
                          dev_counter=self.counter.view(torch.int64), idx_in=idx_in, idx_out=idx_out)
        ops.counter_add(self.counter, 1)


class DiscreteTransitionBuffer:
    """The item buffer of the DQN family (ff_dqn.py:339-347): transitions with one integer action per row, on the discrete ring
    (stx_replay_add_discrete / stx_replay_sample_discrete), with the same add / sample semantics as TransitionBuffer."""

    def __init__(self, max_length: int, min_length: int, sample_batch_size: int, obs_dim: int, device, seed: int = 0):
        self.max_length, self.min_length, self.sample_batch_size = int(max_length), int(min_length), int(sample_batch_size)
        self.ring = ops.DiscreteReplayRing(self.max_length, obs_dim, device)
        self.seed = int(seed) & ((1 << 62) - 1)
        self.counter = torch.zeros(1, dtype=torch.int64, device=device)   # sample calls so far (device-resident RNG stream position)
        self.added = 0                                                    # host mirror of the item count (can_sample)

    def add(self, transition) -> None:
        """transition: anything with .obs (T, E, D), .action (T, E) int32, .reward, .done (T, E), .next_obs."""
        ops.replay_add_discrete(self.ring, transition.obs, transition.action, transition.reward, transition.done, transition.next_obs)
        self.added += int(transition.reward.numel())

    def can_sample(self) -> bool:
        return min(self.added, self.max_length) >= self.min_length

    def sample_into(self, obs, next_obs, action, reward, done, idx_in: Optional[torch.Tensor] = None,
                    idx_out: Optional[torch.Tensor] = None) -> None:
        """Draw one batch of sample_batch_size transitions into the given (M, ...) buffers; advances the stream position.  obs and
        next_obs may be the two halves of one (2M, D) block."""
        ops.replay_sample_discrete(self.ring, self.sample_batch_size, self.seed, obs, next_obs, action, reward, done,
                                   dev_counter=self.counter.view(torch.int64), idx_in=idx_in, idx_out=idx_out)
        ops.counter_add(self.counter, 1)


class PrioritisedTrajectoryBuffer:
    """fbx.make_prioritised_trajectory_buffer as ff_rainbow.py:433-442 builds it, on the prioritised n-step ring
    (stx_replay_add_prioritised / _sample_prioritised / stx_replay_set_priorities): add_batch_size = E envs, max_length_time_axis =
    max_size // E time rows, sequences of n_step rows with period 1.  `sample_into` draws sample_batch_size items in proportion to
    their priorities and writes each as its n-step transition (ff_rainbow.py:222-246) with p_i and the importance weight."""

    def __init__(self, max_size: int, n_step: int, sample_batch_size: int, add_batch_size: int, priority_exponent: float, obs_dim: int, device,
                 seed: int = 0):
        self.max_length_time_axis = int(max_size) // int(add_batch_size)
        self.n_step, self.sample_batch_size, self.add_batch_size = int(n_step), int(sample_batch_size), int(add_batch_size)
        self.ring = ops.PrioritisedRing(self.max_length_time_axis, self.add_batch_size, obs_dim, self.n_step, priority_exponent, device)
        self.seed = int(seed) & ((1 << 62) - 1)
        self.counter = torch.zeros(1, dtype=torch.int64, device=device)   # sample calls so far (device-resident RNG stream position)
        self.added = 0                                                    # host mirror of the items added (T E per add)

    def add(self, transition) -> None:
        """transition: .obs (T, E, D), .action (T, E) int32, .reward, .done (T, E), .next_obs, time-major."""
        ops.replay_add_prioritised(self.ring, transition.obs, transition.action, transition.reward, transition.done, transition.next_obs)
        self.added += int(transition.reward.numel())

    def can_sample(self) -> bool:
        """min_length_time_axis = n_step time rows written."""
        return self.added // self.add_batch_size >= self.n_step

    def sample_into(self, obs, next_obs, action, reward, done, idx, prob, weight, gamma: float, beta0: float, beta_steps: float,
                    count: Optional[torch.Tensor] = None, u_in: Optional[torch.Tensor] = None) -> None:
        """Draw one batch into the given (M, ...) buffers; advances the stream position.  obs and next_obs may be the two halves of
        one (2M, D) block."""
        ops.replay_sample_prioritised(self.ring, self.sample_batch_size, self.seed, obs, next_obs, action, reward, done, idx, prob, weight, gamma,
                                      beta0, beta_steps, count=count, dev_counter=self.counter.view(torch.int64), u_in=u_in)
        ops.counter_add(self.counter, 1)

    def set_priorities(self, idx: torch.Tensor, priorities: torch.Tensor) -> None:
        ops.replay_set_priorities(self.ring, idx, priorities)


class SequenceBuffer:
    """fbx.make_trajectory_buffer as ff_mpo.py:539-546 builds it, on the sequence ring (stx_replay_add_sequence / _sample_sequence):
    add_batch_size = E envs, max_length_time_axis = max_size // E time rows with one write index, sequences of sample_sequence_length
    rows with period 1 that never straddle the write head.  `sample_into` writes the batch time-major (S, B, ...) into the epoch's
    buffers."""

    def __init__(self, max_size: int, sample_batch_size: int, sample_sequence_length: int, add_batch_size: int, obs_dim: int, device,
                 period: int = 1, seed: int = 0, act_dim: int = 0):
        if int(period) != 1:
            raise ValueError(f"SequenceBuffer: period={period}; only period 1 is implemented (both MPO configs use 1)")
        self.max_length_time_axis = int(max_size) // int(add_batch_size)
        self.sample_batch_size, self.sample_sequence_length = int(sample_batch_size), int(sample_sequence_length)
        if self.max_length_time_axis < self.sample_sequence_length:
            raise ValueError(f"SequenceBuffer: max_size={max_size} over {add_batch_size} envs holds {self.max_length_time_axis} time rows, fewer "
                             f"than one sequence of sample_sequence_length={self.sample_sequence_length}")
        self.add_batch_size = int(add_batch_size)
        self.ring = ops.SequenceRing(self.max_length_time_axis, self.add_batch_size, obs_dim, device, act_dim=act_dim)   # act_dim 0: int32
        self.seed = int(seed) & ((1 << 62) - 1)
        self.counter = torch.zeros(1, dtype=torch.int64, device=device)   # sample calls so far (device-resident RNG stream position)
        self.added = 0                                                    # host mirror of the items added (T E per add)

    def add(self, step) -> None:
        """step: a time-major SequenceStep: .obs (T, E, D), .action (T, E) int32 or (T, E, act_dim) float32, .reward, .log_prob float32,
        .done, .truncated uint8."""
        ops.replay_add_sequence(self.ring, step.obs, step.action, step.reward, step.done, step.truncated, step.log_prob)
        self.added += int(step.reward.numel())

    def can_sample(self) -> bool:
        """min_length_time_axis = sample_sequence_length time rows written."""
        return min(self.added // self.add_batch_size, self.max_length_time_axis) >= self.sample_sequence_length

    def sample_into(self, obs, action, reward, done, log_prob, idx_in: Optional[torch.Tensor] = None, idx_out: Optional[torch.Tensor] = None) -> None:
        """Draw sample_batch_size sequences into the (S, B, ...) buffers; advances the stream position."""
        ops.replay_sample_sequence(self.ring, self.sample_sequence_length, self.seed, obs, action, reward, done, log_prob,
                                   dev_counter=self.counter.view(torch.int64), idx_in=idx_in, idx_out=idx_out)
        ops.counter_add(self.counter, 1)


class PrioritisedSequenceBuffer:
    """fbx.make_prioritised_trajectory_buffer as rec_r2d2.py:644-653 builds it, on the prioritised sequence ring (stx_r2d2_ring_add /
    _sample / _set_priorities): add_batch_size = E envs, max_length_time_axis = max_size // E time rows, min_length_time_axis =
    sample_sequence_length = S, items every `period` rows.  `sample_into` draws sample_batch_size sequences in proportion to their
    priorities and writes them time-major (S, B, ...) with the carry at each sequence's start, the items and p_i."""

    def __init__(self, max_size: int, sample_batch_size: int, sample_sequence_length: int, add_batch_size: int, period: int, priority_exponent: float,
                 obs_dim: int, carry_dim: int, device, seed: int = 0):
        self.max_length_time_axis = int(max_size) // int(add_batch_size)
        self.sample_batch_size, self.sample_sequence_length = int(sample_batch_size), int(sample_sequence_length)
        self.add_batch_size, self.period = int(add_batch_size), int(period)
        if self.max_length_time_axis < self.sample_sequence_length:
            raise ValueError(f"PrioritisedSequenceBuffer: max_size={max_size} over {add_batch_size} envs holds {self.max_length_time_axis} time "
                             f"rows, fewer than one sequence of sample_sequence_length={self.sample_sequence_length}")
        if not 1 <= self.period <= self.max_length_time_axis:
            raise ValueError(f"PrioritisedSequenceBuffer: period={period} must lie in [1, {self.max_length_time_axis}] (the time rows per env)")
        self.ring = ops.R2d2Ring(self.max_length_time_axis, self.add_batch_size, obs_dim, carry_dim, self.sample_sequence_length, self.period,
                                 priority_exponent, device)
        self.seed = int(seed) & ((1 << 62) - 1)
        self.counter = torch.zeros(1, dtype=torch.int64, device=device)   # sample calls so far (device-resident RNG stream position)
        self.added = 0                                                    # host mirror of the items added (T E per add)

    def add(self, tr) -> None:
        """tr: a time-major RNNTransition: .obs (T, E, D), .action int32, .reward, .reset_hidden_state, .done, .truncated (T, E) and
        .hstate (T, E, carry_dim), the carry entering each step."""
        ops.r2d2_ring_add(self.ring, tr.obs, tr.action, tr.reward, tr.done, tr.truncated, tr.reset_hidden_state, tr.hstate)
        self.added += int(tr.reward.numel())

    def can_sample(self) -> bool:
        """min_length_time_axis = sample_sequence_length time rows written."""
        return min(self.added // self.add_batch_size, self.max_length_time_axis) >= self.sample_sequence_length

    def sample_into(self, obs, action, reward, done, reset, carry0, idx, prob, u_in: Optional[torch.Tensor] = None) -> None:
        """Draw one batch into the (S, B, ...) buffers, carry0 (B, carry_dim), idx and prob (B); advances the stream position."""
        ops.r2d2_ring_sample(self.ring, self.seed, obs, action, reward, done, reset, carry0, idx, prob, dev_counter=self.counter.view(torch.int64),
                             u_in=u_in)
        ops.counter_add(self.counter, 1)

    def set_priorities(self, idx: torch.Tensor, priorities: torch.Tensor) -> None:
        ops.r2d2_ring_set_priorities(self.ring, idx, priorities)
