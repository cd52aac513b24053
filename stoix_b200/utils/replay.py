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
