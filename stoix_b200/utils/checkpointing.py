"""Checkpoint hooks with the reference's call shape (stoix/utils/checkpointing.py:20-179:
`Checkpointer(...).save(timestep, unreplicated_learner_state, episode_return)` and
`restore_params`).  Storage is torch.save of the flat arenas instead of an orbax tree; like the
reference, restore loads parameters only (warm start, checkpointing.py:129-179)."""
from __future__ import annotations

import time
from pathlib import Path
from typing import Any, Dict, Optional

import torch

from stoix_b200.config import to_container


class Checkpointer:
    def __init__(self, model_name: str, metadata: Optional[Dict] = None, rel_dir: str = "checkpoints",
                 checkpoint_uid: Optional[str] = None, save_interval_steps: int = 1, max_to_keep: Optional[int] = 1,
                 keep_period: Optional[int] = None, **_: Any):
        uid = checkpoint_uid or time.strftime("%Y%m%d%H%M%S")
        self.dir = Path.cwd() / rel_dir / model_name / uid
        self.metadata = metadata or {}
        self.max_to_keep = max_to_keep
        self.save_interval_steps = max(int(save_interval_steps), 1)
        if keep_period is not None:
            raise NotImplementedError("Checkpointer(keep_period=...) is not supported by the torch.save store")
        self.best = -float("inf")
        self._last_saved: Optional[int] = None

    def save(self, timestep: int, unreplicated_learner_state, episode_return: float = 0.0) -> bool:
        """checkpointing.py:88-127: a step is written when it is at least save_interval_steps past the last one."""
        if self._last_saved is not None and int(timestep) - self._last_saved < self.save_interval_steps:
            return False
        self._last_saved = int(timestep)
        self.dir.mkdir(parents=True, exist_ok=True)
        p = unreplicated_learner_state.params.actor_params
        blob = {"timestep": int(timestep), "episode_return": float(episode_return), "metadata": self.metadata,
                "params": p.arena.detach().cpu(), "mu": p.arena_mu.detach().cpu(), "nu": p.arena_nu.detach().cpu(),
                "counts": p.arena_counts.detach().cpu()}
        torch.save(blob, self.dir / f"{int(timestep)}.pt")
        if episode_return >= self.best:
            self.best = episode_return
            torch.save(blob, self.dir / "best.pt")
        if self.max_to_keep:
            ckpts = sorted((q for q in self.dir.glob("*.pt") if q.stem.isdigit()), key=lambda q: int(q.stem))
            for q in ckpts[: -self.max_to_keep]:
                q.unlink()
        return True

    def restore_params(self, arena: torch.Tensor, timestep: Optional[int] = None) -> torch.Tensor:
        """checkpointing.py:129-179: restores the requested step, by default the LATEST saved one."""
        if timestep is None:
            steps = sorted(int(q.stem) for q in self.dir.glob("*.pt") if q.stem.isdigit())
            if not steps:
                raise FileNotFoundError(f"no checkpoint under {self.dir}")
            timestep = steps[-1]
        path = self.dir / f"{timestep}.pt"
        blob = torch.load(path, map_location="cpu")
        arena.copy_(blob["params"])
        return arena


def warm_start(config, arena: torch.Tensor) -> bool:
    """Warm start: with logger.checkpointing.load_model set, load the parameters of the checkpoint logger.checkpointing.load_args
    names into `arena` (parameters only, as the reference restores them).  Returns whether it loaded; the caller then refreshes
    whatever is derived from the arena (a bf16 shadow, target networks)."""
    if not config.logger.checkpointing.load_model:
        return False
    Checkpointer(model_name=config.system.system_name, **to_container(config.logger.checkpointing.load_args)).restore_params(arena)
    return True
