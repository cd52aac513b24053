"""Tiny driver for ncu: runs the GAE kernel a few times at one shape / block shape."""
import sys

import torch

sys.path.insert(0, ".")
from stoix_b200 import _lib, ops  # noqa: E402

T, E, quads = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
dev = torch.device("cuda:0")
r, v, b = (torch.randn(T, E, device=dev) for _ in range(3))
d = torch.rand(T, E, device=dev) < 0.005
tr = (~d) & (torch.rand(T, E, device=dev) < 0.002)
adv, tgt = torch.empty_like(r), torch.empty_like(r)
_lib.check(_lib.load().stx_gae_set_tuning(quads), f"stx_gae_set_tuning({quads})")
for _ in range(3):
    ops.gae_ppo(r, v, b, d, tr, 0.99, 0.95, 1.0, 1, out=(adv, tgt))
torch.cuda.synchronize()
