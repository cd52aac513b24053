"""GAE micro-benchmark: algorithmic 22 B/element vs measured HBM peak (SURVEY 8d).
Times the kernel alone with CUDA events on the launching stream, L2 flushed between iterations."""
import json
import sys
import time

import torch

sys.path.insert(0, ".")
from stoix_b200 import _lib, ops  # noqa: E402


def bench(T, E, quads=0, iters=20, flush=True):
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    r = torch.randn(T, E, device=dev, generator=g)
    v = torch.randn(T, E, device=dev, generator=g)
    b = torch.randn(T, E, device=dev, generator=g)
    d = torch.rand(T, E, device=dev, generator=g) < 0.005
    tr = (~d) & (torch.rand(T, E, device=dev, generator=g) < 0.002)
    adv, tgt = torch.empty_like(r), torch.empty_like(r)
    flush_buf = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    _lib.check(_lib.load().stx_gae_set_tuning(quads), f"stx_gae_set_tuning({quads})")
    for _ in range(3):
        ops.gae_ppo(r, v, b, d, tr, 0.99, 0.95, 1.0, 1, out=(adv, tgt))
    times = []
    for _ in range(iters):
        if flush:
            flush_buf.fill_(1)
        # traffic >> L2 (50 MB): several launches per event pair, so that the pair times the GPU and not the Python call that
        # precedes the first launch on an idle queue (~50 us); smaller shapes: one launch per pair (L2 flushed in between)
        reps = 5 if 22.0 * T * E > 1e9 else 1
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(reps):
            ops.gae_ppo(r, v, b, d, tr, 0.99, 0.95, 1.0, 1, out=(adv, tgt))
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e) * 1e-3 / reps)
    _lib.load().stx_gae_set_tuning(0)
    times.sort()
    med = times[len(times) // 2]
    return {"T": T, "E": E, "quads": quads, "flush": flush, "us_median": med * 1e6, "us_min": times[0] * 1e6,
            "GBps_median": 22.0 * T * E / med / 1e9, "GBps_best": 22.0 * T * E / times[0] / 1e9}


if __name__ == "__main__":
    out = []
    for (T, E) in [(128, 4096), (128, 32768), (128, 65536), (128, 262144), (128, 1048576), (256, 524288), (128, 4194304)]:
        for q in (0, 500, 501, 416):   # 0 = the shipped heuristic, 500 / 501 = TMA-pipelined 32x128 / 64x64 tiles, 416 = 2 x 512 threads
            for fl in (True,):
                out.append(bench(T, E, q, flush=fl))
                print(json.dumps(out[-1]), flush=True)
