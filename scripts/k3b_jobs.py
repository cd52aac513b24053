"""Per-CTA timeline of K3b (`tc_dw_kernel`) at the benchmark shape, summarised per job class.

Runs the minibatch step of `scripts/time_k3.py` (E=4096, T=128, D=64, A=8, mb=32768; K3a -> K3b -> reduce -> K4 chained with
programmatic dependent launch) and reads K3b's per-CTA profile record (`stx_tc_debug_set_prof_buffer`, layout in include/stx.h)
after the last of `--steps` back-to-back steps, `--reps` times.  Per job class (dW1 half 0 / 1, dW2, dW0, per network) it prints:
  start / end    globaltimer after `griddepcontrol.wait` and at exit, relative to the first CTA's start (us);
  busy           end - start (us), i.e. the CTA's own work without the wait for K3a.

    python scripts/k3b_jobs.py --out /tmp/k3b_jobs.json
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import time_k3  # noqa: E402  (sys.path: the shapes and the step come from there)

KINDS = ("dW1 half 0", "dW1 half 1", "dW2", "dW0")
NETS = ("actor", "critic")


def _med(xs):
    return round(statistics.median(xs), 2) if xs else None


def collect(steps: int, reps: int) -> dict:
    import torch

    from stoix_b200 import _lib

    if not torch.cuda.is_available():
        raise SystemExit("k3b_jobs.py measures on a CUDA device; none is visible")
    step, _ = time_k3._setup()
    for i in range(2 * 16):
        step(i)
    torch.cuda.synchronize()
    lib = _lib.load()
    buf = torch.zeros(132 * 8, dtype=torch.int64, device="cuda")
    _lib.check(lib.stx_tc_debug_set_prof_buffer(buf.data_ptr()), "stx_tc_debug_set_prof_buffer")
    records = []
    try:
        for _ in range(reps):
            for i in range(steps):
                step(i)
            torch.cuda.synchronize()
            records.append(buf.view(132, 8).cpu().tolist())
    finally:
        _lib.check(lib.stx_tc_debug_set_prof_buffer(None), "stx_tc_debug_set_prof_buffer")
    return summarise(records)


def summarise(records) -> dict:
    """records: [rep][cta][8] as in include/stx.h."""
    per = {}
    last_finisher = {}
    spans, mhz = [], []
    for rec in records:
        k3b = [r for r in rec if r[0] >= 2]
        t0 = min(r[3] for r in k3b)
        t_end = max(r[4] for r in k3b)
        spans.append((t_end - t0) / 1e3)
        for r in k3b:
            j = r[0] - 2
            key = f"{NETS[j // 4]} {KINDS[j % 4]}"
            d = per.setdefault(key, {"chunks": [], "start": [], "end": [], "busy": []})
            d["chunks"].append(r[5])
            d["start"].append((r[3] - t0) / 1e3)
            d["end"].append((r[4] - t0) / 1e3)
            d["busy"].append((r[4] - r[3]) / 1e3)
            if r[4] > r[3]:
                mhz.append((r[1] - r[2]) / (r[4] - r[3]) * 1e3)
        last = max(k3b, key=lambda r: r[4])
        key = f"{NETS[(last[0] - 2) // 4]} {KINDS[(last[0] - 2) % 4]}"
        last_finisher[key] = last_finisher.get(key, 0) + 1
    n_rep = len(records)
    classes = {}
    for key, d in per.items():
        classes[key] = {"ctas": len(d["chunks"]) // n_rep, "chunks_median": _med(d["chunks"]), "start_us_median": _med(d["start"]),
                        "busy_us_median": _med(d["busy"]), "busy_us_max": round(max(d["busy"]), 2),
                        "end_us_median": _med(d["end"]), "end_us_max": round(max(d["end"]), 2)}
    return {"reps": n_rep, "k3b_span_us_median": _med(spans), "sm_clock_mhz_median": _med(mhz), "last_finisher": last_finisher,
            "classes": classes}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="JSON output path")
    ap.add_argument("--steps", type=int, default=16, help="back-to-back minibatch steps per sample (the last one is recorded)")
    ap.add_argument("--reps", type=int, default=32, help="samples")
    args = ap.parse_args()
    res = {"gpu": time_k3._gpu_info(), "shape": {"E": time_k3.E, "T": time_k3.T, "D": time_k3.D, "A": time_k3.A, "mb": time_k3.MB}}
    res.update(collect(args.steps, args.reps))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    cols = ("ctas", "chunks_median", "start_us_median", "busy_us_median", "busy_us_max", "end_us_median", "end_us_max")
    print(f"K3b span {res['k3b_span_us_median']} us (median of {res['reps']}), SM clock ~{res['sm_clock_mhz_median']} MHz, "
          f"last finisher {res['last_finisher']}")
    print("class".ljust(20) + " ".join(c.replace("_median", "").rjust(14) for c in cols))
    for key in sorted(res["classes"]):
        c = res["classes"][key]
        print(key.ljust(20) + " ".join(str(c[k]).rjust(14) for k in cols))


if __name__ == "__main__":
    main()
