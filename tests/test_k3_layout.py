"""CPU checks of the K3 data layout: the h2 sign-mask fragment order shared by K3a (writer) and K3b (reader), what K3b's
launch plan does at the minibatches the GPU tests run, and the byte and FLOP accounting of scripts/time_k3.py."""
import importlib.util
import os

import numpy as np

from tests import exact_data as X

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# K3b's launch plan (stx_tc_ppo.cu kDwCtasW1 / W2 / W0, kCtaPerNet, kDwStages): split-K CTAs of each job of one network
# (dW1 runs as two row halves) and the stages of each job's input ring
DW_CTAS = {"dW1 half": 19, "dW2": 13, "dW0": 15}
DW_JOBS = ("dW1 half", "dW1 half", "dW2", "dW0")
CTA_PER_NET = 66
DW_STAGES = 4


def _time_k3():
    spec = importlib.util.spec_from_file_location("time_k3", os.path.join(ROOT, "scripts", "time_k3.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _fragment(t, h, i, e):
    """(row, column) of element e of register a[32 h + i] of thread t in a 64 x 256 warpgroup operand (stx_tc_ptx.cuh)."""
    wq, lane = t // 32, t % 32
    return wq * 16 + lane // 4 + 8 * (i & 1), 128 * h + 8 * (i >> 1) + 2 * (lane % 4) + e


def _mask_pos(t, h, i, e):
    """(thread, word, bit) of stx_tc_ppo.cu: mask_word(h, i) = 2 h + i / 16, mask_bit(i, e) = 2 (i % 16) + e."""
    return t, 2 * h + (i >> 4), 2 * (i & 15) + e


def test_mask_fragment_order_covers_the_tile_once_and_round_trips():
    rng = np.random.default_rng(0)
    h2 = rng.random((64, 256)) < 0.5
    words = np.zeros((128, 4), dtype=np.uint64)  # K3a: thread t writes its 4 words (one uint4) at tile * 128 + t
    seen = set()
    for t in range(128):
        for h in range(2):
            for i in range(32):
                for e in range(2):
                    r, c = _fragment(t, h, i, e)
                    tt, w, b = _mask_pos(t, h, i, e)
                    assert b < 32 and (tt, w, b) not in seen
                    seen.add((tt, w, b))
                    words[tt, w] |= np.uint64(int(h2[r, c]) << b)
    assert len(seen) == 64 * 256
    # K3b: thread t of the rebuild warpgroup reads word t, decodes with the same mapping and masks the same (row, column)
    back = np.zeros_like(h2)
    for t in range(128):
        for h in range(2):
            for i in range(32):
                for e in range(2):
                    r, c = _fragment(t, h, i, e)
                    _, w, b = _mask_pos(t, h, i, e)
                    back[r, c] = (int(words[t, w]) >> b) & 1
    assert (back == h2).all()


def _chunks_per_cta(mb, n_cta):
    """64-row chunks of each CTA of a job: CTA c takes chunks c, c + n_cta, ... (my_chunks of tc_dw_kernel)."""
    chunks = mb // 64
    return [(chunks - c + n_cta - 1) // n_cta if c < chunks else 0 for c in range(n_cta)]


def test_k3b_plan_at_the_dispatch_minibatches():
    """The two minibatches of test_tc_exact_gpu.py's dispatch cases reach both ends of K3b's plan: at mb = 128 most CTAs
    have no chunk, and at the benchmark minibatch every CTA of every job runs more chunks than its ring has stages, so
    every ring wraps."""
    assert sum(DW_CTAS[j] for j in DW_JOBS) == CTA_PER_NET
    tk = _time_k3()
    assert tk.DW_SPLIT == (DW_CTAS["dW1 half"], DW_CTAS["dW2"], DW_CTAS["dW0"])
    small, bench = X.CRITIC_CASES[0][2], X.CRITIC_CASES[3][2]
    assert small == 128 and bench == tk.MB
    idle = sum(n == 0 for j in DW_JOBS for n in _chunks_per_cta(small, DW_CTAS[j]))
    assert 2 * idle > CTA_PER_NET, f"mb = {small}: {idle} of {CTA_PER_NET} CTAs idle"
    for j in DW_JOBS:
        assert min(_chunks_per_cta(bench, DW_CTAS[j])) > DW_STAGES, f"mb = {bench}: a {j} CTA does not wrap its ring"


def test_time_k3_accounting_matches_the_layouts():
    acc = _time_k3().k3_accounting
    stored, rebuilt = acc(rebuild=False), acc(rebuild=True)
    mb = 32768
    # stored layout: K3a writes h1, h2, dh1, dh2 (512 B), dz (32 B) per net and x (128 B) once; K3b reads 2720 B per row and net
    assert stored["tc_ppo_fwd_bwd_kernel"]["activation_write_bytes"] == mb * (2 * (4 * 512 + 32) + 128)
    assert stored["tc_dw_kernel"]["activation_read_bytes"] == mb * 2 * (2 * (512 + 256) + (512 + 32) + (512 + 128))
    # rebuild: h1 and dh2 leave the activation stream, the 32 B mask joins it; each dW1 half-job reads x, dz and the mask
    assert rebuilt["tc_ppo_fwd_bwd_kernel"]["activation_write_bytes"] == mb * (2 * (2 * 512 + 32 + 32) + 128)
    assert rebuilt["tc_dw_kernel"]["activation_read_bytes"] == mb * 2 * (2 * (128 + 32 + 32) + (512 + 32) + (512 + 128))
    # dW1 operand rebuild per half-job: h1 half (K 64, N 128) and dh2 (K 16, N 256) per row
    extra = rebuilt["tc_dw_kernel"]["flop"] - stored["tc_dw_kernel"]["flop"]
    assert extra == mb * 2 * 2 * 2 * (64 * 128 + 16 * 256)
    assert rebuilt["tc_ppo_fwd_bwd_kernel"]["flop"] == stored["tc_ppo_fwd_bwd_kernel"]["flop"]
