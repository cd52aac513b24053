"""CPU checks of the exact-data generator (tests/exact_data.py) that the bf16 tensor-core tests rest on.

1. At every shape tests/test_tc_exact_gpu.py runs, the data is exact: the bf16-operand oracle equals the unrounded fp64
   oracle bit for bit, every rounded intermediate is a bf16-exact multiple of its grid and every accumulation stays
   below 2^20 grid units (so any summation order gives the same bits).
2. On that data an exact comparison sees the minibatch faults that the norm-wise 5e-3 bound of tests/test_tc_gpu.py
   lets through."""
import numpy as np
import pytest

from tests import exact_data as X


@pytest.mark.parametrize("M,D,A", X.FORWARD_CASES)
def test_forward_data_is_exact(M, D, A):
    net, x = X.forward_problem(M, D, A)
    bounds = X.check_forward(net, x[:8192])
    print(f"M={M} D={D} A={A}: {bounds}")


@pytest.mark.parametrize("B,mb_off,mb,D,A,use_perm", X.CRITIC_CASES)
def test_critic_data_is_exact(B, mb_off, mb, D, A, use_perm):
    pb = X.critic_problem(B, mb_off, mb, D, A, use_perm)
    acc = X.check_ppo(pb, mb_off, mb)
    print(f"B={B} mb={mb} D={D}: largest accumulations (grid units): " + ", ".join(f"{k} {v:.0f}" for k, v in acc.items()))
    g, _ = X.ppo_oracle(pb, mb_off, mb)
    na = X.arena_layout(D, A)[0]
    assert not g[:na].any(), "advantages 0 and ent_coef 0 must give an actor gradient of exactly zero"


@pytest.mark.parametrize("B,mb_off,mb,D,A", X.HOT_CASES)
def test_hot_row_data_keeps_the_critic_exact(B, mb_off, mb, D, A):
    pb = X.hot_problem(B, mb_off, mb, D, A)
    X.check_ppo(pb, mb_off, mb)
    assert (pb.adv[pb.rows(mb_off, mb)] != 0).sum() == len(X.hot_positions(mb))


def test_stale_workspace_data_is_exact():
    B, D, A, windows = X.STALE_CASE
    pb = X.ppo_problem(B, D, A, windows, seed=B + D)
    for mb_off, mb in windows:
        X.check_ppo(pb, mb_off, mb)


def _per_tensor(g, ref, D, A):
    """{name: (norm-wise relative error, number of differing entries)} over the critic tensors of the flat arena."""
    _, coff, _, _ = X.arena_layout(D, A)
    out, o = {}, coff
    for i, (n_in, n_out) in enumerate(((D, 256), (256, 256), (256, 1))):
        for nm, n in ((f"dW{i}", n_in * n_out), (f"db{i}", n_out)):
            a, b = g[o:o + n], ref[o:o + n]
            out[nm] = (np.linalg.norm(a - b) / np.linalg.norm(b), int((a != b).sum()))
            o += n
    return out


def test_exact_comparison_sees_minibatch_faults():
    """The benchmark's minibatch shape (B = 524352, mb = 32768, D = 64).  Each fault below changes what K3 would sum; the
    faulty critic gradient is compared with the true one per tensor.  Exact comparison flags every fault in every weight
    gradient; the norm-wise 5e-3 bound of the tolerance-based tests does not.  Measured on this data (norm-wise
    relative error per tensor):

        fault                                     dW0      dW1      dW2      db2
        one row dropped                           2.6e-3   2.9e-3   2.8e-3   8.4e-3
        obs of two rows swapped (gather fault)    2.9e-2   3.3e-2   2.5e-2   0
        permutation entry swapped with a row of   4.3e-3   5.2e-3   6.0e-3   2.5e-2
          another minibatch
        one 64-row tile dropped                   4.3e-2   3.6e-2   3.7e-2   1.0e-1
        tile 100 read in place of tile 101        6.2e-2   6.4e-2   7.2e-2   1.9e-1

    A K3b job or a reduce segment is one tensor: a fault that drops or re-reads one row there changes that tensor alone, by
    less than 5e-3."""
    B, mb_off, mb, D, A = 524352, 5 * 32768, 32768, 64, 8
    pb = X.ppo_problem(B, D, A, [(mb_off, mb), (mb_off + mb, mb)], seed=7)
    idx = pb.rows(mb_off, mb)
    ref, _ = X.ppo_oracle(pb, mb_off, mb)
    swapped_obs = idx.copy()
    swapped_obs[[100, 30000]] = swapped_obs[[30000, 100]]
    other = idx.copy()
    other[4321] = pb.perm[mb_off + mb + 5]
    faults = {
        "one row dropped": dict(rows=np.delete(idx, 777)),
        "obs of two rows swapped": dict(obs_rows=swapped_obs),
        "row of another minibatch": dict(rows=other),
        "one 64-row tile dropped": dict(rows=np.r_[idx[:64 * 100], idx[64 * 101:]]),
        "tile 100 read in place of tile 101": dict(rows=np.r_[idx[:64 * 101], idx[64 * 100:64 * 101], idx[64 * 102:]]),
    }
    per_fault = {}
    for label, kw in faults.items():
        g, _ = X.ppo_oracle(pb, mb_off, mb, **kw)
        per = _per_tensor(g, ref, D, A)
        worst = max(e for e, _ in per.values())
        n_diff = sum(n for _, n in per.values())
        print(f"{label:36s} worst norm-wise {worst:.1e}, entries that differ {n_diff}: "
              + ", ".join(f"{k} {e:.1e}" for k, (e, _) in per.items()))
        assert n_diff > 0, f"{label}: the exact comparison must see the fault"
        per_fault[label] = per
    for k in ("dW0", "dW1", "dW2"):
        err, n_diff = per_fault["one row dropped"][k]
        assert n_diff > 0 and err < 5e-3, f"{k}: a dropped row changes {n_diff} entries, norm-wise {err:.1e}"
