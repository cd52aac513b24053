"""Bit-level reference of the fp32 PPO loss paths: every minibatch entry, head-grad entry, value face and KL face.

Seeded NumPy inputs (B = 6144 batch rows, D = 24); each entry runs on the minibatch windows of WINDOWS: a multi-block mb = 4096 and a
ragged mb = 1000, each read through a permutation and as a contiguous row range, with advantage standardisation on.  logp_old is the
current policy's log-prob plus noise, so the ratios fall on both sides of the clip band and every DPO branch occurs (A >= 0 and
A < 0, drift argument above and below 0); the stored tanh-Normal actions include both clipped tails.  Recorded per call: the
SHA-256 of every output (gradient arena, d_head, metrics, eps_out, face outputs), the stx_launch_count() delta, and a seeded
sample of each output's values for diagnosing a mismatch.

These paths are deterministic (fixed-order partials), so the hashes pin every float expression and every summation order.
Generate on an H100 with the build the reference should describe:

    python tests/golden/make_fp32_ppo_reference.py tests/golden/fp32_ppo_reference.json
"""
from __future__ import annotations

import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

B, D, H = 6144, 24, 64
A_CONT = 6                 # tanh-Normal action dims (not a multiple of the 4-wide noise draw)
LO, HI = -1.0, 1.0
WINDOWS = ((0, 4096, True), (1024, 4096, False), (777, 1000, True), (5000, 1000, False))  # (mb_off, mb, permuted)
N_SAMPLE = 64
SEED, OFFSET, COUNTER = 0x9E3779B97F4A7C15, 3, 11  # entropy-noise key of the tanh-Normal entries


def _digest(t) -> dict:
    a = t.detach().cpu().contiguous().numpy()
    flat = a.reshape(-1).view(np.uint32)
    pick = np.random.default_rng(flat.size).choice(flat.size, min(N_SAMPLE, flat.size), replace=False)
    return {"sha256": hashlib.sha256(a.tobytes()).hexdigest(), "sample_index": pick.tolist(), "sample_f32_hex": flat[pick].tobytes().hex()}


def run_all() -> dict:
    """Runs every case on cuda:0 with the library in this tree; returns the record make_fp32_ppo_reference writes."""
    import torch

    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from stoix_b200 import _lib, ops

    dev = torch.device("cuda:0")
    lib = _lib.load()
    rng = np.random.default_rng(20261016)
    T = lambda x, dt=torch.float32: torch.tensor(np.ascontiguousarray(x), dtype=dt, device=dev)
    noise = lambda n: rng.normal(0.0, 0.35, n)
    cases = []

    def record(name, fn, outputs):
        torch.cuda.synchronize()
        l0 = lib.stx_launch_count()
        fn()
        torch.cuda.synchronize()
        cases.append({"name": name, "launches": int(lib.stx_launch_count() - l0), "outputs": {k: _digest(v) for k, v in outputs().items()}})

    obs = rng.standard_normal((B, D)).astype(np.float32)
    adv = (rng.standard_normal(B) * 1.5 + 0.3).astype(np.float32)
    adv_stats = np.array([adv.astype(np.float64).mean(), 1.0 / adv.astype(np.float64).std()], np.float32)
    value = rng.standard_normal(B).astype(np.float32)
    targets = (value + rng.normal(0.0, 0.5, B)).astype(np.float32)
    perm = rng.permutation(B).astype(np.int32)
    obs_t, perm_t = T(obs), T(perm, torch.int32)

    def arena(sa, sc):
        total = ops.arena_offsets(sa, sc)[2]
        return T(rng.standard_normal(total) * 0.15), total

    def rows(mb_off, mb, permuted):
        return perm[mb_off:mb_off + mb] if permuted else np.arange(mb_off, mb_off + mb)

    def logp_old_for(logp_rows, idx):  # batch-wide logp_old whose window rows are the current log-probs plus noise
        out = rng.normal(-2.0, 0.5, B).astype(np.float32)
        out[idx] = (logp_rows + noise(idx.size)).astype(np.float32)
        return out

    def cat_logp(logits, act):
        z = logits.astype(np.float64)
        lse = np.log(np.exp(z - z.max(1, keepdims=True)).sum(1)) + z.max(1)
        return z[np.arange(z.shape[0]), act] - lse

    def tn_logp(head, act):
        return ops.tanh_normal_log_prob(T(head), T(act), LO, HI).cpu().numpy().astype(np.float64)

    def tn_actions(n, A):
        a = np.tanh(rng.normal(0.0, 0.9, (n, A))).astype(np.float32)
        tail = rng.random((n, A))
        a[tail < 0.04] = LO
        a[tail > 0.96] = HI
        return a

    # ---- ppo_minibatch_grads (fp32): default MLP A = 8, A = 32, LayerNorm + tanh torso, and accumulating into a non-zero arena
    for tag, A, act, ln, accumulate in (("a8", 8, "relu", False, False), ("a32", 32, "relu", False, False), ("ln_tanh", 8, "tanh", True, False),
                                        ("accumulate", 8, "relu", False, True)):
        sa, sc = ops.MlpSpec((D, H, H, A), act, ln), ops.MlpSpec((D, H, H, 1), act, ln)
        params, total = arena(sa, sc)
        action = rng.integers(0, A, B).astype(np.int32)
        for mb_off, mb, permuted in WINDOWS:
            idx = rows(mb_off, mb, permuted)
            logits = ops.mlp_forward(sa, params, obs_t, T(idx, torch.int32)).cpu().numpy()
            batch = ops.PpoBatch(obs_t, T(action, torch.int32), T(logp_old_for(cat_logp(logits, action[idx]), idx)), T(value), T(adv),
                                 T(targets), T(adv_stats), perm_t if permuted else None)
            grads = T(rng.standard_normal(total)) if accumulate else torch.zeros(total, device=dev)
            metrics = T(rng.standard_normal(8)) if accumulate else torch.zeros(8, device=dev)
            ws = ops.ppo_workspace(sa, sc, mb, ops.STX_PREC_F32, dev)
            record(f"ppo_minibatch_grads/{tag}/{mb_off}+{mb}/{'perm' if permuted else 'range'}",
                   lambda: ops.ppo_minibatch_grads(sa, sc, params, batch, mb_off, mb, 0.2, 0.01, 0.5, True, grads, metrics, ws,
                                                   ops.STX_PREC_F32, 0.5 if accumulate else 1.0, overwrite=not accumulate),
                   lambda: {"grads": grads, "metrics": metrics})

    # ---- ppo_head_grads: logits and value of the same rows, one launch each
    A = 7
    action = rng.integers(0, A, B).astype(np.int32)
    for mb_off, mb, permuted in WINDOWS:
        idx = rows(mb_off, mb, permuted)
        logits = rng.normal(0.0, 1.2, (mb, A)).astype(np.float32)
        pred = (value[idx] + rng.normal(0.0, 0.4, mb)).astype(np.float32)   # |v - v_old| on both sides of clip_eps
        lt, vt = T(logits), T(pred)
        dl, dv, metrics = torch.empty_like(lt), torch.empty_like(vt), torch.zeros(8, device=dev)
        idx_t = T(idx, torch.int32) if permuted else None
        lo_t = T(logp_old_for(cat_logp(logits, action[idx]), idx))
        record(f"ppo_head_grads/{mb_off}+{mb}/{'perm' if permuted else 'range'}",
               lambda: ops.ppo_head_grads(lt, vt, idx_t, T(action, torch.int32), lo_t, T(value), T(adv), T(targets), T(adv_stats), 0.2, 0.01,
                                          0.5, dl, dv, metrics, weight=0.5, row0=0 if permuted else mb_off),
               lambda: {"d_logits": dl, "d_value": dv, "metrics": metrics})

    # ---- ppo_penalty_head_grads / ppo_variant_tanh_normal_head_grads / ppo_tanh_normal_head_grads
    behaviour_cat = rng.normal(0.0, 1.2, (B, A)).astype(np.float32)
    act_c = tn_actions(B, A_CONT)
    for mb_off, mb, permuted in WINDOWS:
        idx = rows(mb_off, mb, permuted)
        idx_t, row0 = (T(idx, torch.int32), 0) if permuted else (None, mb_off)
        tag = f"{mb_off}+{mb}/{'perm' if permuted else 'range'}"
        logits = rng.normal(0.0, 1.2, (mb, A)).astype(np.float32)
        beh = behaviour_cat.copy()
        beh[idx] = logits + rng.normal(0.0, 0.3, (mb, A))
        beh[idx[:8]] = logits[:8]                                            # KL = 0 rows
        lt, lo_t = T(logits), T(logp_old_for(cat_logp(logits, action[idx]), idx))
        out = {}
        record(f"ppo_penalty_head_grads/{tag}",
               lambda: out.update(zip(("d_logits", "metrics"), ops.ppo_penalty_head_grads(lt, idx_t, T(beh), T(action, torch.int32), lo_t, T(adv),
                                                                                          T(adv_stats), 3.0, 0.01, weight=0.5, row0=row0))),
               lambda: dict(out))

        head = rng.normal(0.0, 0.7, (mb, 2 * A_CONT)).astype(np.float32)
        beh_c = rng.normal(0.0, 0.7, (B, 2 * A_CONT)).astype(np.float32)
        beh_c[idx] = head + rng.normal(0.0, 0.2, (mb, 2 * A_CONT))
        beh_c[idx[:8]] = head[:8]
        ht, lo_t = T(head), T(logp_old_for(tn_logp(head, act_c[idx]), idx))
        eps_in = T(rng.standard_normal((mb, A_CONT)))
        for noise_tag, eps_kw in (("philox", None), ("eps_in", eps_in)):
            common = dict(seed=SEED, offset=OFFSET, dev_counter=T([COUNTER], torch.int64), weight=0.5, row0=row0)
            out = {"eps_out": torch.zeros(mb, A_CONT, device=dev)} if eps_kw is None else {}
            record(f"ppo_tanh_normal_head_grads/{noise_tag}/{tag}",
                   lambda: out.update(zip(("d_head", "metrics"), ops.ppo_tanh_normal_head_grads(
                       ht, idx_t, T(act_c), lo_t, T(adv), T(adv_stats), 0.2, 0.01, LO, HI, eps_in=eps_kw, eps_out=out.get("eps_out"), **common))),
                   lambda: dict(out))
            for kind, kname in ((ops.STX_PPO_KL_PENALTY, "kl_penalty"), (ops.STX_PPO_DPO, "dpo")):
                out = {"eps_out": torch.zeros(mb, A_CONT, device=dev)} if eps_kw is None else {}
                record(f"ppo_variant_tanh_normal_head_grads/{kname}/{noise_tag}/{tag}",
                       lambda: out.update(zip(("d_head", "metrics"), ops.ppo_variant_tanh_normal_head_grads(
                           ht, idx_t, kind, T(act_c), lo_t, T(adv), T(adv_stats), 0.01, LO, HI,
                           behaviour=T(beh_c) if kind == ops.STX_PPO_KL_PENALTY else None, kl_coef=3.0, eps_in=eps_kw,
                           eps_out=out.get("eps_out"), **common))),
                       lambda: dict(out))

    # ---- ppo_penalty_minibatch_grads, ppo_continuous_minibatch_grads, ppo_variant_continuous_minibatch_grads
    sa, sc = ops.MlpSpec((D, H, H, A)), ops.MlpSpec((D, H, H, 1))
    params, total = arena(sa, sc)
    sa_c, sc_c = ops.MlpSpec((D, H, H, 2 * A_CONT)), ops.MlpSpec((D, H, H, 1))
    params_c, total_c = arena(sa_c, sc_c)
    for mb_off, mb, permuted in WINDOWS:
        idx = rows(mb_off, mb, permuted)
        tag = f"{mb_off}+{mb}/{'perm' if permuted else 'range'}"
        p_t = perm_t if permuted else None
        logits = ops.mlp_forward(sa, params, obs_t, T(idx, torch.int32)).cpu().numpy()
        beh = behaviour_cat.copy()
        beh[idx] = logits + rng.normal(0.0, 0.3, (mb, A))
        batch = ops.PpoBatch(obs_t, T(action, torch.int32), T(logp_old_for(cat_logp(logits, action[idx]), idx)), T(value), T(adv), T(targets),
                             T(adv_stats), p_t)
        grads, metrics, ws = torch.zeros(total, device=dev), torch.zeros(8, device=dev), ops.ppo_workspace(sa, sc, mb, ops.STX_PREC_F32, dev)
        record(f"ppo_penalty_minibatch_grads/{tag}",
               lambda: ops.ppo_penalty_minibatch_grads(sa, sc, params, batch, mb_off, mb, T(beh), 3.0, 0.2, 0.01, 0.5, True, grads, metrics, ws,
                                                       overwrite=True),
               lambda: {"grads": grads, "metrics": metrics})

        head = ops.mlp_forward(sa_c, params_c, obs_t, T(idx, torch.int32)).cpu().numpy()
        beh_c = rng.normal(0.0, 0.7, (B, 2 * A_CONT)).astype(np.float32)
        beh_c[idx] = head + rng.normal(0.0, 0.2, (mb, 2 * A_CONT))
        batch = ops.PpoBatch(obs_t, T(act_c), T(logp_old_for(tn_logp(head, act_c[idx]), idx)), T(value), T(adv), T(targets), T(adv_stats), p_t)
        eps_in = T(rng.standard_normal((mb, A_CONT)))
        for noise_tag, eps_kw in (("philox", None), ("eps_in", eps_in)):
            common = dict(seed=SEED, offset=OFFSET, dev_counter=T([COUNTER], torch.int64))
            eps_out = torch.zeros(mb, A_CONT, device=dev) if eps_kw is None else None
            grads, metrics = T(rng.standard_normal(total_c)), T(rng.standard_normal(8))   # accumulating (overwrite=False)
            ws = ops.ppo_workspace(sa_c, sc_c, mb, ops.STX_PREC_F32, dev)
            outs = lambda: {k: v for k, v in (("grads", grads), ("metrics", metrics), ("eps_out", eps_out)) if v is not None}
            record(f"ppo_continuous_minibatch_grads/{noise_tag}/{tag}",
                   lambda: ops.ppo_continuous_minibatch_grads(sa_c, sc_c, params_c, batch, mb_off, mb, 0.2, 0.01, 0.5, True, grads, metrics, ws,
                                                              LO, HI, eps_in=eps_kw, eps_out=eps_out, grad_weight=0.5, **common),
                   outs)
            for kind, kname in ((ops.STX_PPO_KL_PENALTY, "kl_penalty"), (ops.STX_PPO_DPO, "dpo")):
                eps_out = torch.zeros(mb, A_CONT, device=dev) if eps_kw is None else None
                grads, metrics = torch.zeros(total_c, device=dev), torch.zeros(8, device=dev)
                ws = ops.ppo_workspace(sa_c, sc_c, mb, ops.STX_PREC_F32, dev)
                record(f"ppo_variant_continuous_minibatch_grads/{kname}/{noise_tag}/{tag}",
                       lambda: ops.ppo_variant_continuous_minibatch_grads(
                           sa_c, sc_c, params_c, batch, mb_off, mb, kind, 0.2, 0.01, 0.5, True, grads, metrics, ws, LO, HI,
                           behaviour=T(beh_c) if kind == ops.STX_PPO_KL_PENALTY else None, kl_coef=3.0, eps_in=eps_kw, eps_out=eps_out,
                           overwrite=True, **common),
                       outs)

    # ---- the four value faces (a single block, and more rows than the grid cap covers) and the two KL faces
    for n in (1000, 300000):
        lp = rng.normal(-1.0, 0.5, n).astype(np.float32)
        lp_old, gae = (lp + noise(n)).astype(np.float32), rng.standard_normal(n).astype(np.float32)
        v, v_old = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
        tg, kl = rng.standard_normal(n).astype(np.float32), rng.random(n).astype(np.float32)
        out = {}
        record(f"ppo_clip_loss_value/{n}", lambda: out.update(out=ops.ppo_clip_loss_value(T(lp), T(lp_old), T(gae), 0.2)), lambda: dict(out))
        record(f"clipped_value_loss_value/{n}", lambda: out.update(out=ops.clipped_value_loss_value(T(v), T(v_old), T(tg), 0.2)), lambda: dict(out))
        record(f"ppo_penalty_loss_value/{n}", lambda: out.update(zip(("loss", "kl"), ops.ppo_penalty_loss_value(T(lp), T(lp_old), T(gae), T(kl), 3.0))),
               lambda: dict(out))
        out = {}
        record(f"dpo_loss_value/{n}", lambda: out.update(out=ops.dpo_loss_value(T(lp), T(lp_old), T(gae), 2.0, 0.6)), lambda: dict(out))
    zp, zq = rng.normal(0.0, 1.5, (3000, 7)).astype(np.float32), rng.normal(0.0, 1.5, (3000, 7)).astype(np.float32)
    zq[:10] = zp[:10]
    hp, hq = rng.normal(0.0, 1.0, (3000, 2 * A_CONT)).astype(np.float32), rng.normal(0.0, 1.0, (3000, 2 * A_CONT)).astype(np.float32)
    hq[:10] = hp[:10]
    out = {}
    record("categorical_kl", lambda: out.update(out=ops.categorical_kl(T(zp), T(zq))), lambda: dict(out))
    record("tanh_normal_kl", lambda: out.update(out=ops.tanh_normal_kl(T(hp), T(hq))), lambda: dict(out))
    return {"shape": {"B": B, "D": D, "H": H, "A_cont": A_CONT}, "cases": cases}


if __name__ == "__main__":
    rec = run_all()
    with open(sys.argv[1], "w") as f:
        json.dump(rec, f, indent=0)
    print(json.dumps([{"name": c["name"], "launches": c["launches"]} for c in rec["cases"]]))
