#!/usr/bin/env python3
"""Measures a block's anonymous-transfer state updates (zk_balances_anonymous_block) and prints one JSON line:
  - the card's name and power limit, read in this run;
  - transfers/s at each --sizes block over --accounts accounts with a skewed ring-member choice, device-resident (the
    _device form on torch buffers) and from host buffers (the host form with its copies), wall clock around calls that
    end in a stream synchronise, median of --reps;
  - the C oracle's sequential loop on one host core over the same block, and whether every output of both forms equals
    the C oracle's;
  - block import against verification alone, alternated in one process, median of --reps, on an --import-tx block whose
    every transfer carries a valid proof of a toy key of the anonymous shape (52 points, 104 public inputs: the verifier
    does the same work per proof as with the real key): import_anonymous_block (one upload; state, verifier inputs,
    verdicts and final state on the device; one download) and verify_proofs_with_points_device alone on the same points,
    resident on the device; the verdicts and the imported state are checked against the C oracle inside the run.
With --issue-frac f > 0, that fraction of each block is issue calls (zk_anonymous_calls_block and its _device form,
against the C oracle of both calls), and the import block mixes issues proven with a toy key of the confidential shape
(11 points) into the transfers: import_anonymous_calls_block against verifying all of the block's proofs alone.
Blocks come from tests/jubjub_oracle/anon_corpus.py and anon_issue_corpus.py; nothing is written to the repository."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import coracle as co                           # noqa: E402
from tests.jubjub_oracle import anon_coracle as aco        # noqa: E402
from tests.jubjub_oracle import anon_corpus                # noqa: E402
from tests.jubjub_oracle import anon_issue_coracle as aic  # noqa: E402
from tests.jubjub_oracle import anon_issue_corpus          # noqa: E402
from zero_chain_b200 import groth16 as zk                  # noqa: E402
from zero_chain_b200 import synthetic as sy                # noqa: E402


def log(*a):
    print(*a, file=sys.stderr, flush=True)                 # progress: the proving and the C oracle take minutes


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], text=True)
        name, power = [s.strip() for s in out.strip().split("\n")[0].split(",")]
        return name, power
    except Exception as e:                                 # the numbers are still printed, with the reason
        return "unknown (%s)" % e, "unknown"


def toy_key(ctx, n_pts, seed):
    r1cs = sy.make_r1cs(60 + 2 * n_pts, 2 * n_pts + 1, 50, 40, 33, seed=seed)
    crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=seed + 1)
    return r1cs, zk.Parameters.read(ctx, crs.params_bytes, checked=True), zk.PreparedVerifyingKey.prepare(ctx, crs.params_bytes)


def prove_all(ctx, r1cs, params, points, n_pts):
    """one valid proof per row of n_pts point encodings"""
    n = len(points) // (32 * n_pts)
    xy, st = zk.jubjub_into_xy(ctx, points)
    assert not st.any()
    limbs = xy.reshape(n, 2 * n_pts, 4).astype(object)
    proofs = bytearray()
    for k0 in range(0, n, 256):
        provers = []
        for k in range(k0, min(k0 + 256, n)):
            ins = [int(l[0]) | int(l[1]) << 64 | int(l[2]) << 128 | int(l[3]) << 192 for l in limbs[k]]
            z = sy.make_witness(r1cs, k + 1, inputs=ins)
            av, bv, cv = sy.evaluate(r1cs, z)
            provers.append(zk.ProvingAssignment(co.ints_to_limbs(av, 4), co.ints_to_limbs(bv, 4), co.ints_to_limbs(cv, 4),
                                                co.ints_to_limbs(z[:r1cs.n_inputs], 4), co.ints_to_limbs(z[r1cs.n_inputs:], 4),
                                                *sy.densities(r1cs)))
        proofs += zk.create_proof_batch(provers, params, [11 + k for k in range(k0, k0 + len(provers))],
                                        [13 + k for k in range(k0, k0 + len(provers))])
        log("proved", len(proofs) // 192, "of", n)
    return np.frombuffer(bytes(proofs), np.uint8).reshape(n, 192)


def import_block(ctx, n, n_acct, reps, issue_frac=0.0):
    """block import (state + verifier inputs + proofs) against verification alone on a block of n proven transactions"""
    if issue_frac > 0:
        return import_calls_block(ctx, n, n_acct, reps, issue_frac)
    import torch
    n_pts = zk.ANONYMOUS_POINTS
    r1cs, params, pvk = toy_key(ctx, n_pts, 5)
    blk = anon_corpus.make(n_acct, n, 7 + n, skew=1.0, mask_p=(0.0, 1.0, 0.0, 0.0, 0.0))
    # every proof is made on the points its transaction's verifier reads
    _, want0 = aco.block(*blk.args()[:-1], bytes(n))
    points = want0[1]
    proofs = prove_all(ctx, r1cs, params, points, n_pts).tobytes()
    params.free()
    m = blk.members.reshape(n, 12)
    txs = [zk.AnonymousTx(m[k].tolist(), [blk.tx_points[416 * k + 32 * i:416 * k + 32 * i + 32] for i in range(12)],
                          blk.tx_points[416 * k + 384:416 * k + 416], blk.tx_extra[64 * k:64 * k + 32], blk.tx_extra[64 * k + 32:64 * k + 64])
           for k in range(n)]
    accounts = (blk.keys, blk.balances, blk.pendings, blk.flags)
    d_proofs = torch.from_numpy(np.frombuffer(proofs, np.uint8).copy()).cuda()
    d_points = torch.from_numpy(np.frombuffer(points, np.uint8).copy()).cuda()
    d_verdicts = torch.zeros(n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    run_import = lambda: zk.import_anonymous_block(ctx, pvk, accounts, txs, blk.g_epoch, proofs)
    run_verify = lambda: (zk.verify_proofs_with_points_device(pvk, n, d_proofs.data_ptr(), d_points.data_ptr(), n_pts, d_verdicts.data_ptr()),
                          ctx.sync())
    verdicts, state, enc_balances = run_import()
    run_verify()
    _, want = aco.block(*blk.args()[:-1], bytes([1]) * n)
    ok = (verdicts == [1] * n and d_verdicts.cpu().numpy().tolist() == [1] * n and state == want[3:] and enc_balances == want0[0])
    ti, tv = [], []
    for _ in range(reps):                                   # alternated
        t0 = time.perf_counter(); run_import(); ti.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); run_verify(); tv.append(time.perf_counter() - t0)
    pvk.free()
    return {"transfers": n, "accounts": n_acct, "import_ms": 1e3 * float(np.median(ti)), "import_tx_per_s": n / float(np.median(ti)),
            "verify_only_ms": 1e3 * float(np.median(tv)), "verify_only_tx_per_s": n / float(np.median(tv)),
            "import_over_verify": float(np.median(ti) / np.median(tv)), "verdicts_state_equal_c_oracle": bool(ok)}


def import_calls_block(ctx, n, n_acct, reps, issue_frac):
    """import_anonymous_calls_block on a block of n transactions, issue_frac of them issues, every proof valid, against
    verify_proofs_with_points_device alone on the same rows (issues with the confidential key, transfers with the
    anonymous one), resident on the device"""
    import torch
    anon_r1cs, anon_params, anon_pvk = toy_key(ctx, zk.ANONYMOUS_POINTS, 5)
    conf_r1cs, conf_params, conf_pvk = toy_key(ctx, zk.CONFIDENTIAL_POINTS, 8)
    blk = anon_issue_corpus.make(n_acct, n, 7 + n, issue_frac=issue_frac, free=0, skew=1.0, mask_p=(0.0, 1.0, 0.0, 0.0, 0.0))
    kind = np.frombuffer(blk.kind, np.uint8)
    m = blk.members.reshape(n, 12)
    tp, tx = blk.tx_points, blk.tx_extra
    txs = []
    for k in range(n):
        lefts = [tp[416 * k + 32 * i:416 * k + 32 * i + 32] for i in range(12)]
        if kind[k] == zk.ANON_ISSUE:
            txs.append(zk.AnonIssueTx(int(m[k, 0]), lefts[0], lefts[6], lefts[4] + lefts[5], tp[416 * k + 384:416 * k + 416],
                                      tx[64 * k:64 * k + 32], tx[64 * k + 32:64 * k + 64]))
        else:
            txs.append(zk.AnonymousTx(m[k].tolist(), lefts, tp[416 * k + 384:416 * k + 416], tx[64 * k:64 * k + 32], tx[64 * k + 32:64 * k + 64]))
    iss, tr = np.flatnonzero(kind == 1), np.flatnonzero(kind == 0)
    # every issue passes, so the transfers' rows are the oracle's with every issue applied
    _, want0 = aic.block(*blk.args()[:-1], kind.tobytes())
    iss_points = b"".join(txs[k].verify_points(blk.keys, blk.g_epoch) for k in iss.tolist())
    tr_points = np.frombuffer(want0[1], np.uint8).reshape(n, -1)[tr].tobytes()
    proofs = np.zeros((n, 192), np.uint8)
    proofs[iss] = prove_all(ctx, conf_r1cs, conf_params, iss_points, zk.CONFIDENTIAL_POINTS)
    proofs[tr] = prove_all(ctx, anon_r1cs, anon_params, tr_points, zk.ANONYMOUS_POINTS)
    anon_params.free(); conf_params.free()
    accounts = (blk.keys, blk.balances, blk.pendings, blk.flags)
    dv = lambda b: torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()
    d_pi, d_ti, d_pt, d_tt = dv(proofs[iss].tobytes()), dv(iss_points), dv(proofs[tr].tobytes()), dv(tr_points)
    d_verdicts = torch.zeros(n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    run_import = lambda: zk.import_anonymous_calls_block(ctx, anon_pvk, conf_pvk, accounts, txs, blk.g_epoch, proofs.tobytes())
    run_verify = lambda: (zk.verify_proofs_with_points_device(conf_pvk, len(iss), d_pi.data_ptr(), d_ti.data_ptr(), zk.CONFIDENTIAL_POINTS,
                                                              d_verdicts.data_ptr()),
                          zk.verify_proofs_with_points_device(anon_pvk, len(tr), d_pt.data_ptr(), d_tt.data_ptr(), zk.ANONYMOUS_POINTS,
                                                              d_verdicts.data_ptr() + len(iss)),
                          ctx.sync())
    verdicts, state, enc_balances, issued = run_import()
    run_verify()
    _, want = aic.block(*blk.args()[:-1], bytes([1]) * n)
    ok = (verdicts == [1] * n and d_verdicts.cpu().numpy().tolist() == [1] * n and state == want[4:] and enc_balances == want[0]
          and b"".join(c if c is not None else bytes(64) for c in issued) == want[2])
    ti, tv = [], []
    for _ in range(reps):                                   # alternated
        t0 = time.perf_counter(); run_import(); ti.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); run_verify(); tv.append(time.perf_counter() - t0)
    anon_pvk.free(); conf_pvk.free()
    return {"transactions": n, "issues": int(len(iss)), "accounts": n_acct, "import_ms": 1e3 * float(np.median(ti)),
            "import_tx_per_s": n / float(np.median(ti)), "verify_only_ms": 1e3 * float(np.median(tv)),
            "verify_only_tx_per_s": n / float(np.median(tv)), "import_over_verify": float(np.median(ti) / np.median(tv)),
            "verdicts_state_issued_equal_c_oracle": bool(ok)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1024,8192")
    ap.add_argument("--accounts", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--import-tx", type=int, default=256)
    ap.add_argument("--import-accounts", type=int, default=1024)
    ap.add_argument("--issue-frac", type=float, default=0.0)
    ap.add_argument("--no-import", action="store_true")
    a = ap.parse_args()
    import torch
    name, power = card()
    ctx = zk.Context(0)
    aco.lib()                                               # the C oracle is compiled before anything is timed
    res = {"card": name, "power_limit": power, "accounts": a.accounts, "issue_frac": a.issue_frac, "sizes": {}}
    f = a.issue_frac
    dev = lambda b: torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()
    na = a.accounts
    for n in [int(x) for x in a.sizes.split(",")]:
        blk = (anon_issue_corpus.make(na, n, 100 + n, issue_frac=f, free=0, skew=1.0, bad_points=16) if f > 0
               else anon_corpus.make(na, n, 100 + n, skew=1.0, bad_points=16))
        t0 = time.perf_counter()
        bad, want = aic.block(*blk.args()) if f > 0 else aco.block(*blk.args())
        host_loop = time.perf_counter() - t0
        assert bad is None
        log("C oracle:", n, "transfers in %.1f s" % host_loop)
        ins = [dev(blk.keys), dev(blk.balances), dev(blk.pendings), dev(blk.flags)]
        mem = torch.from_numpy(blk.members.astype(np.uint32).view(np.int32)).cuda()
        txi = [dev(blk.tx_points), dev(blk.tx_extra), dev(blk.g_epoch), dev(blk.applied)]
        sizes = (768 * n, 1664 * n, 64 * n, n, 64 * na, 64 * na, na) if f > 0 else (768 * n, 1664 * n, n, 64 * na, 64 * na, na)
        outs = [torch.zeros(k, dtype=torch.uint8, device="cuda") for k in sizes]
        torch.cuda.synchronize()
        pi, pt, po = [t.data_ptr() for t in ins], [t.data_ptr() for t in txi], [t.data_ptr() for t in outs]
        if f > 0:
            d_kind = dev(blk.kind)
            run_dev = lambda: (zk.anonymous_calls_block_device(ctx, na, *pi, n, d_kind.data_ptr(), mem.data_ptr(), *pt, *po), ctx.sync())
            run_host = lambda: zk.anonymous_calls_block(ctx, *blk.args())
        else:
            run_dev = lambda: (zk.anonymous_block_device(ctx, na, *pi, n, mem.data_ptr(), *pt, *po), ctx.sync())
            run_host = lambda: zk.anonymous_block(ctx, *blk.args())
        run_dev(); run_host()                               # warm-up: workspace, modules
        td, th = [], []
        for _ in range(a.reps):                             # the two forms alternate
            torch.cuda.synchronize()
            t0 = time.perf_counter(); run_dev(); td.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); got_h = run_host(); th.append(time.perf_counter() - t0)
        got_d = tuple(t.cpu().numpy().tobytes() for t in outs)
        st = np.frombuffer(want[3 if f > 0 else 2], np.uint8)
        res["sizes"][str(n)] = {
            "device_resident_tx_per_s": n / float(np.median(td)), "device_resident_ms": 1e3 * float(np.median(td)),
            "host_buffers_tx_per_s": n / float(np.median(th)), "host_buffers_ms": 1e3 * float(np.median(th)),
            "c_oracle_one_core_tx_per_s": n / host_loop, "c_oracle_one_core_s": host_loop,
            "most_rings_of_one_account": int(np.bincount(blk.members).max()), "applied": int((st == 0).sum()),
            "host_form_equals_c_oracle": got_h == want, "device_form_equals_c_oracle": got_d == want,
        }
    if not a.no_import:
        res["import"] = import_block(ctx, a.import_tx, a.import_accounts, a.reps, f)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
