#!/usr/bin/env python3
"""Measures a block's confidential-transfer balance updates (zk_balances_confidential_block) and prints one JSON line:
  - the card's name and power limit, read in this run;
  - transfers/s at each --sizes block, device-resident (the _device form on torch buffers) and from host buffers (the
    host form with its copies), wall clock around calls that end in a stream synchronise, median of --reps;
  - the C oracle's sequential loop on one host core over the same block (the runtime applies a block's extrinsics one
    after another), and whether every output of both device forms equals the C oracle's;
  - block import against verification alone, alternated in one process, on an --import-tx block whose every transfer
    carries a valid proof of a toy key of the confidential shape (11 points, 22 public inputs: the verifier does the same
    work per proof as with the real key): import_confidential_block (the state on the device and the proofs checked
    against it) and verify_proofs_with_points on the same transactions' points, both from host buffers; the verdicts, the
    round count and the imported state are checked against the C oracle inside the run.
Blocks come from tests/jubjub_oracle/bal_corpus.py with a skewed sender choice; nothing is written to the repository."""
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
from tests.jubjub_oracle import bal_coracle as bc          # noqa: E402
from tests.jubjub_oracle import bal_corpus                 # noqa: E402
from zero_chain_b200 import groth16 as zk                  # noqa: E402
from zero_chain_b200 import synthetic as sy                # noqa: E402


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], text=True)
        name, power = [s.strip() for s in out.strip().split("\n")[0].split(",")]
        return name, power
    except Exception as e:                                 # the numbers are still printed, with the reason
        return "unknown (%s)" % e, "unknown"


def import_block(ctx, n, n_acct, reps):
    """block import (state + proofs) against verification alone on a block of n proven transfers"""
    n_pts = zk.CONFIDENTIAL_POINTS
    r1cs = sy.make_r1cs(60 + 2 * n_pts, 2 * n_pts + 1, 50, 40, 33, seed=5)
    crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=6)
    params = zk.Parameters.read(ctx, crs.params_bytes, checked=True)
    pvk = zk.PreparedVerifyingKey.prepare(ctx, crs.params_bytes)
    blk = bal_corpus.make(n_acct, n, 7 + n, skew=1.0, zero_frac=0.0, self_frac=0.02)
    misc = bal_corpus.encrypt(np.random.default_rng(8), 3)
    addr_s, addr_r, rvk, g_epoch, nonce = (misc[32 * i:32 * i + 32] for i in range(5))
    pts4 = lambda k: [blk.tx_points[128 * k + 32 * i:128 * k + 32 * i + 32] for i in range(4)]
    txs = [zk.ConfidentialTx(int(blk.sender[k]), int(blk.recipient[k]), addr_s, addr_r, *pts4(k), rvk, g_epoch, nonce) for k in range(n)]
    # every proof is made against the balance its transaction reads when every transfer passes
    bs = zk.confidential_block(ctx, *blk.args())[0]
    points = b"".join(zk.confidential_points(t.address_sender, t.address_recipient, t.amount_sender, t.amount_recipient, t.randomness,
                                             t.fee_sender, bs[64 * k:64 * k + 64], t.rvk, t.g_epoch, t.nonce) for k, t in enumerate(txs))
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
    params.free()
    proofs = bytes(proofs)
    accounts = (blk.balances, blk.pendings, blk.flags)
    run_import = lambda: zk.import_confidential_block(ctx, pvk, accounts, txs, proofs)
    run_verify = lambda: zk.verify_proofs_with_points(pvk, proofs, points, n_pts)
    verdicts, state, after, rounds = run_import()
    _, want = bc.block(*blk.args())
    ok = verdicts == [1] * n and rounds == 1 and run_verify() == [1] * n and state == want[3:] and after == want[1]
    ti, tv = [], []
    for _ in range(reps):                                   # alternated
        t0 = time.perf_counter(); run_import(); ti.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); run_verify(); tv.append(time.perf_counter() - t0)
    pvk.free()
    return {"transfers": n, "accounts": n_acct, "longest_chain": int(np.bincount(blk.sender).max()), "rounds": rounds,
            "import_ms": 1e3 * float(np.median(ti)), "import_tx_per_s": n / float(np.median(ti)),
            "verify_only_ms": 1e3 * float(np.median(tv)), "verify_only_tx_per_s": n / float(np.median(tv)),
            "import_over_verify": float(np.median(ti) / np.median(tv)), "verdicts_state_equal_c_oracle": bool(ok)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8192,65536")
    ap.add_argument("--accounts", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--import-tx", type=int, default=8192)
    ap.add_argument("--import-accounts", type=int, default=1024)
    a = ap.parse_args()
    import torch
    name, power = card()
    ctx = zk.Context(0)
    bc.lib()                                                # the C oracle is compiled before anything is timed
    res = {"card": name, "power_limit": power, "accounts": a.accounts, "sizes": {}}
    dev = lambda b: torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()
    for n in [int(x) for x in a.sizes.split(",")]:
        blk = bal_corpus.make(a.accounts, n, 100 + n, skew=1.0, bad_points=16, self_frac=0.02)
        t0 = time.perf_counter()
        bad, want = bc.block(*blk.args())
        host_loop = time.perf_counter() - t0
        assert bad is None
        ins = [dev(blk.balances), dev(blk.pendings), dev(blk.flags)]
        idx = [torch.from_numpy(v.astype(np.int64).astype(np.uint32).view(np.int32)).cuda() for v in (blk.sender, blk.recipient)]
        tp, apl = dev(blk.tx_points), dev(blk.applied)
        outs = [torch.zeros(k, dtype=torch.uint8, device="cuda") for k in (64 * n, 64 * n, n, 64 * a.accounts, 64 * a.accounts, a.accounts)]
        ptrs = lambda: ([t.data_ptr() for t in ins], [t.data_ptr() for t in idx], [t.data_ptr() for t in outs])
        pi, px, po = ptrs()
        run_dev = lambda: (zk.confidential_block_device(ctx, a.accounts, *pi, n, *px, tp.data_ptr(), apl.data_ptr(), *po), ctx.sync())
        run_host = lambda: zk.confidential_block(ctx, *blk.args())
        run_dev(); run_host()                               # warm-up: workspace, modules
        td, th = [], []
        for _ in range(a.reps):                             # the two forms alternate
            torch.cuda.synchronize()
            t0 = time.perf_counter(); run_dev(); td.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); got_h = run_host(); th.append(time.perf_counter() - t0)
        got_d = [t.cpu().numpy().tobytes() for t in outs]
        st = np.frombuffer(want[2], np.uint8)
        after_ok = np.array_equal(np.frombuffer(got_d[1], np.uint8).reshape(-1, 64)[st == 0],
                                  np.frombuffer(want[1], np.uint8).reshape(-1, 64)[st == 0])
        res["sizes"][str(n)] = {
            "device_resident_tx_per_s": n / float(np.median(td)), "device_resident_ms": 1e3 * float(np.median(td)),
            "host_buffers_tx_per_s": n / float(np.median(th)), "host_buffers_ms": 1e3 * float(np.median(th)),
            "c_oracle_one_core_tx_per_s": n / host_loop, "c_oracle_one_core_s": host_loop,
            "longest_chain": int(np.bincount(blk.sender).max()), "applied": int((st == 0).sum()),
            "host_form_equals_c_oracle": got_h == want,
            "device_form_equals_c_oracle": bool(after_ok and [got_d[0]] + got_d[2:] == [want[0]] + list(want[2:])),
        }
    res["import"] = import_block(ctx, a.import_tx, a.import_accounts, a.reps)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
