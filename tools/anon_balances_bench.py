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
Blocks come from tests/jubjub_oracle/anon_corpus.py; nothing is written to the repository."""
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


def import_block(ctx, n, n_acct, reps):
    """block import (state + verifier inputs + proofs) against verification alone on a block of n proven transfers"""
    import torch
    n_pts = zk.ANONYMOUS_POINTS
    r1cs = sy.make_r1cs(60 + 2 * n_pts, 2 * n_pts + 1, 50, 40, 33, seed=5)
    crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=6)
    params = zk.Parameters.read(ctx, crs.params_bytes, checked=True)
    pvk = zk.PreparedVerifyingKey.prepare(ctx, crs.params_bytes)
    blk = anon_corpus.make(n_acct, n, 7 + n, skew=1.0, mask_p=(0.0, 1.0, 0.0, 0.0, 0.0))
    # every proof is made on the points its transaction's verifier reads
    _, want0 = aco.block(*blk.args()[:-1], bytes(n))
    points = want0[1]
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
    params.free()
    proofs = bytes(proofs)
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1024,8192")
    ap.add_argument("--accounts", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--import-tx", type=int, default=256)
    ap.add_argument("--import-accounts", type=int, default=1024)
    a = ap.parse_args()
    import torch
    name, power = card()
    ctx = zk.Context(0)
    aco.lib()                                               # the C oracle is compiled before anything is timed
    res = {"card": name, "power_limit": power, "accounts": a.accounts, "sizes": {}}
    dev = lambda b: torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()
    na = a.accounts
    for n in [int(x) for x in a.sizes.split(",")]:
        blk = anon_corpus.make(na, n, 100 + n, skew=1.0, bad_points=16)
        t0 = time.perf_counter()
        bad, want = aco.block(*blk.args())
        host_loop = time.perf_counter() - t0
        assert bad is None
        log("C oracle:", n, "transfers in %.1f s" % host_loop)
        ins = [dev(blk.keys), dev(blk.balances), dev(blk.pendings), dev(blk.flags)]
        mem = torch.from_numpy(blk.members.astype(np.uint32).view(np.int32)).cuda()
        txi = [dev(blk.tx_points), dev(blk.tx_extra), dev(blk.g_epoch), dev(blk.applied)]
        outs = [torch.zeros(k, dtype=torch.uint8, device="cuda") for k in (768 * n, 1664 * n, n, 64 * na, 64 * na, na)]
        torch.cuda.synchronize()
        pi, pt, po = [t.data_ptr() for t in ins], [t.data_ptr() for t in txi], [t.data_ptr() for t in outs]
        run_dev = lambda: (zk.anonymous_block_device(ctx, na, *pi, n, mem.data_ptr(), *pt, *po), ctx.sync())
        run_host = lambda: zk.anonymous_block(ctx, *blk.args())
        run_dev(); run_host()                               # warm-up: workspace, modules
        td, th = [], []
        for _ in range(a.reps):                             # the two forms alternate
            torch.cuda.synchronize()
            t0 = time.perf_counter(); run_dev(); td.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); got_h = run_host(); th.append(time.perf_counter() - t0)
        got_d = tuple(t.cpu().numpy().tobytes() for t in outs)
        st = np.frombuffer(want[2], np.uint8)
        res["sizes"][str(n)] = {
            "device_resident_tx_per_s": n / float(np.median(td)), "device_resident_ms": 1e3 * float(np.median(td)),
            "host_buffers_tx_per_s": n / float(np.median(th)), "host_buffers_ms": 1e3 * float(np.median(th)),
            "c_oracle_one_core_tx_per_s": n / host_loop, "c_oracle_one_core_s": host_loop,
            "most_rings_of_one_account": int(np.bincount(blk.members).max()), "applied": int((st == 0).sum()),
            "host_form_equals_c_oracle": got_h == want, "device_form_equals_c_oracle": got_d == want,
        }
    res["import"] = import_block(ctx, a.import_tx, a.import_accounts, a.reps)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
