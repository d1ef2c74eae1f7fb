#!/usr/bin/env python3
"""Measures a block's encrypted-asset calls (zk_assets_block) and prints one JSON line:
  - the card's name and power limit, read in this run;
  - transactions/s at each --sizes block of mixed transfers, issues and destroys, device-resident (the _device form on
    torch buffers) and from host buffers (the host form with its copies), wall clock around calls that end in a stream
    synchronise, median of --reps;
  - the C oracle's sequential loop on one host core over the same block (the runtime applies a block's extrinsics one
    after another), and whether every output of both device forms equals the C oracle's;
  - block import against verification alone, alternated in one process, on an --import-tx block (transfers of asset 0,
    with issues and destroys among them) whose every transaction carries a valid proof of a toy key of the confidential
    shape (11 points, 22 public inputs: the verifier does the same work per proof as with the real key):
    import_assets_block and verify_proofs_with_points on the same transactions' points, both from host buffers; the
    verdicts, the asset ids, the round count and the imported state are checked against the C oracle inside the run.
Blocks come from tests/jubjub_oracle/assets_corpus.py with a skewed slot choice; nothing is written to the repository."""
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
from tests.jubjub_oracle import assets_coracle as ac       # noqa: E402
from tests.jubjub_oracle import assets_corpus              # noqa: E402
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


def import_block(ctx, n, n_slots, reps):
    """block import (state + proofs) against verification alone on a block of n proven transactions"""
    n_pts = zk.CONFIDENTIAL_POINTS
    r1cs = sy.make_r1cs(60 + 2 * n_pts, 2 * n_pts + 1, 50, 40, 33, seed=5)
    crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=6)
    params = zk.Parameters.read(ctx, crs.params_bytes, checked=True)
    pvk = zk.PreparedVerifyingKey.prepare(ctx, crs.params_bytes)
    blk = assets_corpus.make(n_slots, n, 7 + n, skew=1.0, issue_frac=0.02, destroy_frac=0.01, zero_frac=0.0, self_frac=0.02)
    rng = np.random.default_rng(8)
    keys = bal_corpus.encrypt(rng, n_slots)                # slot s is (0, keys[s]): distinct points
    key = lambda s: keys[64 * s:64 * s + 32]
    misc = bal_corpus.encrypt(rng, 3)
    rvk, g_epoch, nonce, fee = (misc[32 * i:32 * i + 32] for i in range(4))
    dummy_ct = misc[64:128]
    kinds = np.frombuffer(blk.kind, np.uint8)
    pts4 = lambda k: [blk.tx_points[128 * k + 32 * i:128 * k + 32 * i + 32] for i in range(4)]
    txs, slot_a, slot_b = [], blk.slot_a.copy(), blk.slot_b.copy()
    n_table = n_slots
    for k in range(n):
        p = pts4(k)
        if kinds[k] == zk.ASSET_ISSUE:                      # issue j creates asset j + 1, appended as slot n_slots + j
            txs.append(zk.IssueTx(key(int(blk.slot_a[k])), p[0], fee, dummy_ct, p[3], rvk, g_epoch, nonce))
            slot_a[k] = n_table
            n_table += 1
        elif kinds[k] == zk.ASSET_DESTROY:
            txs.append(zk.DestroyTx(key(int(blk.slot_a[k])), 0, misc[:32], fee, dummy_ct, misc[32:64], rvk, g_epoch, nonce))
        else:
            txs.append(zk.AssetTransferTx(0, key(int(blk.slot_a[k])), key(int(blk.slot_b[k])), *p, rvk, g_epoch, nonce))
    new_flags = zk.ACCOUNT_DUE
    table = (blk.balances + bytes(64 * (n_table - n_slots)), blk.pendings + bytes(64 * (n_table - n_slots)),
             blk.flags + bytes([new_flags] * (n_table - n_slots)))
    args = table + (blk.kind, slot_a, slot_b, b"".join(t.points() for t in txs), b"\x01" * n)
    bs = zk.assets_block(ctx, *args)[0]
    points = b"".join(t.verify_points(bs[64 * k:64 * k + 64]) if t.kind == zk.ASSET_TRANSFER else t.verify_points()
                      for k, t in enumerate(txs))
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
    state = ([(0, key(s)) for s in range(n_slots)], blk.balances, blk.pendings, blk.flags)
    run_import = lambda: zk.import_assets_block(ctx, pvk, state, txs, proofs, 1, new_flags)
    run_verify = lambda: zk.verify_proofs_with_points(pvk, proofs, points, n_pts)
    verdicts, ids, events, (slots, nb, npd, nf), rounds = run_import()
    _, want = ac.block(*args)
    n_issue = int((kinds == zk.ASSET_ISSUE).sum())
    ok = (verdicts == [1] * n and rounds == 1 and run_verify() == [1] * n and (nb, npd, nf) == want[5:] and len(slots) == n_table
          and [i for i in ids if i is not None] == list(range(1, 1 + n_issue)))
    ti, tv = [], []
    for _ in range(reps):                                   # alternated
        t0 = time.perf_counter(); run_import(); ti.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); run_verify(); tv.append(time.perf_counter() - t0)
    pvk.free()
    return {"transactions": n, "issues": n_issue, "destroys": int((kinds == zk.ASSET_DESTROY).sum()), "slots": n_table,
            "rounds": rounds, "import_ms": 1e3 * float(np.median(ti)), "import_tx_per_s": n / float(np.median(ti)),
            "verify_only_ms": 1e3 * float(np.median(tv)), "verify_only_tx_per_s": n / float(np.median(tv)),
            "import_over_verify": float(np.median(ti) / np.median(tv)), "verdicts_ids_state_equal_c_oracle": bool(ok)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8192,65536")
    ap.add_argument("--slots", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--import-tx", type=int, default=4096)
    ap.add_argument("--import-slots", type=int, default=1024)
    a = ap.parse_args()
    import torch
    name, power = card()
    ctx = zk.Context(0)
    ac.lib()                                                # the C oracle is compiled before anything is timed
    res = {"card": name, "power_limit": power, "slots": a.slots, "sizes": {}}
    dev = lambda b: torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()
    for n in [int(x) for x in a.sizes.split(",")]:
        blk = assets_corpus.make(a.slots, n, 100 + n, skew=1.0, bad_points=16, self_frac=0.02)
        t0 = time.perf_counter()
        bad, want = ac.block(*blk.args())
        host_loop = time.perf_counter() - t0
        assert bad is None
        ins = [dev(blk.balances), dev(blk.pendings), dev(blk.flags), dev(blk.kind)]
        idx = [torch.from_numpy(v.astype(np.int64).astype(np.uint32).view(np.int32)).cuda() for v in (blk.slot_a, blk.slot_b)]
        tp, apl = dev(blk.tx_points), dev(blk.applied)
        outs = [torch.zeros(k, dtype=torch.uint8, device="cuda") for k in (64 * n, 64 * n, 128 * n, n, n, 64 * a.slots, 64 * a.slots, a.slots)]
        pi, px, po = [t.data_ptr() for t in ins], [t.data_ptr() for t in idx], [t.data_ptr() for t in outs]
        run_dev = lambda: (zk.assets_block_device(ctx, a.slots, *pi[:3], n, pi[3], *px, tp.data_ptr(), apl.data_ptr(), *po), ctx.sync())
        run_host = lambda: zk.assets_block(ctx, *blk.args())
        run_dev(); run_host()                               # warm-up: workspace, modules
        td, th = [], []
        for _ in range(a.reps):                             # the two forms alternate
            torch.cuda.synchronize()
            t0 = time.perf_counter(); run_dev(); td.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); got_h = run_host(); th.append(time.perf_counter() - t0)
        got_d = [t.cpu().numpy().tobytes() for t in outs]   # zero where nothing is written, as the C oracle's
        st = np.frombuffer(want[4], np.uint8)
        kinds = np.frombuffer(blk.kind, np.uint8)
        res["sizes"][str(n)] = {
            "device_resident_tx_per_s": n / float(np.median(td)), "device_resident_ms": 1e3 * float(np.median(td)),
            "host_buffers_tx_per_s": n / float(np.median(th)), "host_buffers_ms": 1e3 * float(np.median(th)),
            "c_oracle_one_core_tx_per_s": n / host_loop, "c_oracle_one_core_s": host_loop,
            "longest_chain": int(np.bincount(blk.slot_a[blk.slot_a < a.slots]).max()), "applied": int((st == 0).sum()),
            "issues": int((kinds == 1).sum()), "destroys": int((kinds == 2).sum()),
            "host_form_equals_c_oracle": got_h == want, "device_form_equals_c_oracle": tuple(got_d) == want,
        }
    res["import"] = import_block(ctx, a.import_tx, a.import_slots, a.reps)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
