#!/usr/bin/env python3
"""Measures block import with the verify / apply rounds, and prints one JSON line:
  - the card's name and power limit, read in this run;
  - for a block of --conf-tx confidential transfers over --accounts accounts, and one of --asset-tx encrypted-asset calls
    (transfers, with --issue-frac issues and --destroy-frac destroys) over --slots slots, alternated in one process, median
    of --reps, wall clock around calls that end in a stream synchronise:
      driver   the Python drivers import_confidential_block / import_assets_block (a state call from host buffers and a
               verification launch per round, the rounds assembled in numpy)
      call     the one C call, confidential_import / assets_import (zk_import_confidential_block / zk_import_assets_block:
               one upload, the rounds on the device, one download; assets_import verifies the issues and destroys first)
      verify   verify_proofs_with_points_device alone on every proof of the block, on device-resident points
  - the rounds, and the ratios call / verify and driver / verify.
  - in the asset leg, a fourth arm alternated with the other three:
      calls    asset_calls_import (zk_import_asset_calls: the issue / destroy verification, the asset numbering and the
               slot resolution on the device too, from the slot table and the extrinsic fields)
      calls_c  zk_import_asset_calls alone, on host arrays built once before the reps: what a node calling the C ABI on
               the fields it already holds pays (asset_calls_import also joins each transaction's verifier row in Python)
    and the host-clock split of assets_import's host work, each part restated from it and timed in the same reps: the
    issue / destroy batch (their rows joined, verify_proofs_with_points from host buffers), _asset_slots, and the joins of
    the transfer rows and tx_points.
  - for a block of --anon-tx anonymous-balances calls (transfers, with --issue-frac issues) over --accounts accounts, the
    same three arms: the driver import_anonymous_calls_block (torch index ops between the launches), the one C call
    anonymous_import (zk_import_anonymous_block), and the two verify_proofs_with_points_device launches alone (issues on
    11 points, transfers on 52) on device-resident rows.  Proofs are forged from toy keys of the real shapes' input counts
    (tests/import_anon_corpus.py); the outputs are checked against anon_issue_coracle.c.
  - with --block, instead of the three legs above, one block of all three (the same sizes, one signature per
    transaction: 256 distinct signatures tiled, z_i drawn once before the reps), three arms alternated:
      block    block_import (zk_import_block: the signatures, then every section on one schedule of shared launches)
      calls    the four calls in sequence: redjubjub_verify_batched, confidential_import, asset_calls_import,
               anonymous_import
      verify   one 11-point verify_proofs_with_points_device launch over every confidential, asset and anonymous-issue
               proof and one 52-point launch over the anonymous transfers, on device-resident rows
    and the verifier launches each import arm makes.  Every output is checked against the others and the C oracles.
A leg with 0 transactions is skipped.
--fail-rate is the fraction of transfers (and of issues and destroys) whose proof fails; a transfer after a failure in its
chain is proven against the balance without it, so each failure costs a round.  Proofs are forged from a toy key's
trapdoor (tests/import_corpus.py, 22 public inputs: the verifier does the work of the real key per proof).  Every output
of every timed call is checked inside the run: the driver's and the call's equal, and the final state, balance_after,
events and verdicts equal the C oracle's (balances_oracle.c, assets_oracle.c) for the intended verdicts.  Nothing is
written to the repository."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import import_anon_corpus as iac               # noqa: E402
from tests import import_corpus as ic                     # noqa: E402
from zero_chain_b200 import groth16 as zk                  # noqa: E402


def log(*a):
    print(*a, file=sys.stderr, flush=True)                 # progress: the corpus and the C oracle take minutes


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], text=True)
        name, power = [s.strip() for s in out.strip().split("\n")[0].split(",")]
        return name, power
    except Exception as e:                                 # the numbers are still printed, with the reason
        return "unknown (%s)" % e, "unknown"


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--conf-tx", type=int, default=8192)
    ap.add_argument("--accounts", type=int, default=1024)
    ap.add_argument("--asset-tx", type=int, default=4096)
    ap.add_argument("--anon-tx", type=int, default=4096)
    ap.add_argument("--slots", type=int, default=1024)
    ap.add_argument("--issue-frac", type=float, default=0.05)
    ap.add_argument("--destroy-frac", type=float, default=0.02)
    ap.add_argument("--fail-rate", type=float, default=0.01)
    ap.add_argument("--skew", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--block", action="store_true", help="the whole-block leg instead of the three pallet legs")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("import_bench: no CUDA device (the measurement runs on the GPU only)")
    name, power = card()
    ctx = zk.Context(0)
    key = ic.ForgeKey(5)
    pvk = zk.PreparedVerifyingKey.prepare(ctx, key.params_bytes)
    res = {"card": name, "power_limit": power, "fail_rate": a.fail_rate, "reps": a.reps}
    dev = torch.device("cuda", 0)

    def verify_alone(rows, proofs):
        n = len(proofs)
        d_rows = torch.frombuffer(bytearray(rows), dtype=torch.uint8).to(dev)
        d_proofs = torch.frombuffer(bytearray(b"".join(proofs)), dtype=torch.uint8).to(dev)
        d_out = torch.zeros(n, dtype=torch.uint8, device=dev)
        torch.cuda.synchronize()

        def run():
            zk.verify_proofs_with_points_device(pvk, n, d_proofs.data_ptr(), d_rows.data_ptr(), zk.CONFIDENTIAL_POINTS, d_out.data_ptr())
            ctx.sync()
            return d_out.cpu().numpy().tobytes()
        return run

    def measure(label, driver, call, verify, check, extra=(), names=("driver", "call")):
        """the arms driver, call, verify and any (name, fn) in extra, alternated; name_over_verify for every arm"""
        arms = [(names[0], driver), (names[1], call), ("verify", verify)] + list(extra)
        for _, fn in arms:                           # warm-up: module loads, workspace growth
            fn()
        times = {k: [] for k, _ in arms}
        for r in range(a.reps):
            for k, fn in arms:
                ms, out = timed(fn)
                times[k].append(ms)
                check(k, out)
            log(label, "rep", r, {k: round(v[-1], 2) for k, v in times.items()})
        med = {k: float(np.median(v)) for k, v in times.items()}
        res = {"ms": {k: round(v, 3) for k, v in med.items()}}
        res.update({"%s_over_verify" % k: round(med[k] / med["verify"], 3) for k, _ in arms if k != "verify"})
        return res

    if a.block:
        res["block"] = block_leg(a, ctx, measure)
    if a.conf_tx and not a.block:
        res["confidential"] = confidential_leg(a, ctx, key, pvk, measure, verify_alone)
    if a.asset_tx and not a.block:
        res["assets"] = assets_leg(a, ctx, key, pvk, measure, verify_alone)
    if a.anon_tx and not a.block:
        res["anonymous"] = anonymous_leg(a, ctx, measure)
    res["outputs_equal_oracle"] = True
    pvk.free()
    ctx.close()
    print(json.dumps(res))


def confidential_leg(a, ctx, key, pvk, measure, verify_alone):
    log("confidential corpus: %d transfers over %d accounts" % (a.conf_tx, a.accounts))
    blk = ic.confidential(key, a.accounts, a.conf_tx, a.seed, fail_frac=a.fail_rate, skew=a.skew,
                          state_call=lambda *x: zk.confidential_block(ctx, *x))
    want = zk.confidential_import(ctx, pvk, blk.accounts, blk.txs, blk.proofs)
    log("C oracle (confidential)")
    o = blk.oracle(want[0])
    assert want[0] == blk.intended, "verdicts differ from the intended ones"
    assert (o[0],) + o[2:] == (want[2],) + want[1], "the import differs from the C oracle"
    v_want = bytes(want[0])

    def check_conf(k, out):
        if k == "verify":
            assert out == v_want, "verification alone differs"
        else:
            assert out == want, "%s differs" % k
    return dict(measure("confidential", lambda: zk.import_confidential_block(ctx, pvk, blk.accounts, blk.txs, blk.proofs),
                                       lambda: zk.confidential_import(ctx, pvk, blk.accounts, blk.txs, blk.proofs),
                                       verify_alone(blk.rows, blk.proofs), check_conf),
                n_tx=a.conf_tx, accounts=a.accounts, rounds=want[3], failures=sum(v != 1 for v in want[0]))


def assets_leg(a, ctx, key, pvk, measure, verify_alone):
    log("asset corpus: %d calls over %d slots" % (a.asset_tx, a.slots))
    ab = ic.assets(key, a.slots, a.asset_tx, a.seed + 1, fail_frac=a.fail_rate, fixed_fail_frac=a.fail_rate, issue_frac=a.issue_frac,
                   destroy_frac=a.destroy_frac, skew=a.skew, state_call=lambda *x: zk.assets_block(ctx, *x))
    awant = zk.assets_import(ctx, pvk, *ab.args())
    log("C oracle (assets)")
    ao = ab.oracle(awant[0])
    assert awant[0] == ab.intended, "asset verdicts differ from the intended ones"
    assert awant[3][1:] == ao[5:], "the asset import differs from the C oracle"
    assert all(awant[2][k] == ao[1][64 * k:64 * k + 64] for k, t in enumerate(ab.txs) if t.kind == zk.ASSET_TRANSFER and ao[4][k] == 0)
    av_want = bytes(awant[0])

    split = {"fixed_batch": [], "asset_slots": [], "row_joins": []}

    def host_split():
        """assets_import's host steps, as it runs them, each on the host clock; returns what it computed"""
        slots = [(int(x), zk._pt32(k)) for x, k in ab.state[0]]
        proofs = zk._cat(ab.proofs, 192)
        t0 = time.perf_counter()
        n = len(ab.txs)
        proof_rows = np.frombuffer(proofs, np.uint8).reshape(n, 192)
        kinds = np.array([t.kind for t in ab.txs], np.uint8)
        fixed_v = np.zeros(n, np.uint8)
        fixed = np.flatnonzero(kinds != zk.ASSET_TRANSFER)
        if len(fixed):
            pts = b"".join(ab.txs[k].verify_points() for k in fixed.tolist())
            fixed_v[fixed] = zk.verify_proofs_with_points(pvk, proof_rows[fixed].tobytes(), pts, zk.CONFIDENTIAL_POINTS)
        t1 = time.perf_counter()
        table = zk._asset_slots("import_bench", slots, *ab.state[1:], ab.txs, fixed_v, ab.next_asset_id, ab.new_slot_flags)
        t2 = time.perf_counter()
        rows = b"".join(t.verify_points(bytes(64)) if t.kind == zk.ASSET_TRANSFER else bytes(32 * zk.CONFIDENTIAL_POINTS) for t in ab.txs)
        tp = b"".join(t.points() for t in ab.txs)
        t3 = time.perf_counter()
        for k, (u, v) in zip(split, ((t0, t1), (t1, t2), (t2, t3))):
            split[k].append((v - u) * 1e3)
        return fixed_v, table, len(rows) + len(tp)
    split_want = host_split()

    import ctypes as C
    from zero_chain_b200 import _lib
    slots, bal, pend, fl = ab.state
    n, ns = len(ab.txs), len(slots)
    u8 = lambda b: np.frombuffer(bytes(b), np.uint8).copy()
    c_in = [np.array([x for x, _ in slots], np.uint32), u8(b"".join(k for _, k in slots)), u8(bal), u8(pend), u8(fl),
            u8(bytes(t.kind for t in ab.txs)), np.array([t.asset_id if t.kind != zk.ASSET_ISSUE else 0 for t in ab.txs], np.uint32),
            u8(b"".join(t.verify_points(bytes(64)) if t.kind == zk.ASSET_TRANSFER else t.verify_points() for t in ab.txs)),
            u8(b"".join(ab.proofs))]

    def c_call():
        nr = ns + 2 * n
        out = [np.zeros(m, np.uint8) for m in (n, 4 * n, 64 * n, 128 * n, n, n, 4 * nr, 32 * nr, 64 * nr, 64 * nr, nr)]
        n_out, rounds = C.c_size_t(0), C.c_uint(0)
        zk._ck(_lib.lib().zk_import_asset_calls(ctx._h, pvk._h, ns, *[zk._p(x) for x in c_in[:5]], ab.next_asset_id, ab.new_slot_flags, n,
                                                *[zk._p(x) for x in c_in[5:]], *[zk._p(o) for o in out], C.byref(n_out), C.byref(rounds)))
        m = n_out.value
        return (out[0].tobytes(), out[8][:64 * m].tobytes(), out[9][:64 * m].tobytes(), out[10][:m].tobytes(), rounds.value)
    c_want = (bytes(awant[0]),) + awant[3][1:] + (awant[4],)

    def check_assets(k, out):
        if k == "calls_c":
            assert out == c_want, "the C call differs"
        elif k == "verify":
            assert out == av_want, "verification alone differs"
        elif k == "split":
            assert all(np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y for x, y in zip(out[1][1:], split_want[1][1:]))
            assert out[1][0] == split_want[1][0] and bytes(out[0]) == bytes(split_want[0]) and out[2] == split_want[2]
        else:
            assert out == awant, "%s differs" % k
    r = dict(measure("assets", lambda: zk.import_assets_block(ctx, pvk, *ab.args()), lambda: zk.assets_import(ctx, pvk, *ab.args()),
                     verify_alone(ab.rows, ab.proofs), check_assets,
                     extra=[("calls", lambda: zk.asset_calls_import(ctx, pvk, *ab.args())), ("calls_c", c_call), ("split", host_split)]),
             n_tx=a.asset_tx, slots=a.slots, rounds=awant[4], failures=sum(v != 1 for v in awant[0]))
    # the split arm is host work timed in parts: its medians, not its ratio, are the result
    r["ms"].pop("split")
    r.pop("split_over_verify")
    r["assets_import_host_ms"] = {k: round(float(np.median(v[-a.reps:])), 3) for k, v in split.items()}
    return r


def anonymous_leg(a, ctx, measure):
    import torch
    anon, conf = iac.ForgeKey(zk.ANONYMOUS_POINTS, 71), iac.ForgeKey(zk.CONFIDENTIAL_POINTS, 171)
    apvk, cpvk = zk.PreparedVerifyingKey.prepare(ctx, anon.params_bytes), zk.PreparedVerifyingKey.prepare(ctx, conf.params_bytes)
    log("anonymous corpus: %d calls over %d accounts" % (a.anon_tx, a.accounts))
    blk = iac.block(anon, conf, a.accounts, a.anon_tx, a.seed + 2, issue_frac=a.issue_frac, fail_frac=a.fail_rate, skew=a.skew)
    want = zk.anonymous_import(ctx, apvk, cpvk, *blk.args())
    log("C oracle (anonymous)")
    o = blk.oracle(want[0])
    assert want[0] == blk.intended, "anonymous verdicts differ from the intended ones"
    assert want[2] == o[0] and want[1] == o[4:], "the anonymous import differs from the C oracle"
    assert all(x == (o[2][64 * k:64 * k + 64] if x is not None else None) for k, x in enumerate(want[3])), "issued differs from the C oracle"
    iss = [k for k, t in enumerate(blk.txs) if t.kind == zk.ANON_ISSUE]
    tr = [k for k, t in enumerate(blk.txs) if t.kind == zk.ANON_TRANSFER]
    # the verifier's rows, device-resident: the issues' 11 points, the transfers' 52 from the state the oracle gives
    dev = torch.device("cuda", 0)
    up = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev) if b else torch.zeros(1, dtype=torch.uint8, device=dev)
    d_iss = up(b"".join(blk.txs[k].verify_points(blk.accounts[0], blk.g_epoch) for k in iss))
    d_tr = up(b"".join(o[1][1664 * k:1664 * k + 1664] for k in tr))
    d_ip, d_tp = up(b"".join(blk.proofs[k] for k in iss)), up(b"".join(blk.proofs[k] for k in tr))
    d_out = torch.zeros(len(blk.txs) + 1, dtype=torch.uint8, device=dev)
    v_want = bytes(blk.intended[k] for k in iss + tr)
    torch.cuda.synchronize()

    def verify():
        if iss:
            zk.verify_proofs_with_points_device(cpvk, len(iss), d_ip.data_ptr(), d_iss.data_ptr(), zk.CONFIDENTIAL_POINTS, d_out.data_ptr())
        if tr:
            zk.verify_proofs_with_points_device(apvk, len(tr), d_tp.data_ptr(), d_tr.data_ptr(), zk.ANONYMOUS_POINTS,
                                                d_out.data_ptr() + len(iss))
        ctx.sync()
        return d_out[:len(blk.txs)].cpu().numpy().tobytes()

    def check(k, out):
        assert out == (v_want if k == "verify" else want), "%s differs" % k
    r = dict(measure("anonymous", lambda: zk.import_anonymous_calls_block(ctx, apvk, cpvk, *blk.args()),
                     lambda: zk.anonymous_import(ctx, apvk, cpvk, *blk.args()), verify, check),
             n_tx=a.anon_tx, accounts=a.accounts, issues=len(iss), failures=sum(v != 1 for v in want[0]))
    apvk.free()
    cpvk.free()
    return r


def block_leg(a, ctx, measure):
    import torch
    from tests.jubjub_oracle import redjubjub as rj
    conf, anon = iac.ForgeKey(zk.CONFIDENTIAL_POINTS, 171), iac.ForgeKey(zk.ANONYMOUS_POINTS, 71)
    cpvk, apvk = zk.PreparedVerifyingKey.prepare(ctx, conf.params_bytes), zk.PreparedVerifyingKey.prepare(ctx, anon.params_bytes)
    log("block corpus: %d confidential, %d asset, %d anonymous calls" % (a.conf_tx, a.asset_tx, a.anon_tx))
    cb = ic.confidential(conf, a.accounts, a.conf_tx, a.seed, fail_frac=a.fail_rate, skew=a.skew)
    ab = ic.assets(conf, a.slots, a.asset_tx, a.seed + 1, fail_frac=a.fail_rate, fixed_fail_frac=a.fail_rate, issue_frac=a.issue_frac,
                   destroy_frac=a.destroy_frac, skew=a.skew, state_call=lambda *x: zk.assets_block(ctx, *x))
    nb = iac.block(anon, conf, a.accounts, a.anon_tx, a.seed + 2, issue_frac=a.issue_frac, fail_frac=a.fail_rate, skew=a.skew)
    n_sig = a.conf_tx + a.asset_tx + a.anon_tx
    distinct = []
    for i in range(256):
        sk = rj.spending_key(b"bench-%d" % i)
        msg = b"extrinsic %d" % i
        distinct.append((rj.public_key(sk), rj.sign(sk, msg, bytes([i]) * 80), msg))
    vks, sigs, msgs = ([distinct[i % 256][j] for i in range(n_sig)] for j in range(3))
    sig = (vks, sigs, msgs, zk.random_batch_scalars(n_sig))    # drawn once: neither arm times the draw
    c_args, a_args, n_args = (cb.accounts, cb.txs, cb.proofs), ab.args(), nb.args()
    want = (zk.confidential_import(ctx, cpvk, *c_args), zk.asset_calls_import(ctx, cpvk, *a_args), zk.anonymous_import(ctx, apvk, cpvk, *n_args))
    log("C oracles (block)")
    assert [w[0] for w in want] == [cb.intended, ab.intended, nb.intended], "verdicts differ from the intended ones"
    co, ao, no = cb.oracle(want[0][0]), ab.oracle(want[1][0]), nb.oracle(want[2][0])
    assert want[0][2] == co[0] and want[0][1] == tuple(co[2:]), "the confidential import differs from the C oracle"
    assert want[1][3][1:] == ao[5:], "the asset import differs from the C oracle"
    assert want[2][2] == no[0] and want[2][1] == no[4:], "the anonymous import differs from the C oracle"
    iss = [k for k, t in enumerate(nb.txs) if t.kind == zk.ANON_ISSUE]
    tr = [k for k, t in enumerate(nb.txs) if t.kind == zk.ANON_TRANSFER]
    dev = torch.device("cuda", 0)
    up = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev) if b else torch.zeros(1, dtype=torch.uint8, device=dev)
    rows11 = cb.rows + ab.rows + b"".join(nb.txs[k].verify_points(nb.accounts[0], nb.g_epoch) for k in iss)
    proofs11 = b"".join(cb.proofs) + b"".join(ab.proofs) + b"".join(nb.proofs[k] for k in iss)
    n11 = len(proofs11) // 192
    d_r11, d_p11 = up(rows11), up(proofs11)
    d_r52, d_p52 = up(b"".join(no[1][1664 * k:1664 * k + 1664] for k in tr)), up(b"".join(nb.proofs[k] for k in tr))
    d_out = torch.zeros(n11 + len(tr) + 1, dtype=torch.uint8, device=dev)
    v_want = bytes(cb.intended + ab.intended + [nb.intended[k] for k in iss + tr])
    torch.cuda.synchronize()

    def verify():
        zk.verify_proofs_with_points_device(cpvk, n11, d_p11.data_ptr(), d_r11.data_ptr(), zk.CONFIDENTIAL_POINTS, d_out.data_ptr())
        if tr:
            zk.verify_proofs_with_points_device(apvk, len(tr), d_p52.data_ptr(), d_r52.data_ptr(), zk.ANONYMOUS_POINTS,
                                                d_out.data_ptr() + n11)
        ctx.sync()
        return d_out[:n11 + len(tr)].cpu().numpy().tobytes()

    launches = {}

    def block():
        r = zk.block_import(ctx, cpvk, apvk, sig, c_args, a_args, n_args)
        launches["block"] = r.launches
        return r[:3]

    def calls():
        assert zk.redjubjub_verify_batched(ctx, *sig) == [zk.REDJUBJUB_OK] * n_sig
        out = (zk.confidential_import(ctx, cpvk, *c_args), zk.asset_calls_import(ctx, cpvk, *a_args),
               zk.anonymous_import(ctx, apvk, cpvk, *n_args))
        launches["calls"] = (out[0][3] + out[1][4] + any(t.kind != zk.ASSET_TRANSFER for t in ab.txs) + (len(iss) > 0) + (len(tr) > 0))
        return out

    def check(k, out):
        assert out == (v_want if k == "verify" else want), "%s differs" % k
    r = dict(measure("block", calls, block, verify, check, names=("calls", "block")), signatures=n_sig,
             failures=sum(v != 1 for w in want for v in w[0]), rounds={"confidential": want[0][3], "assets": want[1][4]})
    r["launches"] = launches
    cpvk.free()
    apvk.free()
    return r


if __name__ == "__main__":
    main()
