"""Throughput of RedJubjub signature verification (zk_redjubjub_verify_batch), one JSON line:
  sigs_per_s[batch][msg_len]     host buffers (copies included) and device-resident, at batch 8192 / 65536, 32- / 256-byte messages
  host_sigs_per_s[msg_len]       the C oracle's verification on every host core (OpenMP), the CPU baseline
  tx_per_s_both_device           zk_groth16_verify_points_batch_device + zk_redjubjub_verify_batch_device on one context for the
                                 same 8192 confidential-shape transactions, each signed by its rvk point (32-byte messages)
  tx_per_s_proof_only_device     the proof check alone on the same transactions (alternated with the line above)
with the card's name and power limit read in the same run.  Every timed result is checked against the C oracle's verdicts.
Usage: python tools/redjubjub_bench.py [--reps 5]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import coracle as co                              # noqa: E402
from tests.jubjub_oracle import rj_coracle as cj              # noqa: E402
from tests.jubjub_oracle import pyref as jj                   # noqa: E402
from tests.jubjub_oracle import redjubjub as rj               # noqa: E402
from tools.verify_tx_bench import card, timed                 # noqa: E402
from zero_chain_b200 import groth16 as zk                     # noqa: E402
from zero_chain_b200 import synthetic as sy                   # noqa: E402

BASE = 1024                                                   # distinct signatures, tiled to the batch


def corpus(rng, msg_len, n):
    sks = [int.from_bytes(rng.bytes(32), "little") % rj.R_J for _ in range(BASE)]
    msgs = [rng.bytes(msg_len) for _ in range(BASE)]
    vks = cj.redjubjub_public_key(sks)
    sigs = cj.redjubjub_sign(sks, rng.bytes(80 * BASE), msgs)
    idx = np.arange(n) % BASE
    vk = np.frombuffer(vks, np.uint8).reshape(BASE, 32)[idx].tobytes()
    sg = np.frombuffer(sigs, np.uint8).reshape(BASE, 64)[idx].tobytes()
    return vk, sg, [msgs[i] for i in idx], sks


def to_dev(b: bytes):
    return torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()


def device_verify(ctx, n, vk, sg, msgs):
    dvk, dsg, dm = to_dev(vk), to_dev(sg), to_dev(b"".join(msgs))
    doff = torch.from_numpy(zk.message_offsets(msgs).view(np.int64)).cuda()
    dv = torch.zeros(n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def run():
        zk.redjubjub_verify_device(ctx, n, dvk.data_ptr(), dsg.data_ptr(), dm.data_ptr(), doff.data_ptr(), dv.data_ptr()); ctx.sync()
    return run, dv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    ctx = zk.Context(0)
    rng = np.random.default_rng(1)
    out = {"metric": "redjubjub_verify", "sigs_per_s_host": {}, "sigs_per_s_device": {}, "host_sigs_per_s": {}}
    for msg_len in (32, 256):
        vk, sg, msgs, _ = corpus(rng, msg_len, 65536)
        want = cj.redjubjub_verify(vk[:32 * BASE], sg[:64 * BASE], msgs[:BASE])
        assert (want == 1).all()
        for n in (8192, 65536):
            v, s, m = vk[:32 * n], sg[:64 * n], msgs[:n]
            assert zk.redjubjub_verify(ctx, v, s, m) == [1] * n
            key = "%d/%dB" % (n, msg_len)
            out["sigs_per_s_host"][key] = n / timed(lambda: zk.redjubjub_verify(ctx, v, s, m), a.reps)
            run, dv = device_verify(ctx, n, v, s, m)
            run(); assert bool((dv == 1).all())
            out["sigs_per_s_device"][key] = n / timed(run, a.reps)
            assert bool((dv == 1).all())
        hn = 4096
        t = timed(lambda: cj.redjubjub_verify(vk[:32 * hn], sg[:64 * hn], msgs[:hn]), max(1, a.reps // 2))
        out["host_sigs_per_s"]["%dB" % msg_len] = hn / t

    # both checks of a confidential transfer on one context: the signer is the transaction's rvk point
    n, n_pts = 8192, zk.CONFIDENTIAL_POINTS
    r1cs = sy.make_r1cs(60 + 2 * n_pts, 2 * n_pts + 1, 50, 40, 33, seed=1)
    crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=2)
    params = zk.Parameters.read(ctx, crs.params_bytes, checked=True)
    pvk = zk.PreparedVerifyingKey.prepare(ctx, crs.params_bytes)
    base_proofs, base_pts, base_sig, base_msg = [], [], [], []
    for s in range(64):
        sk = int.from_bytes(rng.bytes(32), "little") % rj.R_J
        pts = [jj.prime_order_point(int.from_bytes(rng.bytes(32), "little")) for _ in range(n_pts)]
        pts[8] = jj.read(cj.redjubjub_public_key([sk]))[1]      # rvk: 9th point of verify_confidential_proof's push order
        z = sy.make_witness(r1cs, s + 1, inputs=[c for p in pts for c in p])
        av, bv, cv = sy.evaluate(r1cs, z)
        pa = zk.ProvingAssignment(co.ints_to_limbs(av, 4), co.ints_to_limbs(bv, 4), co.ints_to_limbs(cv, 4),
                                  co.ints_to_limbs(z[:r1cs.n_inputs], 4), co.ints_to_limbs(z[r1cs.n_inputs:], 4), *sy.densities(r1cs))
        base_proofs.append(zk.create_proof(pa, params, 11 + s, 13 + s))
        base_pts.append(b"".join(jj.encode(p) for p in pts))
        msg = rng.bytes(32)                                      # blake2_256 of a payload over 256 bytes
        base_msg.append(msg)
        base_sig.append(cj.redjubjub_sign([sk], rng.bytes(80), [msg]))
    params.free()
    proofs = b"".join(base_proofs[i % 64] for i in range(n))
    points = b"".join(base_pts[i % 64] for i in range(n))
    signers = b"".join(base_pts[i % 64][256:288] for i in range(n))
    sigs = b"".join(base_sig[i % 64] for i in range(n))
    msgs = [base_msg[i % 64] for i in range(n)]
    assert (cj.redjubjub_verify(signers, sigs, msgs) == 1).all()
    assert zk.verify_proofs_with_points(pvk, proofs, points, n_pts) == [1] * n
    dp, dpt, dvp = to_dev(proofs), to_dev(points), torch.zeros(n, dtype=torch.uint8, device="cuda")
    run_sig, dvs = device_verify(ctx, n, signers, sigs, msgs)

    def proof_only():
        zk.verify_proofs_with_points_device(pvk, n, dp.data_ptr(), dpt.data_ptr(), n_pts, dvp.data_ptr()); ctx.sync()

    def both():
        zk.verify_proofs_with_points_device(pvk, n, dp.data_ptr(), dpt.data_ptr(), n_pts, dvp.data_ptr())
        run_sig()                                                # same stream; run_sig ends with the context sync

    both(); proof_only()
    ta, tb = [], []
    for _ in range(a.reps):                                      # A/B alternated in one process
        ta.append(timed(both, 1)); assert bool((dvp == 1).all()) and bool((dvs == 1).all())
        tb.append(timed(proof_only, 1)); assert bool((dvp == 1).all())
    name, plimit = card()
    out.update({"gpu_name": name, "power_limit_w": plimit, "tx_batch": n,
                "tx_per_s_both_device": n / float(np.median(ta)), "tx_per_s_proof_only_device": n / float(np.median(tb)),
                "ab_ms": {"both": [round(x * 1e3, 3) for x in ta], "proof_only": [round(x * 1e3, 3) for x in tb]},
                "host_threads": cj.threads(), "host_cpus": os.cpu_count()})
    pvk.free(); ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
