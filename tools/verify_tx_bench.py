"""Throughput of the zk-system verification path that starts from point bytes (confidential-transfer shape: 11 Jubjub points,
22 public inputs), one JSON line:
  decode_points_per_s        zk_jubjub_into_xy on host buffers (copies included)
  points_tx_per_s_host       zk_groth16_verify_points_batch, host buffers
  points_tx_per_s_device     zk_groth16_verify_points_batch_device, device-resident proofs and points
  decoded_tx_per_s_device    zk_groth16_verify_batch_device on the same transactions' pre-decoded inputs (alternated with the
                             line above in the same process: A/B)
  host_decode_tx_per_s       the C oracle's decoding of the same points on every host core (OpenMP), the CPU baseline
with the card's name and power limit read in the same run.  Usage: python tools/verify_tx_bench.py [--batch 8192] [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import coracle as co                              # noqa: E402
from tests.jubjub_oracle import coracle as cj                 # noqa: E402
from tests.jubjub_oracle import pyref as jj                   # noqa: E402
from zero_chain_b200 import groth16 as zk                     # noqa: E402
from zero_chain_b200 import synthetic as sy                   # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30).stdout.strip().split(",")
    return q[0].strip(), float(q[1])


def timed(fn, reps):
    fn()                                                      # warm-up (workspace allocation, module load)
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    n, n_pts = a.batch, zk.CONFIDENTIAL_POINTS
    ctx = zk.Context(0)
    r1cs = sy.make_r1cs(60 + 2 * n_pts, 2 * n_pts + 1, 50, 40, 33, seed=1)
    crs = sy.make_toy_crs(r1cs, co.g1_fixed_base, co.g2_fixed_base, seed=2)
    params = zk.Parameters.read(ctx, crs.params_bytes, checked=True)
    pvk = zk.PreparedVerifyingKey.prepare(ctx, crs.params_bytes)
    rng = np.random.default_rng(1)
    # 64 distinct transactions (704 distinct points) tiled to the batch
    base_tx, base_proofs = [], []
    for s in range(64):
        pts = [jj.prime_order_point(int.from_bytes(rng.bytes(32), "little")) for _ in range(n_pts)]
        z = sy.make_witness(r1cs, s + 1, inputs=[c for p in pts for c in p])
        av, bv, cv = sy.evaluate(r1cs, z)
        pa = zk.ProvingAssignment(co.ints_to_limbs(av, 4), co.ints_to_limbs(bv, 4), co.ints_to_limbs(cv, 4),
                                  co.ints_to_limbs(z[:r1cs.n_inputs], 4), co.ints_to_limbs(z[r1cs.n_inputs:], 4), *sy.densities(r1cs))
        base_proofs.append(zk.create_proof(pa, params, 11 + s, 13 + s))
        base_tx.append(pts)
    params.free()
    proofs = b"".join(base_proofs[i % 64] for i in range(n))
    points = b"".join(b"".join(jj.encode(p) for p in base_tx[i % 64]) for i in range(n))
    inputs = np.stack([co.ints_to_limbs([c for p in base_tx[i % 64] for c in p], 4).reshape(-1) for i in range(64)])
    inputs = np.ascontiguousarray(inputs[np.arange(n) % 64])

    # results first: both paths give verdict 1 everywhere, the decoder gives the oracle's coordinates
    xy, st = zk.jubjub_into_xy(ctx, points)
    hxy, hst = cj.into_xy(points)
    assert not st.any() and not hst.any() and np.array_equal(xy, hxy)
    assert np.array_equal(xy.reshape(n, -1), inputs)
    assert zk.verify_proofs_with_points(pvk, proofs, points, n_pts) == [1] * n

    t_decode = timed(lambda: zk.jubjub_into_xy(ctx, points), a.reps)
    t_host = timed(lambda: zk.verify_proofs_with_points(pvk, proofs, points, n_pts), a.reps)
    dp = torch.from_numpy(np.frombuffer(proofs, np.uint8).copy()).cuda()
    dpt = torch.from_numpy(np.frombuffer(points, np.uint8).copy()).cuda()
    din = torch.from_numpy(inputs.view(np.int64)).cuda()
    dv = torch.zeros(n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def with_points():
        zk.verify_proofs_with_points_device(pvk, n, dp.data_ptr(), dpt.data_ptr(), n_pts, dv.data_ptr()); ctx.sync()

    def pre_decoded():
        zk.verify_proofs_device(pvk, n, dp.data_ptr(), din.data_ptr(), 2 * n_pts, dv.data_ptr()); ctx.sync()

    with_points(); pre_decoded()
    ta, tb = [], []
    for _ in range(a.reps):                                   # A/B alternated in one process
        ta.append(timed(with_points, 1)); assert bool((dv == 1).all())
        tb.append(timed(pre_decoded, 1)); assert bool((dv == 1).all())
    t_cpu = timed(lambda: cj.into_xy(points), max(1, a.reps // 2))
    name, plimit = card()
    out = {
        "metric": "verify_tx_points", "batch": n, "points_per_tx": n_pts, "gpu_name": name, "power_limit_w": plimit,
        "decode_points_per_s": n * n_pts / t_decode,
        "points_tx_per_s_host": n / t_host,
        "points_tx_per_s_device": n / float(np.median(ta)),
        "decoded_tx_per_s_device": n / float(np.median(tb)),
        "ab_ms": {"with_points": [round(x * 1e3, 3) for x in ta], "pre_decoded": [round(x * 1e3, 3) for x in tb]},
        "host_decode_tx_per_s": n / t_cpu, "host_threads": cj.threads(), "host_cpus": os.cpu_count(),
    }
    pvk.free(); ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
