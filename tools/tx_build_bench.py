#!/usr/bin/env python3
"""Throughput of building confidential transfers on the device: keys from seeds, confidential fields and RedJubjub
signatures per second, for batches of 8192 and 65536, device-resident (the _device forms on torch buffers, CUDA events)
and from host buffers (the host forms, wall clock, copies included).  Every output of the run is checked: the device and
host forms agree byte for byte, every signature verifies under its key (zk_redjubjub_verify_batch), every amount_sender
decrypts to its amount under the derived dk (zk_elgamal_decrypt_batch), and a few rows of each equal the Python oracle.
The host baseline is the C oracle (tests/jubjub_oracle/tx_build_oracle.c, redjubjub_oracle.c for signing) on all host
cores, timed on the first HOST_ROWS rows of each batch, whose outputs must equal the device's.  Prints one JSON line with
the card's name and power limit, read in the same run.

Usage: python tools/tx_build_bench.py [--sizes 8192,65536] [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.jubjub_oracle import redjubjub as rj     # noqa: E402
from tests.jubjub_oracle import rj_coracle as cj    # noqa: E402
from tests.jubjub_oracle import tx_coracle as tc    # noqa: E402
from tests.jubjub_oracle import tx_build as tb      # noqa: E402
from zero_chain_b200 import groth16 as zk           # noqa: E402

HOST_ROWS = 2048     # rows of each batch the host baseline computes (it runs at a few thousand rows per second)


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"]).decode().splitlines()[0]
    name, power = [s.strip() for s in out.split(",")]
    return name, power


def timed_device(ctx, fn, reps):
    import torch
    fn()
    ctx.sync()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record(torch.cuda.ExternalStream(ctx.stream))
    for _ in range(reps):
        fn()
    e.record(torch.cuda.ExternalStream(ctx.stream))
    ctx.sync()
    return s.elapsed_time(e) / 1e3 / reps


def timed_host(fn, reps):
    out = fn()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t0) / reps, out


def run(ctx, n, reps, rng):
    import torch
    t = lambda b: torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()
    u32 = lambda v: torch.from_numpy(np.ascontiguousarray(v, np.uint32).view(np.int32).copy()).cuda()
    u64 = lambda v: torch.from_numpy(np.ascontiguousarray(v, np.uint64).view(np.int64).copy()).cuda()
    zeros = lambda k: torch.zeros(k, dtype=torch.uint8, device="cuda")
    rows = lambda x, size: [x[size * i:size * (i + 1)] for i in range(n)]
    res = {}
    # keys
    seeds = [b"bench seed %d" % i for i in range(n)]
    sec, (sks, dks, eks) = timed_host(lambda: zk.keys_from_seed(ctx, seeds), reps)
    ds, doff, kout = t(b"".join(seeds)), u64(zk.message_offsets(seeds)), [zeros(32 * n) for _ in range(3)]
    dsec = timed_device(ctx, lambda: zk.keys_from_seed_device(ctx, n, ds.data_ptr(), doff.data_ptr(), *(o.data_ptr() for o in kout)), reps)
    assert [rows(o.cpu().numpy().tobytes(), 32) for o in kout] == [sks, dks, eks]
    for i in (0, n // 2, n - 1):
        assert (sks[i], dks[i], eks[i]) == tb.keys(seeds[i])
    h = min(n, HOST_ROWS)
    t0 = time.perf_counter()
    want = tc.keys(seeds[:h])
    hsec = time.perf_counter() - t0
    assert list(want) == [sks[:h], dks[:h], eks[:h]]
    res["keys_per_s"] = {"device": n / dsec, "host_buffers": n / sec, "host_cores": h / hsec}
    # fields
    snd, rcp = rng.integers(0, n, n), rng.integers(0, n, n)
    fs = lambda: int.from_bytes(rng.bytes(64), "little") % rj.R_J
    amounts, fees = [int(v) for v in rng.integers(0, 10 ** 6, n)], [int(v) for v in rng.integers(0, 1000, n)]
    rs, alphas = [fs() for _ in range(n)], [fs() for _ in range(n)]
    g = zk.g_epoch(ctx, [1])[0]
    f_sks, f_eks = [sks[s] for s in snd], [eks[r] for r in rcp]
    sec, (fields, rsks, fdks, st) = timed_host(lambda: zk.confidential_fields(ctx, f_sks, f_eks, amounts, fees, rs, alphas, g), reps)
    assert st == [0] * n and fdks == [dks[s] for s in snd]
    sc = lambda v: b"".join(x.to_bytes(32, "little") for x in v)
    ins = [t(b"".join(f_sks)), t(b"".join(f_eks)), u32(amounts), u32(fees), t(sc(rs)), t(sc(alphas)), t(g)]
    fout = [zeros(288 * n), zeros(32 * n), zeros(32 * n), zeros(n)]
    dsec = timed_device(ctx, lambda: zk.confidential_fields_device(ctx, n, *(x.data_ptr() for x in ins + fout)), reps)
    assert rows(fout[0].cpu().numpy().tobytes(), 288) == [b"".join(f[k] for k in zk.CONFIDENTIAL_FIELDS) for f in fields]
    assert rows(fout[1].cpu().numpy().tobytes(), 32) == rsks
    dec = zk.elgamal_decrypt(ctx, fdks, [f["amount_sender"] + f["randomness"] for f in fields])
    assert dec == ([zk.ELGAMAL_OK] * n, amounts)
    for i in (0, n - 1):
        want = tb.confidential_fields(int.from_bytes(f_sks[i], "little"), f_eks[i], amounts[i], fees[i], rs[i], alphas[i], g)
        assert (b"".join(fields[i][k] for k in zk.CONFIDENTIAL_FIELDS), rsks[i], fdks[i], st[i]) == want
    t0 = time.perf_counter()
    want = tc.confidential_fields(b"".join(f_sks[:h]), b"".join(f_eks[:h]), amounts[:h], fees[:h], sc(rs[:h]), sc(alphas[:h]), g)
    hsec = time.perf_counter() - t0
    assert want == [(b"".join(fields[i][k] for k in zk.CONFIDENTIAL_FIELDS), rsks[i], fdks[i], st[i]) for i in range(h)]
    res["fields_per_s"] = {"device": n / dsec, "host_buffers": n / sec, "host_cores": h / hsec}
    # signatures with rsk over 100-byte messages
    msgs = [rng.bytes(100) for _ in range(n)]
    ts = [rng.bytes(80) for _ in range(n)]
    sec, sigs = timed_host(lambda: zk.redjubjub_sign(ctx, rsks, msgs, ts), reps)
    dsk, dts, dm, dmo, sout = t(b"".join(rsks)), t(b"".join(ts)), t(b"".join(msgs)), u64(zk.message_offsets(msgs)), zeros(64 * n)
    dsec = timed_device(ctx, lambda: zk.redjubjub_sign_device(ctx, n, dsk.data_ptr(), dts.data_ptr(), dm.data_ptr(), dmo.data_ptr(),
                                                              sout.data_ptr()), reps)
    assert rows(sout.cpu().numpy().tobytes(), 64) == sigs
    assert zk.redjubjub_verify(ctx, [f["rvk"] for f in fields], sigs, msgs) == [zk.REDJUBJUB_OK] * n
    assert sigs[0] == rj.sign(int.from_bytes(rsks[0], "little"), msgs[0], ts[0])
    t0 = time.perf_counter()
    want = cj.redjubjub_sign([int.from_bytes(k, "little") for k in rsks[:h]], b"".join(ts[:h]), msgs[:h])
    hsec = time.perf_counter() - t0
    assert want == b"".join(sigs[:h])
    res["signatures_per_s"] = {"device": n / dsec, "host_buffers": n / sec, "host_cores": h / hsec}
    for v in res.values():
        v["device_over_host_cores"] = v["device"] / v["host_cores"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8192,65536")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    name, power = card()
    ctx = zk.Context(0)
    rng = np.random.default_rng(7)
    tc.lib(), cj.lib()                                   # compiled before anything is timed
    out = {"gpu": name, "power_limit": power, "reps": a.reps, "host_threads": tc.threads(), "host_rows": HOST_ROWS, "results_checked": True}
    for n in [int(s) for s in a.sizes.split(",")]:
        out[str(n)] = {k: {f: round(v, 2) for f, v in d.items()} for k, d in run(ctx, n, a.reps, rng).items()}
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
