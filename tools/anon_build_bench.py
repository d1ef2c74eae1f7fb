#!/usr/bin/env python3
"""Throughput of building anonymous transfers on the device (zk_anonymous_fields_batch): rows per second for batches of
8192 and 65536 rows over key tables of 1024 and 65536 keys, device-resident (the _device form on torch buffers, CUDA
events) and from host buffers (the host form through groth16, wall clock, copies and the wrapper's packing included),
with confidential fields (zk_confidential_fields_batch) timed the same way in the same run for comparison.  Every output
of the run is checked: the device and host forms agree byte for byte; every recipient's ciphertext decrypts to its amount
and, on the first DECOY_ROWS rows, every decoy's to 0 under the decryption key of its account (zk_elgamal_decrypt_batch);
and the first HOST_ROWS rows equal the C oracle's.  The host baseline is that C oracle (tests/jubjub_oracle/
anon_build_oracle.c) on all host cores, timed on those HOST_ROWS rows.  Prints one JSON line with the card's name and power
limit, read in the same run.

The bound: about 47 k Fr products per row (11 variable-base products of ~3.8 k, six fixed-base products of 448, 13
inversions of ~300), from operation counts only; at the calibrated 5.24e10 Fr products/s of DESIGN.md §3 that is about
1.1 M rows/s, and "of_bound" is the device rate over it.

--profile: one call of each size under torch.profiler instead, and one JSON line of CUDA time per kernel.

Usage: python tools/anon_build_bench.py [--sizes 8192,65536] [--tables 1024,65536] [--reps 5] [--profile]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.jubjub_oracle import anon_build_coracle as abc  # noqa: E402
from tests.jubjub_oracle import redjubjub as rj     # noqa: E402
from zero_chain_b200 import groth16 as zk           # noqa: E402

HOST_ROWS = 512      # rows the host baseline computes (it runs at a few hundred rows per second)
DECOY_ROWS = 2048    # rows whose ten decoy ciphertexts are decrypted too
PRODUCTS_PER_ROW = 47_000
FR_PRODUCTS_PER_S = 5.24e10


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


class Inputs:
    """n rows over a table of the first n_keys derived keys: distinct ring members, random positions"""

    def __init__(self, ctx, keys, n, n_keys, rng):
        import torch
        self.sks_all, self.dks, self.eks = (k[:n_keys] for k in keys)
        self.n, self.n_keys = n, n_keys
        self.snd = rng.integers(0, n_keys, n)
        self.rings = rng.integers(0, n_keys, (n, 11)).astype(np.uint32)
        self.pos = np.array([rng.choice(12, 2, replace=False) for _ in range(n)], np.uint8)
        self.amounts = rng.integers(0, 10 ** 6, n).astype(np.uint32)
        fs = lambda: (int.from_bytes(rng.bytes(64), "little") % rj.R_J).to_bytes(32, "little")
        self.sks = b"".join(self.sks_all[s] for s in self.snd)
        self.rs, self.alphas = b"".join(fs() for _ in range(n)), b"".join(fs() for _ in range(n))
        self.g = zk.g_epoch(ctx, [1])[0]
        t = lambda b: torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()
        u32 = lambda v: torch.from_numpy(np.ascontiguousarray(v, np.uint32).reshape(-1).view(np.int32).copy()).cuda()
        self.d_in = [t(b"".join(self.eks)), t(self.sks), u32(self.rings), t(self.pos.tobytes()), u32(self.amounts), t(self.rs), t(self.alphas),
                     t(self.g)]
        self.d_out = [torch.zeros(k, dtype=torch.uint8, device="cuda") for k in (864 * n, 32 * n, 32 * n, n)]

    def device(self, ctx):
        ky, sk, rg, ps, am, r, al, g = (x.data_ptr() for x in self.d_in)
        zk.anonymous_fields_device(ctx, self.n_keys, ky, self.n, sk, rg, ps, am, r, al, g, *(x.data_ptr() for x in self.d_out))

    def host(self, ctx):
        return zk.anonymous_fields(ctx, self.eks, self.sks, self.rings, self.pos, self.amounts, self.rs, self.alphas, self.g)


def check(ctx, inp, host_out):
    """every output of the run: the device form equals the host form; the ciphertexts decrypt"""
    fields, rsks, fdks, st = host_out
    n = inp.n
    assert st == [0] * n and fdks == [inp.dks[s] for s in inp.snd]
    flat = b"".join(b"".join(f["enc_keys"]) + b"".join(f["left_ciphertexts"]) + f["right_ciphertext"] + f["rvk"] + f["nonce"] for f in fields)
    assert inp.d_out[0].cpu().numpy().tobytes() == flat
    assert inp.d_out[1].cpu().numpy().tobytes() == b"".join(rsks) and inp.d_out[2].cpu().numpy().tobytes() == b"".join(fdks)
    assert not inp.d_out[3].cpu().numpy().any()
    keys, cts, want = [], [], []
    for i, f in enumerate(fields):
        s, t = int(inp.pos[i, 0]), int(inp.pos[i, 1])
        keys.append(inp.dks[inp.rings[i, 0]]); cts.append(f["left_ciphertexts"][t] + f["right_ciphertext"]); want.append(int(inp.amounts[i]))
        if i < DECOY_ROWS:
            others = [p for p in range(12) if p not in (s, t)]
            for p, k in zip(others, inp.rings[i, 1:]):
                keys.append(inp.dks[k]); cts.append(f["left_ciphertexts"][p] + f["right_ciphertext"]); want.append(0)
    assert zk.elgamal_decrypt(ctx, keys, cts) == ([zk.ELGAMAL_OK] * len(want), want)
    return flat, rsks, fdks


def run(ctx, keys, n, n_keys, reps, rng):
    inp = Inputs(ctx, keys, n, n_keys, rng)
    sec, out = timed_host(lambda: inp.host(ctx), reps)
    dsec = timed_device(ctx, lambda: inp.device(ctx), reps)
    flat, rsks, fdks = check(ctx, inp, out)
    h = min(n, HOST_ROWS)
    t0 = time.perf_counter()
    want = abc.anonymous_fields(b"".join(inp.eks), inp.sks[:32 * h], inp.rings[:h], inp.pos[:h], inp.amounts[:h], inp.rs[:32 * h],
                               inp.alphas[:32 * h], inp.g)
    hsec = time.perf_counter() - t0
    assert want == [(flat[864 * i:864 * (i + 1)], rsks[i], fdks[i], 0) for i in range(h)]
    dev = n / dsec
    return {"device": dev, "host_buffers": n / sec, "host_cores": h / hsec, "device_over_host_cores": dev * hsec / h,
            "of_bound": dev / (FR_PRODUCTS_PER_S / PRODUCTS_PER_ROW)}


def run_confidential(ctx, keys, n, reps, rng):
    import torch
    sks, dks, eks = keys
    nk = len(eks)
    snd, rcp = rng.integers(0, nk, n), rng.integers(0, nk, n)
    fs = lambda: int.from_bytes(rng.bytes(64), "little") % rj.R_J
    amounts, fees = [int(v) for v in rng.integers(0, 10 ** 6, n)], [int(v) for v in rng.integers(0, 1000, n)]
    rs, alphas = [fs() for _ in range(n)], [fs() for _ in range(n)]
    g = zk.g_epoch(ctx, [1])[0]
    f_sks, f_eks = [sks[s] for s in snd], [eks[r] for r in rcp]
    t = lambda b: torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()
    u32 = lambda v: torch.from_numpy(np.ascontiguousarray(v, np.uint32).view(np.int32).copy()).cuda()
    sc = lambda v: b"".join(x.to_bytes(32, "little") for x in v)
    ins = [t(b"".join(f_sks)), t(b"".join(f_eks)), u32(amounts), u32(fees), t(sc(rs)), t(sc(alphas)), t(g)]
    out = [torch.zeros(k, dtype=torch.uint8, device="cuda") for k in (288 * n, 32 * n, 32 * n, n)]
    dsec = timed_device(ctx, lambda: zk.confidential_fields_device(ctx, n, *(x.data_ptr() for x in ins + out)), reps)
    fields, _, fdks, st = zk.confidential_fields(ctx, f_sks, f_eks, amounts, fees, rs, alphas, g)
    assert st == [0] * n and out[0].cpu().numpy().tobytes() == b"".join(b"".join(f[k] for k in zk.CONFIDENTIAL_FIELDS) for f in fields)
    assert zk.elgamal_decrypt(ctx, [dks[r] for r in rcp], [f["amount_recipient"] + f["randomness"] for f in fields]) == \
        ([zk.ELGAMAL_OK] * n, amounts)
    return {"device": n / dsec}


def profile(ctx, keys, sizes, tables, rng):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    inps = [Inputs(ctx, keys, n, nk, rng) for n in sizes for nk in tables]
    for inp in inps:
        inp.device(ctx)
    ctx.sync()
    out = {}
    for inp in inps:
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            inp.device(ctx)
            ctx.sync()
            torch.cuda.synchronize()
        k = {e.key: round(e.device_time_total / 1e3, 3) for e in p.key_averages() if e.device_time_total > 0}
        out["%d rows, %d keys" % (inp.n, inp.n_keys)] = dict(sorted(k.items(), key=lambda kv: -kv[1]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8192,65536")
    ap.add_argument("--tables", default="1024,65536")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    sizes, tables = [int(s) for s in a.sizes.split(",")], [int(s) for s in a.tables.split(",")]
    name, power = card()
    ctx = zk.Context(0)
    rng = np.random.default_rng(11)
    keys = zk.keys_from_seed(ctx, [b"anon bench %d" % i for i in range(max(tables))])
    if a.profile:
        print(json.dumps({"gpu": name, "power_limit": power, "kernel_ms": profile(ctx, keys, sizes, tables, rng)}))
        ctx.close()
        return
    abc.lib()                                             # compiled before anything is timed
    out = {"gpu": name, "power_limit": power, "reps": a.reps, "host_threads": abc.threads(), "host_rows": HOST_ROWS,
           "bound_rows_per_s": round(FR_PRODUCTS_PER_S / PRODUCTS_PER_ROW), "results_checked": True}
    for n in sizes:
        row = {}
        for nk in tables:
            row["anonymous_per_s_%d_keys" % nk] = {k: round(v, 4 if k == "of_bound" else 2) for k, v in run(ctx, keys, n, nk, a.reps, rng).items()}
        row["confidential_per_s"] = {k: round(v, 2) for k, v in run_confidential(ctx, keys, n, a.reps, rng).items()}
        out[str(n)] = row
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
