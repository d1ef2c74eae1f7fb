#!/usr/bin/env python3
"""Measures lifted-ElGamal balance decryption (zk_elgamal_decrypt_batch) and prints one JSON line:
  - the card's name and power limit, read in this run;
  - the first call's table build (the 10^6 multiples of P_G and their index), timed with CUDA events;
  - device-resident decryptions/s at --batch, without and with pending transfers (CUDA events, median of --reps);
  - the host form including its copies (wall clock, median of --reps);
  - the C oracle's reference loop on all host cores: uniform amounts below 10^6, and the None case (the full 10^6 steps).
The corpus is made by the C oracle (random keys, amounts and randomness); nothing is written to the repository tree."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.jubjub_oracle import eg_coracle as ec          # noqa: E402
from tests.jubjub_oracle import pyref as jj               # noqa: E402
from tests.jubjub_oracle import rj_coracle as cj          # noqa: E402
from zero_chain_b200 import groth16 as zk                 # noqa: E402


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], text=True)
        name, power = [s.strip() for s in out.strip().split("\n")[0].split(",")]
        return name, power
    except Exception as e:                                 # the numbers are still printed, with the reason
        return "unknown (%s)" % e, "unknown"


def corpus(n, seed, bound=1_000_000):
    rng = np.random.default_rng(seed)
    keys = [int.from_bytes(rng.bytes(32), "little") % jj.R_J or 1 for _ in range(n)]
    eks = cj.redjubjub_public_key(keys)
    amounts = rng.integers(0, bound, n)
    rs = [int.from_bytes(rng.bytes(32), "little") % jj.R_J for _ in range(2 * n)]
    dks = b"".join(k.to_bytes(32, "little") for k in keys)
    cts = ec.encrypt(amounts // 2, rs[:n], eks)
    pds = ec.encrypt(amounts - amounts // 2, rs[n:], eks)
    return dks, cts, pds, amounts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-n", type=int, default=64, help="ciphertexts per case for the C oracle's loop")
    a = ap.parse_args()
    import torch
    name, power = card()
    stream = torch.cuda.Stream()                           # the context runs on it, so the events bracket its kernels
    ctx = zk.Context(0, stream.cuda_stream)
    n = a.batch
    dks, cts, pds, amounts = corpus(n, 1)
    t = lambda b: torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()
    d_dk, d_ct, d_pd = t(dks), t(cts), t(pds)
    d_val = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_st = torch.zeros(n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def run(pend_ptr):
        zk.elgamal_decrypt_device(ctx, n, d_dk.data_ptr(), d_ct.data_ptr(), pend_ptr, d_val.data_ptr(), d_st.data_ptr())

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    # the first call builds the table; time the build alone with one ciphertext
    e0.record(stream)
    zk.elgamal_decrypt_device(ctx, 1, d_dk.data_ptr(), d_ct.data_ptr(), 0, d_val.data_ptr(), d_st.data_ptr())
    e1.record(stream)
    torch.cuda.synchronize()
    build_ms = e0.elapsed_time(e1)

    def device_rate(pend_ptr):
        run(pend_ptr)
        torch.cuda.synchronize()
        ms = []
        for _ in range(a.reps):
            e0.record(stream)
            run(pend_ptr)
            e1.record(stream)
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return n / (float(np.median(ms)) * 1e-3)

    rate_plain = device_rate(0)
    ok_plain = (d_st.cpu().numpy() == 0).all() and np.array_equal(d_val.cpu().numpy().astype(np.int64), amounts // 2)
    rate_pend = device_rate(d_pd.data_ptr())
    ok_pend = (d_st.cpu().numpy() == 0).all() and np.array_equal(d_val.cpu().numpy().astype(np.int64), amounts)
    wall = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        st, val = zk.elgamal_decrypt(ctx, dks, cts, pds)
        wall.append(time.perf_counter() - t0)
    ok_host = st == [0] * n and val == [int(x) for x in amounts]
    # the C oracle's walk: uniform amounts below 10^6 (the pending halves added), and wrong keys (None: all 10^6 steps)
    hn = a.host_n
    t0 = time.perf_counter()
    hst, hval = ec.decrypt(dks[:32 * hn], cts[:64 * hn], pds[:64 * hn])
    host_uniform = hn / (time.perf_counter() - t0)
    ok_oracle = (hst == 0).all() and np.array_equal(hval.astype(np.int64), amounts[:hn])
    wrong = dks[32:32 * (hn + 1)]
    t0 = time.perf_counter()
    hst, _ = ec.decrypt(wrong, cts[:64 * hn], pds[:64 * hn])
    host_none = hn / (time.perf_counter() - t0)
    ok_oracle = ok_oracle and (hst == 1).all()
    ctx.close()
    print(json.dumps({
        "card": name, "power_limit": power, "batch": n,
        "table_build_ms": round(build_ms, 2),
        "device_decrypt_per_s": round(rate_plain), "device_decrypt_with_pending_per_s": round(rate_pend),
        "host_form_with_pending_per_s": round(n / float(np.median(wall))),
        "oracle_loop_uniform_per_s": round(host_uniform, 1), "oracle_loop_none_per_s": round(host_none, 1),
        "oracle_threads": ec.threads(), "host_n": hn,
        "results_match": bool(ok_plain and ok_pend and ok_host and ok_oracle),
    }))


if __name__ == "__main__":
    main()
