#!/usr/bin/env python3
"""Throughput of wallet-key derivation on the device (zk_xsk_master_batch, zk_xsk_derive_batch, zk_xpgk_derive_batch):
rows per second of the _device forms on torch buffers, timed with CUDA events, for
  master          xsk_master of N seeds of 64 bytes, with xpgk, dk and ek
  scan_outputs    xsk_derive of one parent with N indices (account scanning), with xpgk, dk and ek
  scan_bare       the same with no optional output: hashes and one Fs addition per row
  level_outputs   xsk_derive of N distinct parents, one index each (one level of N paths), with xpgk, dk and ek
  watch_only      xpgk_derive of one parent with N non-hardened indices, with dk and ek
Every output of the timed run is checked byte for byte against the C oracle (tests/jubjub_oracle/hd_keys_oracle.c), which
also gives the host baseline: the oracle on all host cores, timed on the same N rows.  Prints one JSON line with the card's
name and power limit, read in the same run.

Usage: python tools/hd_bench.py [--rows 65536] [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.jubjub_oracle import hd_coracle as hc   # noqa: E402
from zero_chain_b200 import groth16 as zk          # noqa: E402

XK = zk.XK_BYTES


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


def _t(b: bytes):
    import torch
    return torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()


def _u32(v):
    import torch
    return torch.from_numpy(np.ascontiguousarray(v, np.uint32).view(np.int32).copy()).cuda()


def _z(k: int):
    import torch
    return torch.zeros(k, dtype=torch.uint8, device="cuda")


def _rows(t, size, n):
    b = t.cpu().numpy().tobytes()
    return [b[size * i:size * (i + 1)] for i in range(n)]


def _oracle(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, time.perf_counter() - t0


def bench_master(ctx, n, reps, rng):
    seeds = [rng.bytes(64) for _ in range(n)]
    sd, off = _t(b"".join(seeds)), _t(zk.message_offsets(seeds).tobytes())
    outs = [_z(XK * n), _z(XK * n), _z(32 * n), _z(32 * n)]
    sec = timed_device(ctx, lambda: zk.xsk_master_device(ctx, n, sd.data_ptr(), off.data_ptr(), *(o.data_ptr() for o in outs)), reps)
    want, hsec = _oracle(lambda: hc.master(seeds))
    got = list(zip(_rows(outs[0], XK, n), _rows(outs[1], XK, n), _rows(outs[2], 32, n), _rows(outs[3], 32, n)))
    assert got == want
    return n / sec, n / hsec


def bench_xsk(ctx, parents, pidx, cidx, outputs, reps):
    n = len(pidx)
    pb, pi, ci = _t(b"".join(parents)), _u32(pidx), _u32(cidx)
    outs = [_z(XK * n)] + ([_z(XK * n), _z(32 * n), _z(32 * n)] if outputs else [None] * 3) + [_z(n)]
    ptrs = [o.data_ptr() if o is not None else 0 for o in outs]
    sec = timed_device(ctx, lambda: zk.xsk_derive_device(ctx, len(parents), pb.data_ptr(), n, pi.data_ptr(), ci.data_ptr(), *ptrs), reps)
    want, hsec = _oracle(lambda: hc.xsk_derive(parents, pidx, cidx, outputs=outputs))
    st = [int(v) for v in outs[4].cpu().numpy()]
    assert st == [w[4] for w in want] == [0] * n
    assert _rows(outs[0], XK, n) == [w[0] for w in want]
    if outputs:
        assert _rows(outs[1], XK, n) == [w[1] for w in want]
        assert _rows(outs[2], 32, n) == [w[2] for w in want] and _rows(outs[3], 32, n) == [w[3] for w in want]
    return n / sec, n / hsec


def bench_xpgk(ctx, parents, pidx, cidx, reps):
    n = len(pidx)
    pb, pi, ci = _t(b"".join(parents)), _u32(pidx), _u32(cidx)
    outs = [_z(XK * n), _z(32 * n), _z(32 * n), _z(n)]
    sec = timed_device(ctx, lambda: zk.xpgk_derive_device(ctx, len(parents), pb.data_ptr(), n, pi.data_ptr(), ci.data_ptr(),
                                                          *(o.data_ptr() for o in outs)), reps)
    want, hsec = _oracle(lambda: hc.xpgk_derive(parents, pidx, cidx))
    got = list(zip(_rows(outs[0], XK, n), _rows(outs[1], 32, n), _rows(outs[2], 32, n), [int(v) for v in outs[3].cpu().numpy()]))
    assert got == want and all(w[3] == 0 for w in want)
    return n / sec, n / hsec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    n = a.rows
    name, power = card()
    ctx = zk.Context(0)
    hc.lib()                                              # compiled before anything is timed
    rng = np.random.default_rng(5)
    master = zk.xsk_master(ctx, [b"bench wallet seed"])
    one, idx = master[0], [int(v) for v in rng.integers(0, 2 ** 31, n)]
    level = zk.xsk_derive(ctx, one, [0] * n, [2 ** 31 + i for i in range(n)], xpgk=False, dk=False, ek=False)[0]
    res = {"master": bench_master(ctx, n, a.reps, rng),
           "scan_outputs": bench_xsk(ctx, one, [0] * n, idx, True, a.reps),
           "scan_bare": bench_xsk(ctx, one, [0] * n, idx, False, a.reps),
           "level_outputs": bench_xsk(ctx, level, list(range(n)), idx, True, a.reps),
           "watch_only": bench_xpgk(ctx, master[1], [0] * n, idx, a.reps)}
    out = {"gpu": name, "power_limit": power, "rows": n, "reps": a.reps, "host_threads": hc.threads(), "results_checked": True}
    for k, (dev, host) in res.items():
        out[k] = {"device_per_s": round(dev, 1), "host_cores_per_s": round(host, 1), "device_over_host_cores": round(dev / host, 1)}
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
