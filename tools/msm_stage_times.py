"""Where the time of the headline G1 MSM goes, kernel by kernel, without Nsight.

    python tools/msm_stage_times.py [--out DIR] [--log-n 20] [--steps 10] [--warmup 3]

Runs the shape bench.py measures (2^20 uniform subgroup bases b_i * G with window tables, the library's default window,
seeded scalars) and prints one JSON line:
- `blocking_ms` / `in_flight_ms`: wall time per MSM as one blocking call and with two MSMs in flight on two contexts (CUDA
  events, profiler off);
- `stage_ms`: the bucket-accumulation stage (batched-affine rounds + XYZZ pass) per MSM, from zk_ctx_profile's events;
- `kernels_ms`: per MSM, the summed kernel time of each part (sort, every round's forward / invert / backward / offsets, task
  setup, accumulate, tail) from a separate blocking run under torch.profiler (CUDA activities).  `rounds` also gives each
  round's wall span and how much of its forward and invert time lay under a running backward pass (0 while a round's
  kernels run one after another on one stream);
- `byte_model`: for every round's forward and backward pass, the DRAM bytes per pair the code has to move (a MODEL worked out
  from the kernels, not a measurement), the round's pair count estimated from the shape, and the effective GB/s those bytes
  make over the measured kernel time;
- the card's name and power limit.
The profiled runs' chrome traces are written to DIR (a new temporary directory if --out is not given).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_SETS = 8                     # as bench.py: distinct scalar vectors, together larger than L2


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu_name": q[0].strip(), "power_limit_w": float(q[1])}
    except Exception as e:
        return {"gpu_name": None, "power_limit_w": None, "error": repr(e)}


def kernel_events(path):
    with open(path) as f:
        tr = json.load(f)
    ev = [e for e in tr.get("traceEvents", []) if e.get("cat") == "kernel"]
    ev.sort(key=lambda e: e["ts"])
    return [(e["name"], float(e["ts"]), float(e["ts"]) + float(e["dur"])) for e in ev]


def short(name):
    base = name.split("(")[0].split("<")[0]
    return base.replace("void ", "").split("::")[-1].strip()


def overlap(a0, a1, spans):
    return sum(max(0.0, min(a1, b1) - max(a0, b0)) for b0, b1 in spans)


def breakdown(events):
    """Split a blocking run's kernels into MSMs (each starts with k_msm_digits) and attribute each kernel to a part."""
    msms, cur = [], None
    for e in events:
        if short(e[0]) == "k_msm_digits":
            cur = []
            msms.append(cur)
        if cur is not None:
            cur.append(e)
    parts, spans, walls = {}, {}, {}        # spans[round][part]: kernel intervals; walls[round]: first-to-last per MSM
    for m in msms:
        phase, rnd, inv_ends, first_last = "sort", 0, [], {}     # inv_ends: (end, round) of every inversion so far
        for name, t0, t1 in m:
            k, key, r = short(name), None, None
            if k == "k_half_sizes":
                phase, rnd = "rounds", rnd + 1
                key = "offsets"
            elif k in ("k_ba_forward", "k_ba_invert"):
                key, r = k[5:], rnd
                if k == "k_ba_invert":
                    inv_ends.append((t1, rnd))
            elif k == "k_ba_backward":       # the round of the last inversion that ended before it started
                key, r = "backward", max((x for x in inv_ends if x[0] <= t0), default=(0, rnd))[1]
            elif k == "k_pick_task_len":
                phase = "task_setup"
            elif k == "k_accumulate":
                phase, key = "tail", "accumulate"
            if key is None:
                key = "offsets" if phase == "rounds" else phase
            if key in ("offsets", "forward", "invert", "backward"):
                r = rnd if r is None else r
                spans.setdefault(r, {}).setdefault(key, []).append((t0, t1))
                if key != "offsets":
                    a, b = first_last.get(r, (t0, t1))
                    first_last[r] = (min(a, t0), max(b, t1))
                key = "round%d.%s" % (r, key)
            parts[key] = parts.get(key, 0.0) + (t1 - t0)
        for r, (a, b) in first_last.items():
            walls.setdefault(r, []).append(b - a)
    n = max(1, len(msms))
    out_rounds = {}
    for r, sp in sorted(spans.items()):
        bwd = sp.get("backward", [])
        fi = sp.get("forward", []) + sp.get("invert", [])
        out_rounds["round%d" % r] = {"wall_span_ms": float(np.mean(walls.get(r, [0.0]))) / 1e3, "slabs": len(bwd) / n,
                                     "forward_invert_ms": sum(b - a for a, b in fi) / n / 1e3,
                                     "forward_invert_under_backward_ms": sum(overlap(a, b, bwd) for a, b in fi) / n / 1e3}
    return {k: v / n / 1e3 for k, v in sorted(parts.items())}, out_rounds, len(msms)


FQ = 48                        # bytes of an Fq element; a G1 affine point is 2 FQ
SECTOR = 32                    # DRAM / L2 sector


def sectors(nbytes, offset=0):
    """Bytes moved at sector granularity for nbytes at a random address with the given offset within a sector."""
    return ((offset + nbytes + SECTOR - 1) // SECTOR) * SECTOR


def byte_model(n, window_bits, rounds):
    """DRAM bytes per pair of each batched-affine pass (msm_batchaff.cuh), from the data layout, and the pair counts of the
    rounds estimated from the shape: E = n W entries (zero digits ignored), each round pairs half of its inputs and keeps one
    odd leftover in about half of the 2^(c-1) buckets.  Round 1 gathers window-table rows (x | y, 96-byte rows, so a row starts
    on a sector) at random; later rounds read the previous round's x and y planes in order.  Per pair:
      forward   round 1: two entry codes (8) + two x gathers (2 x 64 at sector granularity) + prefix store (48)
                round r>1: two x (96) + prefix store (48)
      backward  round 1: two entry codes (8) + two row gathers (2 x 96) + prefix (48) + the sum's x and y stored (96)
                round r>1: two points (192) + prefix (48) + the sum's x and y stored (96)
    The bucket offsets are read once per bucket crossed and are left out."""
    W = 255 // window_bits + 1
    nb = 1 << (window_bits - 1)
    entries, out = float(n * W), {}
    for r in range(1, rounds + 1):
        pairs = entries / 2 - nb / 4
        if r == 1:
            fwd = 8 + 2 * sectors(FQ) + FQ
            bwd = 8 + 2 * sectors(2 * FQ) + FQ + 2 * FQ
        else:
            fwd = 2 * FQ + FQ
            bwd = 2 * 2 * FQ + FQ + 2 * FQ
        out["round%d" % r] = {"entries": entries, "pairs": pairs, "forward_bytes_per_pair": fwd, "backward_bytes_per_pair": bwd}
        entries = pairs + nb / 2           # outputs: the pairs' sums and the odd leftovers
    return out


def with_rates(model, parts):
    """Adds each pass's modelled bytes and the effective GB/s over its measured time (kernels_ms, per MSM)."""
    for rnd, m in model.items():
        for p in ("forward", "backward"):
            ms = parts.get("%s.%s" % (rnd, p))
            m["%s_model_bytes" % p] = m["pairs"] * m["%s_bytes_per_pair" % p]
            m["%s_ms" % p] = ms
            m["%s_effective_GBps" % p] = m["%s_model_bytes" % p] / (ms * 1e-3) / 1e9 if ms else None
    return model


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for the profiler traces (default: a new temporary directory)")
    ap.add_argument("--log-n", dest="log_n", type=int, default=20)
    ap.add_argument("--window-bits", dest="window_bits", type=int, default=0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--label", default="msm")
    args = ap.parse_args()
    out = args.out or tempfile.mkdtemp(prefix="msm_stage_times_")
    os.makedirs(out, exist_ok=True)

    import torch
    from torch.profiler import ProfilerActivity, profile
    from zero_chain_b200 import groth16 as zk
    from zero_chain_b200 import synthetic as sy

    n = 1 << args.log_n
    ctx, ctx2 = zk.Context(0), zk.Context(0)
    bases_limbs = zk.scalar_mul_many(ctx, 1, zk.G1_GENERATOR, sy.random_fr_limbs(n, 7))      # bench.py's seeds
    bases = zk.Bases(ctx, 1, bases_limbs, window_bits=args.window_bits, precompute=True)
    del bases_limbs
    d_sets = [torch.from_numpy(sy.random_fr_limbs(n, 1000 + k).view(np.int64)).cuda() for k in range(N_SETS)]
    torch.cuda.synchronize()

    def blocking(k):
        return zk.multiexp_device(bases, d_sets[k % N_SETS].data_ptr(), n)

    def in_flight(k0, k1):
        ctxs, pending, res = (ctx, ctx2), [None, None], {}
        for k in range(k0, k1):
            c = k % 2
            if pending[c] is not None:
                res[pending[c]] = zk.multiexp_end(ctxs[c], bases)
            zk.multiexp_device_begin(ctxs[c], bases, d_sets[k % N_SETS].data_ptr(), n)
            pending[c] = k
        for k in sorted(x for x in pending if x is not None):
            res[k] = zk.multiexp_end(ctxs[k % 2], bases)
        return res

    def wall(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1e3 / args.steps

    for k in range(args.warmup):
        blocking(k)
    in_flight(0, max(2, args.warmup))
    res_b = {}
    blocking_ms = wall(lambda: res_b.update({k: blocking(k) for k in range(args.steps)}))
    res_p = {}
    in_flight_ms = wall(lambda: res_p.update(in_flight(0, args.steps)))
    if res_b != res_p:
        raise SystemExit("PARITY FAILURE: blocking and in-flight MSM results differ")

    ctx.profile(True)
    for k in range(args.steps):
        blocking(k)
    stage_ms, launches = ctx.profile_read()
    ctx.profile(False)

    traces = {}
    for what, fn in (("blocking", lambda: [blocking(k) for k in range(args.steps)]), ("in_flight", lambda: in_flight(0, args.steps))):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        traces[what] = os.path.join(out, "%s_%s.pt.trace.json" % (args.label, what))
        prof.export_chrome_trace(traces[what])

    parts, rounds, n_msm = breakdown(kernel_events(traces["blocking"]))
    model = with_rates(byte_model(n, bases.window_bits, len(rounds)), parts)
    by_name = {}
    for name, t0, t1 in kernel_events(traces["in_flight"]):
        by_name[short(name)] = by_name.get(short(name), 0.0) + (t1 - t0) / args.steps / 1e3
    line = {"label": args.label, "log_n": args.log_n, "window_bits": bases.window_bits, "steps": args.steps,
            "blocking_ms": blocking_ms, "in_flight_ms": in_flight_ms,
            "stage_ms": stage_ms / max(1, launches), "kernels_ms": parts, "rounds": rounds, "byte_model": model, "profiled_msms": n_msm,
            "in_flight_kernels_ms": dict(sorted(by_name.items(), key=lambda kv: -kv[1])),
            "card": card(), "traces": traces}
    with open(os.path.join(out, "%s.json" % args.label), "w") as f:
        json.dump(line, f, indent=1)
    print(json.dumps(line), flush=True)
    bases.free()
    ctx2.close()
    ctx.close()


if __name__ == "__main__":
    main()
