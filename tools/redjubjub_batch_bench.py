"""Throughput of RedJubjub batch verification (zk_redjubjub_batch_verify) against the per-signature kernel
(zk_redjubjub_verify_batch), one JSON line:
  batch_sigs_per_s_device[batch/msg_len]   zk_redjubjub_batch_verify_device, device-resident inputs
  per_sig_sigs_per_s_device[batch/msg_len] zk_redjubjub_verify_batch_device on the same inputs, alternated with the line above
                                           (median of --reps A/B pairs in one process)
  batch_sigs_per_s_host[batch/msg_len]     the host form, copies included
  msm_points_per_s                         zk_jubjub_msm alone over 2^17 points
  kernel_us[batch]                         per-kernel device time of one batch check (torch.profiler), 32-byte messages
  host_batch_sigs_per_s[msg_len]           the C oracle's batch_verify on every host core (OpenMP), the CPU baseline
with the card's name and power limit read in the same run.  Every verdict is checked inside the run: each timed batch
must pass, and a copy with one swapped signature must fail.
Usage: python tools/redjubjub_batch_bench.py [--reps 5]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests.jubjub_oracle import rj_coracle as cj              # noqa: E402
from tests.jubjub_oracle import redjubjub as rj               # noqa: E402
from tests.jubjub_oracle import rjb_coracle as cjb            # noqa: E402
from tools.redjubjub_bench import corpus, to_dev              # noqa: E402
from tools.verify_tx_bench import card, timed                 # noqa: E402
from zero_chain_b200 import groth16 as zk                     # noqa: E402


def zs_bytes(rng, n):
    return b"".join((int.from_bytes(rng.bytes(64), "little") % rj.R_J).to_bytes(32, "little") for _ in range(n))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    ctx = zk.Context(0)
    rng = np.random.default_rng(1)
    out = {"metric": "redjubjub_batch_verify", "batch_sigs_per_s_device": {}, "per_sig_sigs_per_s_device": {},
           "batch_sigs_per_s_host": {}, "ab_ms": {}, "kernel_us": {}, "host_batch_sigs_per_s": {}}
    for msg_len in (32, 256):
        vk, sg, msgs, _ = corpus(rng, msg_len, 65536)
        for n in (8192, 65536):
            v, s, m = vk[:32 * n], sg[:64 * n], msgs[:n]
            z = zs_bytes(rng, n)
            key = "%d/%dB" % (n, msg_len)
            assert zk.redjubjub_batch_verify(ctx, v, s, m, z) == (1, None)
            swapped = s[:64] + s[128:192] + s[128:]                  # entry 1's signature on entry 0
            assert zk.redjubjub_batch_verify(ctx, v, swapped, m, z)[0] == 0
            out["batch_sigs_per_s_host"][key] = n / timed(lambda: zk.redjubjub_batch_verify(ctx, v, s, m, z), a.reps)
            dvk, dsg, dm, dz = to_dev(v), to_dev(s), to_dev(b"".join(m)), to_dev(z)
            doff = torch.from_numpy(zk.message_offsets(m).view(np.int64)).cuda()
            dver = torch.zeros(1, dtype=torch.uint8, device="cuda")
            dvs = torch.zeros(n, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()

            def batch():
                zk.redjubjub_batch_verify_device(ctx, n, dvk.data_ptr(), dsg.data_ptr(), dm.data_ptr(), doff.data_ptr(), dz.data_ptr(),
                                                 dver.data_ptr()); ctx.sync()

            def per_sig():
                zk.redjubjub_verify_device(ctx, n, dvk.data_ptr(), dsg.data_ptr(), dm.data_ptr(), doff.data_ptr(), dvs.data_ptr()); ctx.sync()

            batch(); per_sig()
            ta, tb = [], []
            for _ in range(a.reps):                                  # A/B alternated in one process
                dver.zero_(); ta.append(timed(batch, 1)); assert int(dver.cpu()[0]) == 1
                dvs.zero_(); tb.append(timed(per_sig, 1)); assert bool((dvs == 1).all())
            out["batch_sigs_per_s_device"][key] = n / float(np.median(ta))
            out["per_sig_sigs_per_s_device"][key] = n / float(np.median(tb))
            out["ab_ms"][key] = {"batch": [round(x * 1e3, 3) for x in ta], "per_sig": [round(x * 1e3, 3) for x in tb]}
            if msg_len == 32:
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    batch()
                ku = {}
                for ev in prof.key_averages():
                    if ev.device_type == torch.autograd.DeviceType.CUDA:
                        ku[ev.key[:40]] = round(ev.device_time_total, 1)
                out["kernel_us"][str(n)] = dict(sorted(ku.items(), key=lambda kv: -kv[1]))
        hn = 2048
        hz = zs_bytes(rng, hn)
        assert cjb.redjubjub_batch_verify(vk[:32 * hn], sg[:64 * hn], msgs[:hn], hz) == (1, None)
        t = timed(lambda: cjb.redjubjub_batch_verify(vk[:32 * hn], sg[:64 * hn], msgs[:hn], hz), max(1, a.reps // 2))
        out["host_batch_sigs_per_s"]["%dB" % msg_len] = hn / t

    # the MSM alone: 2^17 points k_i P_G, checked against the closed form
    n = 1 << 17
    ks = [int.from_bytes(rng.bytes(32), "little") % rj.R_J for _ in range(1024)]
    base = cj.redjubjub_public_key(ks)
    idx = np.arange(n) % 1024
    pts = np.frombuffer(base, np.uint8).reshape(1024, 32)[idx].tobytes()
    ss = [int.from_bytes(rng.bytes(32), "little") % rj.R_J for _ in range(n)]
    sb = b"".join(x.to_bytes(32, "little") for x in ss)
    want = cj.redjubjub_public_key([sum(ks[i % 1024] * x for i, x in enumerate(ss)) % rj.R_J])
    assert zk.jubjub_msm(ctx, pts, sb) == want
    out["msm_points"] = n
    out["msm_points_per_s"] = n / timed(lambda: zk.jubjub_msm(ctx, pts, sb), a.reps)
    name, plimit = card()
    out.update({"gpu_name": name, "power_limit_w": plimit, "host_threads": cj.threads(), "host_cpus": os.cpu_count()})
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
