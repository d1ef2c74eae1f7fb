"""CPU check of zk_import_block's shared launch (zero_chain_b200/csrc/import.cuh, compiled with ZK_HOST_EMUL): the sections'
rows compacted at their offsets into one launch, and each section's verdicts read back and decided at its own offset,
give every section exactly what it gets in a launch of its own; a failure in one section never decides a transaction of
another.  The real PTX path is covered by tests/test_gpu_block_import.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ROW = 352
UNDECIDED = 0xFF


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_block_import") / "libemul_block_import.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_block_import.cpp")])
    lib = C.CDLL(so)
    lib.emu_block_launch.restype = C.c_size_t
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def chain_section(rng, n, n_keys, fail_p, undecided_p=0.7):
    """(n_keys, keys, rows, verdicts): row byte 0 is the model verifier's verdict"""
    key = rng.integers(0, n_keys, n).astype(np.uint32)
    rows = rng.integers(0, 256, (n, ROW)).astype(np.uint8)
    rows[:, 0] = [int(rng.choice([0, 2, 4])) if rng.random() < fail_p else 1 for _ in range(n)]
    verdict = np.where(rng.random(n) < undecided_p, UNDECIDED, rng.integers(0, 2, n)).astype(np.uint8)
    return n_keys, key, rows.reshape(-1), verdict


def issue_section(rng, n, fail_p):
    kind = rng.integers(0, 3, n).astype(np.uint8)
    rows = rng.integers(0, 256, (n, ROW)).astype(np.uint8)
    rows[:, 0] = [int(rng.choice([0, 3])) if rng.random() < fail_p else 1 for _ in range(n)]
    return kind, rows.reshape(-1)


def launch(emu, secs, issues):
    """per section (verdicts, applied, failures, left, its rows, its proofs), then (issue verdicts, rows, proofs)"""
    S = len(secs)
    n = [len(s[1]) for s in secs]
    ne = len(issues[0]) if issues else 0
    cap = sum(n) + ne + 1
    keep = []
    arr = lambda a: keep.append(np.ascontiguousarray(a) if len(a) else np.zeros(1, a.dtype)) or keep[-1]
    verdicts = [arr(s[3].copy()) for s in secs]
    applied = [arr(np.zeros(len(s[1]), np.uint8)) for s in secs]
    ptrs = lambda xs: (C.c_void_p * max(S, 1))(*[x.ctypes.data for x in xs])
    cnt = np.zeros(2 * S + 1, np.uint32)
    ekind, erows = issues if issues else (np.zeros(0, np.uint8), np.zeros(0, np.uint8))
    ev = np.zeros(max(ne, 1), np.uint8)
    rr, rp = np.zeros(cap * ROW, np.uint8), np.zeros(cap * 192, np.uint8)
    off = np.zeros(S + 1, np.uint64)
    total = emu.emu_block_launch(S, _p(np.array(n or [0], np.uint64)), _p(np.array([s[0] for s in secs] or [0], np.uint64)),
                                 ptrs([arr(s[1]) for s in secs]), ptrs([arr(s[2]) for s in secs]), ptrs(verdicts), ptrs(applied), _p(cnt),
                                 C.c_size_t(ne), _p(arr(ekind)), _p(arr(erows)), _p(ev), _p(rr), _p(rp), _p(off))
    bounds = [int(o) for o in off] + [total]
    part = lambda i: (rr[ROW * bounds[i]:ROW * bounds[i + 1]].tobytes(), rp[192 * bounds[i]:192 * bounds[i + 1]].tobytes())
    out = [(verdicts[s][:n[s]].tolist(), applied[s][:n[s]].tolist(), int(cnt[2 * s]), int(cnt[2 * s + 1])) + part(s) for s in range(S)]
    return out, (ev[:ne].tolist(),) + part(S)


@pytest.mark.parametrize("seed", range(24))
def test_a_shared_launch_gives_each_section_its_own_launch(emu, seed):
    rng = np.random.default_rng(4000 + seed)
    secs = [chain_section(rng, int(rng.choice([0, 1, 7, 40, 90])), int(rng.integers(1, 9)), float(rng.choice([0, 0.1, 0.5])))
            for _ in range(int(rng.integers(1, 4)))]
    issues = issue_section(rng, int(rng.choice([0, 5, 30])), 0.3) if rng.random() < 0.7 else None
    joint, joint_issues = launch(emu, secs, issues)
    for s, sec in enumerate(secs):
        assert joint[s] == launch(emu, [sec], None)[0][0]
    if issues:
        assert joint_issues == launch(emu, [], issues)[1]


def test_a_failure_in_one_section_never_decides_another(emu):
    rng = np.random.default_rng(4100)
    failing = chain_section(rng, 60, 3, 1.0, undecided_p=1.0)
    passing = chain_section(rng, 50, 3, 0.0, undecided_p=1.0)
    for ip, secs in ((1, [failing, passing]), (0, [passing, failing])):
        out, _ = launch(emu, secs, issue_section(rng, 20, 1.0))
        v, applied, fails, left = out[ip][:4]
        assert v == [1] * 50 and applied == [1] * 50 and (fails, left) == (0, 0)
        v, _, fails, left = out[1 - ip][:4]
        chains = len(set(failing[1].tolist()))
        assert fails == 60 and left == 60 - chains              # each chain's first failure decided, the rest wait
        assert sum(x != UNDECIDED for x in v) == chains
