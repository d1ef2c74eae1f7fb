"""CPU check of the PRODUCT's passes of zk_import_anonymous_block (zero_chain_b200/csrc/import.cuh, section 5) compiled
with ZK_HOST_EMUL: the start pass against the index checks of the Python driver import_anonymous_calls_block, the issue
rows against AnonIssueTx.verify_points byte for byte, and the compaction, scatter and gather against a numpy
restatement.  Random kinds, rings and fields, including empty, all-issue and all-transfer blocks.  The real PTX path is
covered by tests/test_gpu_import_anon.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from zero_chain_b200 import groth16 as zk

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RING = zk.ANONIMITY_SIZE
ISSUES, BAD, TRANSFERS = 0, 2, 3          # the counter block's words
NONE = 0xFFFFFFFF


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_import_anon") / "libemul_import_anon.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_import_anon.cpp")])
    return C.CDLL(so)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _u8(b):
    return np.frombuffer(bytes(b), np.uint8).copy() if len(b) else np.zeros(1, np.uint8)


class Block:
    """random transactions over n_acct accounts; every byte a random pattern (the passes copy bytes, they decode nothing)"""

    def __init__(self, rng, n_acct, n_tx, issue_frac):
        rnd = lambda m: rng.integers(0, 256, m, dtype=np.uint8).tobytes()
        self.n_acct = n_acct
        self.keys, self.g_epoch = rnd(32 * n_acct), rnd(32)
        self.txs = []
        for _ in range(n_tx):
            if rng.random() < issue_frac:
                self.txs.append(zk.AnonIssueTx(int(rng.integers(0, n_acct)), rnd(32), rnd(32), rnd(64), rnd(32), rnd(32), rnd(32)))
            else:
                self.txs.append(zk.AnonymousTx(rng.integers(0, n_acct, RING), [rnd(32) for _ in range(RING)], rnd(32), rnd(32), rnd(32)))
        self.proofs = rnd(192 * n_tx)

    @property
    def n(self):
        return len(self.txs)

    def arrays(self):
        """kind, members (an issue's ignored members 1..11 hold garbage), tx_points, tx_extra, issue_fields, as the call takes them"""
        kind = np.array([t.kind for t in self.txs] or [0], np.uint8)
        mem = np.array([t.members for t in self.txs] or [[0] * RING], np.uint32)
        for k, t in enumerate(self.txs):
            if t.kind == zk.ANON_ISSUE:
                mem[k, 1:] = (np.arange(1, RING) * 977 + k) % (2 * self.n_acct + 3)
        fields = b"".join(t.fee + t.balance if t.kind == zk.ANON_ISSUE else bytes(96) for t in self.txs)
        return (kind, mem.reshape(-1), _u8(b"".join(t.points() for t in self.txs)), _u8(b"".join(t.rvk + t.nonce for t in self.txs)),
                _u8(fields))


def start(emu, n_acct, kind, members, n, issues_ok=True):
    flag, cnt = np.zeros(max(n, 1), np.uint32), np.zeros(4, np.uint32)
    emu.emu_an_start(C.c_size_t(n), C.c_uint32(n_acct), C.c_int(int(issues_ok)), _p(kind) if kind is not None else None, _p(members),
                     _p(flag), _p(cnt))
    return flag[:n], cnt


def exclusive_sum(flag):
    return (np.cumsum(flag) - flag).astype(np.uint32) if len(flag) else np.zeros(1, np.uint32)


CASES = [(40, 300, 0.1), (5, 64, 0.5), (12, 50, 1.0), (12, 50, 0.0), (7, 1, 1.0), (7, 1, 0.0), (3, 0, 0.3), (200, 1000, 0.05)]


@pytest.mark.parametrize("n_acct, n_tx, frac", CASES)
def test_issue_rows_equal_verify_points(emu, n_acct, n_tx, frac):
    rng = np.random.default_rng(n_acct * 1000 + n_tx)
    b = Block(rng, n_acct, n_tx, frac)
    kind, mem, tp, tx, fields = b.arrays()
    flag, cnt = start(emu, n_acct, kind, mem, b.n)
    is_issue = np.array([t.kind == zk.ANON_ISSUE for t in b.txs], bool)
    assert cnt[BAD] == NONE and cnt[ISSUES] == is_issue.sum() and cnt[TRANSFERS] == b.n - is_issue.sum()
    assert np.array_equal(flag, is_issue.astype(np.uint32))
    pos = exclusive_sum(flag)
    n_iss = int(is_issue.sum())
    rows, proofs = np.full(max(352 * b.n, 1), 0xAB, np.uint8), np.full(max(192 * b.n, 1), 0xAB, np.uint8)
    emu.emu_an_issue_rows(C.c_size_t(b.n), _p(kind), _p(pos), _p(_u8(b.keys)), _p(mem), _p(tp), _p(fields), _p(tx), _p(_u8(b.g_epoch)),
                          _p(_u8(b.proofs)), _p(rows), _p(proofs))
    iss = np.flatnonzero(is_issue).tolist()
    want = b"".join(b.txs[k].verify_points(b.keys, b.g_epoch) for k in iss)
    assert rows[:352 * n_iss].tobytes() == want
    assert proofs[:192 * n_iss].tobytes() == b"".join(b.proofs[192 * k:192 * k + 192] for k in iss)
    assert not (rows[352 * n_iss:] != 0xAB).any() and not (proofs[192 * n_iss:] != 0xAB).any()     # nothing past the issues


@pytest.mark.parametrize("n_acct, n_tx, frac", CASES)
def test_scatter_and_gather_equal_numpy(emu, n_acct, n_tx, frac):
    rng = np.random.default_rng(7 + n_acct * 1000 + n_tx)
    b = Block(rng, n_acct, n_tx, frac)
    kind, mem, _, _, _ = b.arrays()
    flag, _ = start(emu, n_acct, kind, mem, b.n)
    pos = exclusive_sum(flag)
    n = b.n
    is_issue = flag.astype(bool)
    iss, tr = np.flatnonzero(is_issue), np.flatnonzero(~is_issue)
    # the issue verdicts, then the transfers' rows out of the state pass's verify_points, then their verdicts
    rv1 = np.zeros(max(n, 1), np.uint8)
    rv1[:len(iss)] = rng.choice([0, 1, 2, 3, 4], len(iss))
    verdicts = np.full(max(n, 1), 0xAB, np.uint8)
    emu.emu_an_scatter(C.c_size_t(n), 1, _p(kind), _p(pos), _p(rv1), _p(verdicts))
    want = np.zeros(n, np.uint8)
    want[iss] = rv1[:len(iss)]
    assert np.array_equal(verdicts[:n], want)
    vp = rng.integers(0, 256, max(1664 * n, 1), dtype=np.uint8)
    rows, proofs = np.full(max(1664 * n, 1), 0xAB, np.uint8), np.full(max(192 * n, 1), 0xAB, np.uint8)
    emu.emu_an_gather(C.c_size_t(n), _p(kind), _p(pos), _p(vp), _p(_u8(b.proofs)), _p(rows), _p(proofs))
    assert np.array_equal(rows[:1664 * len(tr)].reshape(-1, 1664), vp[:1664 * n].reshape(n, 1664)[tr])
    assert np.array_equal(proofs[:192 * len(tr)].reshape(-1, 192), np.frombuffer(b.proofs, np.uint8).reshape(n, 192)[tr])
    assert not (rows[1664 * len(tr):] != 0xAB).any()
    rv2 = np.zeros(max(n, 1), np.uint8)
    rv2[:len(tr)] = rng.choice([0, 1, 2, 4], len(tr))
    emu.emu_an_scatter(C.c_size_t(n), 0, _p(kind), _p(pos), _p(rv2), _p(verdicts))
    want[tr] = rv2[:len(tr)]
    assert np.array_equal(verdicts[:n], want)


def driver_bad(b: Block, kind):
    """the lowest transaction the driver's check (every member of t.members in range; an issue's members are its issuer) or
    the call's other rules (an unknown kind) reject, or -1"""
    for k, t in enumerate(b.txs):
        if kind[k] > zk.ANON_ISSUE or not all(0 <= m < b.n_acct for m in t.members):
            return k
    return -1


@pytest.mark.parametrize("seed", range(10))
def test_start_names_the_lowest_bad_transaction(emu, seed):
    rng = np.random.default_rng(300 + seed)
    n_acct = int(rng.integers(1, 30))
    b = Block(rng, n_acct, int(rng.integers(1, 200)), float(rng.choice([0.0, 0.1, 0.5, 1.0])))
    kind, mem, _, _, _ = b.arrays()
    for k in rng.choice(b.n, min(b.n, 3), replace=False).tolist():
        what = int(rng.integers(0, 3))
        if what == 0 and b.txs[k].kind == zk.ANON_TRANSFER:
            j = int(rng.integers(0, RING))
            b.txs[k].members[j] = n_acct + int(rng.integers(0, 5))
            mem[RING * k + j] = b.txs[k].members[j]
        elif what == 1 and b.txs[k].kind == zk.ANON_ISSUE:
            b.txs[k].issuer = n_acct + int(rng.integers(0, 5))
            mem[RING * k] = b.txs[k].issuer
        elif what == 2:
            kind[k] = int(rng.choice([2, 3, 255]))
    _, cnt = start(emu, n_acct, kind, mem, b.n)
    want = driver_bad(b, kind)
    assert (int(cnt[BAD]) if cnt[BAD] != NONE else -1) == want
    # without a confidential key (or issue_fields) the first issue is bad too
    first_issue = next((k for k in range(b.n) if kind[k] == zk.ANON_ISSUE), -1)
    _, cnt = start(emu, n_acct, kind, mem, b.n, issues_ok=False)
    cands = [x for x in (want, first_issue) if x >= 0]
    assert (int(cnt[BAD]) if cnt[BAD] != NONE else -1) == (min(cands) if cands else -1)


def test_start_rules_on_a_hand_made_block(emu):
    """an issue's members 1..11 are ignored; a NULL kind makes every transaction a transfer"""
    kind = np.array([1, 0, 1, 0], np.uint8)
    mem = np.zeros((4, RING), np.uint32)
    mem[0, 1:] = NONE                       # ignored
    mem[2, 0] = 4                           # issuer out of range
    mem[3, 11] = 4                          # transfer member out of range
    _, cnt = start(emu, 4, kind, mem.reshape(-1), 4)
    assert list(cnt) == [2, 0, 2, 2]
    mem[2, 0] = 3
    flag, cnt = start(emu, 4, kind, mem.reshape(-1), 4)
    assert cnt[BAD] == 3 and list(flag) == [1, 0, 1, 0]
    flag, cnt = start(emu, 4, None, mem.reshape(-1), 4)
    assert cnt[BAD] == 0 and cnt[ISSUES] == 0 and cnt[TRANSFERS] == 4 and not flag.any()   # transaction 0's members 1..11 count now
    _, cnt = start(emu, 4, np.zeros(1, np.uint8), mem.reshape(-1), 0)
    assert list(cnt) == [0, 0, NONE, 0]
