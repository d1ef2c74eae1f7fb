"""CPU check of the PRODUCT's passes of zk_import_asset_calls (zero_chain_b200/csrc/import.cuh, section 6) compiled with
ZK_HOST_EMUL: asset numbering and slot resolution against the Python driver's _asset_slots, exactly (ids, slot_a, slot_b,
the appended rows and their order), with the product's hash table and with every key forced into one probe chain; the
issue / destroy compaction and verdict scatter against numpy; the state pass's tx_points against each transaction's
points(); and the id-overflow and repeated-row checks.  The real PTX path is covered by tests/test_gpu_asset_calls.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from zero_chain_b200 import groth16 as zk

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FIXED, NEW, BAD, DUP, OVF = range(5)          # the counter block's words
NONE = 0xFFFFFFFF
ROW = 32 * zk.CONFIDENTIAL_POINTS


def _build(tmp_path_factory, name, defines):
    so = str(tmp_path_factory.mktemp(name) / ("lib%s.so" % name))
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", *defines, "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_import_assets.cpp")])
    return C.CDLL(so)


@pytest.fixture(scope="module", params=["product", "one_chain"])
def emu(request, tmp_path_factory):
    defines = [] if request.param == "product" else ["-DZK_IAS_HASH(id,key)=0u", "-DZK_IAS_CAPACITY(n)=((n)+1)"]
    return _build(tmp_path_factory, "emul_import_assets_" + request.param, defines)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _u8(b):
    return np.frombuffer(bytes(b), np.uint8).copy() if len(b) else np.zeros(1, np.uint8)


class Block:
    """random calls over a pool of keys and asset ids; every point a random pattern (the passes copy bytes and compare
    them, they decode nothing)"""

    def __init__(self, rng, n_keys, n_slots, n_tx, ids=(3, 4, 7), issue_frac=0.2, destroy_frac=0.1, fail_frac=0.3, next_id=10,
                 new_flags=zk.ACCOUNT_DUE | 0xF3):
        rnd = lambda m: rng.integers(0, 256, m, dtype=np.uint8).tobytes()
        keys = [rnd(32) for _ in range(n_keys)]
        pool = sorted({(int(rng.choice(ids)), keys[int(rng.integers(0, n_keys))]) for _ in range(n_slots)})
        self.slots = [pool[i] for i in rng.permutation(len(pool))]
        ns = len(self.slots)
        self.balances, self.pendings, self.flags = rnd(64 * ns), rnd(64 * ns), rnd(ns)
        key = lambda: keys[int(rng.integers(0, n_keys))]
        self.txs, self.verdicts = [], []
        for _ in range(n_tx):
            u = rng.random()
            if u < issue_frac:
                self.txs.append(zk.IssueTx(key(), rnd(32), rnd(32), rnd(64), rnd(32), rnd(32), rnd(32), rnd(32)))
            elif u < issue_frac + destroy_frac:
                self.txs.append(zk.DestroyTx(key(), int(rng.choice(ids)), rnd(32), rnd(32), rnd(64), rnd(32), rnd(32), rnd(32), rnd(32)))
            else:
                a = int(rng.choice(ids + (next_id, next_id + 1)))        # also the ids this block's issues create
                self.txs.append(zk.AssetTransferTx(a, key(), key(), rnd(32), rnd(32), rnd(32), rnd(32), rnd(32), rnd(32), rnd(32)))
            self.verdicts.append(0 if self.txs[-1].kind == zk.ASSET_TRANSFER else (1 if rng.random() >= fail_frac else int(rng.choice([0, 2, 4]))))
        self.next_id, self.new_flags = next_id, new_flags

    def rows(self):
        return b"".join(t.verify_points(bytes(64)) if t.kind == zk.ASSET_TRANSFER else t.verify_points() for t in self.txs)


def resolve(emu, b):
    """the emulated passes 1, 3 and 4: (cnt, asset_ids, slot_a, slot_b, (slots, balances, pendings, flags) of the grown table)"""
    n, ns = len(b.txs), len(b.slots)
    nr = ns + 2 * n
    u32 = lambda a: np.array(list(a) or [0], np.uint32)
    aid, sa, sb = u32([7] * n), u32([7] * n), u32([7] * n)
    nid, nk, nb, npd, nf = u32([0] * nr), np.zeros(32 * nr + 1, np.uint8), np.zeros(64 * nr + 1, np.uint8), np.zeros(64 * nr + 1, np.uint8), \
        np.zeros(nr + 1, np.uint8)
    cnt = np.zeros(5, np.uint32)
    emu.emu_as_resolve(C.c_size_t(ns), _p(u32(a for a, _ in b.slots)), _p(_u8(b"".join(k for _, k in b.slots))), _p(_u8(b.balances)),
                       _p(_u8(b.pendings)), _p(_u8(b.flags)), C.c_uint32(b.next_id), C.c_uint8(b.new_flags), C.c_size_t(n),
                       _p(_u8(bytes(t.kind for t in b.txs))), _p(u32(t.asset_id if t.kind != zk.ASSET_ISSUE else 0 for t in b.txs)),
                       _p(_u8(b.rows())), _p(_u8(bytes(b.verdicts))), _p(aid), _p(sa), _p(sb), _p(nid), _p(nk), _p(nb), _p(npd), _p(nf), _p(cnt))
    m = ns + int(cnt[NEW])
    slots = [(int(nid[r]), nk[32 * r:32 * r + 32].tobytes()) for r in range(m)]
    return cnt, aid[:n], sa[:n], sb[:n], (slots, nb[:64 * m].tobytes(), npd[:64 * m].tobytes(), nf[:m].tobytes())


def check(emu, b):
    """the emulation against _asset_slots; returns the number of new rows"""
    slots = list(b.slots)
    (bal, pend, fl), ids, slot_a, slot_b = zk._asset_slots("t", slots, b.balances, b.pendings, b.flags, b.txs, b.verdicts, b.next_id,
                                                           b.new_flags)
    cnt, aid, sa, sb, grown = resolve(emu, b)
    assert (cnt[BAD], cnt[DUP], cnt[OVF]) == (NONE, NONE, NONE)
    assert cnt[FIXED] == sum(t.kind != zk.ASSET_TRANSFER for t in b.txs)
    assert [int(x) for x in aid] == [0 if i is None else i for i in ids]
    assert list(sa) == list(slot_a) and list(sb) == list(slot_b)
    assert grown == (slots, bal, pend, fl)
    return int(cnt[NEW])


@pytest.mark.parametrize("n_keys, n_slots, n_tx, seed", [(8, 12, 60, 1), (30, 100, 400, 2), (3, 0, 50, 3), (5, 9, 0, 4), (0, 0, 0, 5),
                                                       (200, 1000, 2000, 6), (2, 6, 300, 7)])
def test_random_blocks_equal_asset_slots(emu, n_keys, n_slots, n_tx, seed):
    b = Block(np.random.default_rng(seed), max(n_keys, 1), n_slots, n_tx)
    check(emu, b)


def test_issue_whose_new_slot_is_an_existing_row(emu):
    rng = np.random.default_rng(11)
    b = Block(rng, 4, 0, 0)
    issuer = bytes(range(32))
    b.slots = [(3, bytes(32)), (10, issuer), (11, issuer)]
    b.balances, b.pendings, b.flags = bytes(range(192)), bytes(range(1, 193)), bytes([1, 2, 3])
    b.txs = [zk.IssueTx(issuer, *[bytes([k]) * 32 for k in range(2)], bytes(64), *[bytes([9]) * 32] * 4) for _ in range(3)]
    b.verdicts = [1, 1, 1]
    assert check(emu, b) == 1          # ids 10 and 11 are rows 1 and 2; id 12 is new


def test_transfers_of_new_unknown_and_self_assets(emu):
    rng = np.random.default_rng(12)
    b = Block(rng, 4, 0, 0)
    alice, bob = bytes([1]) * 32, bytes([2]) * 32
    pt = lambda: rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
    tr = lambda a, s, r: zk.AssetTransferTx(a, s, r, pt(), pt(), pt(), pt(), pt(), pt(), pt())
    b.slots, b.balances, b.pendings, b.flags = [(3, alice)], bytes(64), bytes(64), bytes(1)
    b.txs = [zk.IssueTx(alice, pt(), pt(), bytes(64), pt(), pt(), pt(), pt()),   # id 10: (10, alice), row 1
             tr(10, alice, bob),                                                 # issued earlier in the block: (10, bob) row 2
             tr(77, bob, alice),                                                 # never issued: rows 3, 4
             tr(3, bob, bob),                                                    # self-transfer: one new row, 5
             zk.DestroyTx(bob, 10, pt(), pt(), bytes(64), pt(), pt(), pt(), pt())]
    b.verdicts = [1, 0, 0, 0, 1]
    assert check(emu, b) == 5
    _, aid, sa, sb, grown = resolve(emu, b)
    assert list(aid) == [10, 0, 0, 0, 0] and list(sa) == [1, 1, 3, 5, 2] and list(sb) == [NONE, 2, 4, 5, NONE]
    assert grown[0] == [(3, alice), (10, alice), (10, bob), (77, bob), (77, alice), (3, bob)]


def test_failing_issues_and_destroys_consume_nothing(emu):
    rng = np.random.default_rng(13)
    b = Block(rng, 6, 10, 200, issue_frac=0.5, destroy_frac=0.5, fail_frac=1.0)
    assert check(emu, b) == 0
    cnt, aid, sa, sb, _ = resolve(emu, b)
    assert not aid.any() and set(sa) == set(sb) == {NONE}
    # half passing: ids run 10, 11, ... over the passing issues only
    b.verdicts = [k % 2 for k in range(len(b.txs))]
    check(emu, b)
    _, aid, _, _, _ = resolve(emu, b)
    passing = [k for k, t in enumerate(b.txs) if t.kind == zk.ASSET_ISSUE and b.verdicts[k] == 1]
    assert [int(aid[k]) for k in passing] == list(range(10, 10 + len(passing)))


@pytest.mark.parametrize("extra", [0, 1])
def test_asset_id_overflow(emu, extra):
    """next_asset_id = 2^32 - m with m passing issues is accepted; one more passing issue is refused, naming it"""
    b = Block(np.random.default_rng(14), 5, 4, 80, issue_frac=0.5, fail_frac=0.3)
    passing = [k for k, t in enumerate(b.txs) if t.kind == zk.ASSET_ISSUE and b.verdicts[k] == 1]
    m = len(passing) - extra
    b.next_id = 2**32 - m
    if not extra:
        check(emu, b)
        assert resolve(emu, b)[1][passing[-1]] == 2**32 - 1
        return
    with pytest.raises(ValueError):
        zk._asset_slots("t", list(b.slots), b.balances, b.pendings, b.flags, b.txs, b.verdicts, b.next_id, b.new_flags)
    assert resolve(emu, b)[0][OVF] == passing[-1]


def test_repeated_table_key_names_the_lowest_repeating_row(emu):
    b = Block(np.random.default_rng(15), 400, 80, 30)
    s = b.slots
    assert len(s) > 60
    assert resolve(emu, b)[0][DUP] == NONE
    s[37], s[52], s[20] = s[5], s[5], s[44]          # rows 5, 37, 52 share a key; 20 and 44 share another
    assert resolve(emu, b)[0][DUP] == 37
    s[50] = s[49]
    assert resolve(emu, b)[0][DUP] == 37
    s[8] = s[2]
    assert resolve(emu, b)[0][DUP] == 8
    b.slots[8] = (s[2][0] + 1, s[2][1])              # same key, another id: distinct
    assert resolve(emu, b)[0][DUP] == 37


@pytest.mark.parametrize("n_tx, seed", [(0, 1), (1, 2), (90, 3), (400, 4)])
def test_compaction_scatter_and_tx_points(emu, n_tx, seed):
    rng = np.random.default_rng(20 + seed)
    b = Block(rng, 10, 10, n_tx, issue_frac=0.3, destroy_frac=0.2)
    n = len(b.txs)
    kind = _u8(bytes(t.kind for t in b.txs))
    rows, proofs = b.rows(), rng.integers(0, 256, 192 * n, dtype=np.uint8).tobytes()
    fixed = [k for k, t in enumerate(b.txs) if t.kind != zk.ASSET_TRANSFER]
    pos, cnt = np.zeros(n + 1, np.uint32), np.zeros(5, np.uint32)
    rr, rp = np.zeros(ROW * n + 1, np.uint8), np.zeros(192 * n + 1, np.uint8)
    rv = _u8(rng.integers(0, 5, n, dtype=np.uint8).tobytes())
    verdicts = np.full(n + 1, 0xAB, np.uint8)
    emu.emu_as_compact(C.c_size_t(n), _p(kind), _p(_u8(rows)), _p(_u8(proofs)), _p(pos), _p(cnt), _p(rr), _p(rp), _p(rv), _p(verdicts))
    assert cnt[FIXED] == len(fixed) and cnt[BAD] == NONE
    m = len(fixed)
    assert rr[:ROW * m].tobytes() == b"".join(b.txs[k].verify_points() for k in fixed)
    assert rp[:192 * m].tobytes() == b"".join(proofs[192 * k:192 * k + 192] for k in fixed)
    want = np.zeros(n, np.uint8)
    want[fixed] = rv[:m]
    assert (verdicts[:n] == want).all()
    tp = np.zeros(128 * n + 1, np.uint8)
    emu.emu_as_tx_points(C.c_size_t(n), _p(kind), _p(_u8(rows)), _p(tp))
    assert tp[:128 * n].tobytes() == b"".join(t.points() for t in b.txs)


def test_unknown_kind_is_counted(emu):
    kind = _u8(bytes([0, 1, 2, 3, 0, 9]))
    pos, cnt = np.zeros(7, np.uint32), np.zeros(5, np.uint32)
    z = np.zeros(ROW * 6 + 192 * 6, np.uint8)
    emu.emu_as_compact(C.c_size_t(6), _p(kind), _p(z), _p(z), _p(pos), _p(cnt), _p(z.copy()), _p(z.copy()), _p(z), _p(z.copy()))
    assert cnt[BAD] == 3 and cnt[FIXED] == 2
