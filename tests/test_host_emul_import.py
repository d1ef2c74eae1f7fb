"""CPU check of the PRODUCT's round decisions of zk_import_confidential_block / zk_import_assets_block
(zero_chain_b200/csrc/import.cuh) compiled with ZK_HOST_EMUL, against the Python drivers import_confidential_block and
import_assets_block, round by round.

Both sides get the same model verifier: each transfer has an intended verdict, the one its proof gets against the balance
it was made for (the chain's earlier intended passes applied); against any other balance it fails.  The drivers run
unchanged with their state call and their verifier replaced by the model, which records the transactions each round
verifies.  The real PTX path is covered by tests/test_gpu_import.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from zero_chain_b200 import groth16 as zk

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MAX_ROUNDS = 64


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_import") / "libemul_import.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "zero_chain_b200", "csrc"),
                           "-o", so, os.path.join(HERE, "host_emul", "emul_import.cpp")])
    lib = C.CDLL(so)
    lib.emu_import.restype = C.c_longlong
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def run_header(emu, n_keys, kind, key_a, key_b, fixed, intended):
    """(bad, verdicts, rounds, [the set verified in each round]) from the header's passes"""
    n = len(key_a)
    arr = lambda v, t: np.array(list(v) or [0], t)
    verdicts, rounds = np.zeros(max(n, 1), np.uint8), np.zeros(1, np.uint32)
    und = np.zeros(max(MAX_ROUNDS * n, 1), np.uint8)
    bad = emu.emu_import(C.c_size_t(n_keys), C.c_size_t(n), _p(arr(kind, np.uint8)) if kind is not None else None, _p(arr(key_a, np.uint32)),
                         _p(arr(key_b, np.uint32)), _p(arr(fixed, np.uint8)), _p(arr(intended, np.uint8)), _p(verdicts), _p(rounds), _p(und),
                         C.c_size_t(MAX_ROUNDS))
    r = int(rounds[0])
    sets = [set(np.flatnonzero(und[i * n:(i + 1) * n]).tolist()) for i in range(r)]
    return int(bad), [int(v) for v in verdicts[:n]], r, sets


class _Model:
    """The model verifier and state call the drivers run on: a transfer's balance_sender carries, in its first byte,
    whether every earlier applied transfer of its chain passes (the balance its proof was made for)."""

    def __init__(self, key_a, is_transfer, intended):
        self.key_a, self.is_transfer, self.intended = list(key_a), list(is_transfer), list(intended)
        self.rounds = []

    def balance_sender(self, mask) -> bytes:
        out = bytearray(64 * len(self.key_a))
        for k in range(len(self.key_a)):
            out[64 * k] = all(not (self.is_transfer[q] and self.key_a[q] == self.key_a[k] and mask[q] == 1 and self.intended[q] != 1)
                              for q in range(k))
        return bytes(out)

    def verify(self, pvk, proofs, points, n_points):
        assert n_points == zk.CONFIDENTIAL_POINTS
        ks = [int.from_bytes(proofs[192 * i:192 * i + 4], "little") for i in range(len(proofs) // 192)]
        got = []
        for i, k in enumerate(ks):
            exact = points[352 * i + 192]
            got.append(self.intended[k] if self.intended[k] != 1 or not self.is_transfer[k] else int(bool(exact)))
        if all(self.is_transfer[k] for k in ks):
            self.rounds.append(set(ks))
        return got


def _proofs(n):
    return b"".join(k.to_bytes(4, "little") + bytes(188) for k in range(n))


def _pt(i):
    return (i + 1).to_bytes(32, "little")


def run_confidential_driver(monkeypatch, n_acct, sender, recipient, intended):
    n = len(sender)
    model = _Model(sender, [True] * n, intended)

    def state(ctx, balances, pendings, flags, s, r, tx_points, applied):
        return (model.balance_sender(applied), bytes(64 * n), bytes(n), balances, pendings, flags)
    monkeypatch.setattr(zk, "confidential_block", state)
    monkeypatch.setattr(zk, "verify_proofs_with_points", model.verify)
    txs = [zk.ConfidentialTx(int(s), int(r), *[_pt(i) for i in range(9)]) for s, r in zip(sender, recipient)]
    accounts = (bytes(64 * n_acct), bytes(64 * n_acct), bytes(n_acct))
    verdicts, _, _, rounds = zk.import_confidential_block(None, None, accounts, txs, _proofs(n))
    return verdicts, rounds, model.rounds


def chains(rng, n_keys, n, fail_p, codes=(0, 2, 3, 4)):
    sender = rng.integers(0, n_keys, n).astype(np.uint32)
    recipient = rng.integers(0, n_keys, n).astype(np.uint32)
    intended = [int(rng.choice(codes)) if rng.random() < fail_p else 1 for _ in range(n)]
    return sender, recipient, intended


def check_confidential(emu, monkeypatch, n_keys, sender, recipient, intended):
    want_v, want_r, want_sets = run_confidential_driver(monkeypatch, n_keys, sender, recipient, intended)
    bad, got_v, got_r, got_sets = run_header(emu, n_keys, None, sender, recipient, [0] * len(sender), intended)
    assert bad == -1
    assert got_v == want_v == intended                     # the model makes every intended verdict the final one
    assert got_r == want_r and got_sets == want_sets
    return got_r


@pytest.mark.parametrize("seed", range(12))
def test_random_chains_equal_the_driver(emu, monkeypatch, seed):
    rng = np.random.default_rng(900 + seed)
    n_keys = int(rng.integers(1, 12))
    sender, recipient, intended = chains(rng, n_keys, int(rng.integers(1, 80)), float(rng.choice([0.0, 0.05, 0.2, 0.5])))
    check_confidential(emu, monkeypatch, n_keys, sender, recipient, intended)


def test_several_failures_in_one_chain(emu, monkeypatch):
    sender = np.zeros(10, np.uint32)
    intended = [1, 0, 1, 1, 2, 1, 0, 1, 1, 1]
    assert check_confidential(emu, monkeypatch, 1, sender, sender, intended) == 4


def test_failure_at_the_first_and_the_last_transfer(emu, monkeypatch):
    sender = np.zeros(6, np.uint32)
    assert check_confidential(emu, monkeypatch, 2, sender, sender + 1, [0, 1, 1, 1, 1, 1]) == 2
    assert check_confidential(emu, monkeypatch, 2, sender, sender + 1, [1, 1, 1, 1, 1, 4]) == 1     # the failure ends the chain
    assert check_confidential(emu, monkeypatch, 2, sender, sender + 1, [3, 1, 1, 1, 1, 0]) == 2


def test_every_transfer_fails(emu, monkeypatch):
    rng = np.random.default_rng(950)
    sender, recipient, _ = chains(rng, 5, 40, 0.0)
    rounds = check_confidential(emu, monkeypatch, 5, sender, recipient, [0] * 40)
    assert rounds == np.bincount(sender).max()              # one failure decided per chain and round, the last ends its chain


def test_chains_interleaved_across_senders(emu, monkeypatch):
    sender = np.array([0, 1, 2, 0, 1, 2, 0, 1, 2, 0, 1, 2], np.uint32)
    intended = [1, 0, 1, 0, 1, 1, 1, 0, 1, 1, 1, 1]
    assert check_confidential(emu, monkeypatch, 3, sender, (sender + 1) % 3, intended) == 3


def test_no_failures_take_one_round_and_an_empty_block_none(emu, monkeypatch):
    rng = np.random.default_rng(951)
    sender, recipient, intended = chains(rng, 7, 50, 0.0)
    assert check_confidential(emu, monkeypatch, 7, sender, recipient, intended) == 1
    assert run_header(emu, 3, None, [], [], [], [])[1:] == ([], 0, [])


def test_index_out_of_range_names_the_lowest_transaction(emu):
    sender = np.array([0, 1, 4, 0, 9], np.uint32)
    recipient = np.array([1, 1, 0, 7, 0], np.uint32)
    assert run_header(emu, 4, None, sender, recipient, [0] * 5, [1] * 5)[0] == 2
    kind = [1, 2, 0, 2, 3]                                   # a failing destroy's slot is ignored; kind 3 is unknown
    assert run_header(emu, 4, kind, [9, 9, 0, 1, 0], [9, 9, 1, 9, 9], [0, 0, 0, 1, 1], [1] * 5)[0] == 4
    assert run_header(emu, 4, kind[:4], [9, 9, 0, 1], [9, 9, 1, 9], [0, 1, 0, 1], [1] * 4)[0] == 1


def test_tx_points_come_from_slots_2_3_5_4(emu):
    rows = np.random.default_rng(952).integers(0, 256, 3 * 352).astype(np.uint8)
    out = np.zeros(3 * 128, np.uint8)
    emu.emu_tx_points(C.c_size_t(3), _p(rows), _p(out))
    r = rows.reshape(3, 11, 32)
    assert np.array_equal(out.reshape(3, 4, 32), r[:, [2, 3, 5, 4], :])


# ---- encrypted assets ---------------------------------------------------------------------------------------------------
def assets_block(rng, n_keys, n, fail_p, issue_frac=0.15, destroy_frac=0.1):
    """asset 0 held by n_keys keys; transfers between them, issues of new assets, destroys of (0, owner)"""
    keys = [_pt(100 + i) for i in range(n_keys)]
    txs, intended = [], []
    for _ in range(n):
        u = rng.random()
        fail = rng.random() < fail_p
        if u < issue_frac:
            txs.append(zk.IssueTx(keys[int(rng.integers(0, n_keys))], *[_pt(1)] * 2, bytes(64), *[_pt(2)] * 4))
        elif u < issue_frac + destroy_frac:
            txs.append(zk.DestroyTx(keys[int(rng.integers(0, n_keys))], 0, *[_pt(3)] * 2, bytes(64), *[_pt(4)] * 4))
        else:
            a, b = (keys[int(i)] for i in rng.integers(0, n_keys, 2))
            txs.append(zk.AssetTransferTx(0, a, b, *[_pt(5)] * 4, *[_pt(6)] * 3))
        # a failing issue's or destroy's verdict is the caller's byte: any value but 1, the undecided marker 0xFF included
        codes = [0, 2, 4] if txs[-1].kind == zk.ASSET_TRANSFER else [0, 2, 4, 0xFF, 0x80]
        intended.append(int(rng.choice(codes)) if fail else 1)
    return keys, txs, intended


def check_assets(emu, monkeypatch, keys, txs, intended):
    n = len(txs)
    kinds = np.array([t.kind for t in txs], np.uint8)
    fixed = [intended[k] if kinds[k] != zk.ASSET_TRANSFER else 0 for k in range(n)]
    state = ([(0, k) for k in keys], bytes(64 * len(keys)), bytes(64 * len(keys)), bytes(len(keys)))
    (_, _, fl), _, slot_a, slot_b = zk._asset_slots("t", list(state[0]), *state[1:], txs, fixed, 7, 0)
    model = _Model(slot_a, kinds == zk.ASSET_TRANSFER, intended)

    def state_call(ctx, bal, pend, flags, kind, sa, sb, tx_points, applied):
        assert np.array_equal(sa, slot_a) and np.array_equal(sb, slot_b)
        return (model.balance_sender(applied), bytes(64 * n), bytes(128 * n), bytes(n), bytes(n), bal, pend, flags)
    monkeypatch.setattr(zk, "assets_block", state_call)
    monkeypatch.setattr(zk, "verify_proofs_with_points", model.verify)
    want_v, _, _, _, want_r = zk.import_assets_block(None, None, state, txs, _proofs(n), 7, 0)
    bad, got_v, got_r, got_sets = run_header(emu, len(fl), kinds, slot_a, slot_b, fixed, intended)
    assert bad == -1
    assert got_v == want_v == intended
    assert got_r == want_r and got_sets == model.rounds
    return got_r


@pytest.mark.parametrize("seed", range(8))
def test_random_asset_blocks_equal_the_driver(emu, monkeypatch, seed):
    rng = np.random.default_rng(960 + seed)
    n_keys = int(rng.integers(1, 8))
    keys, txs, intended = assets_block(rng, n_keys, int(rng.integers(1, 60)), float(rng.choice([0.0, 0.1, 0.3])))
    check_assets(emu, monkeypatch, keys, txs, intended)


def test_asset_block_whose_issues_and_destroys_all_fail(emu, monkeypatch):
    rng = np.random.default_rng(970)
    keys, txs, intended = assets_block(rng, 3, 40, 0.0, issue_frac=0.3, destroy_frac=0.3)
    intended = [0 if t.kind != zk.ASSET_TRANSFER else v for t, v in zip(txs, intended)]
    assert check_assets(emu, monkeypatch, keys, txs, intended) == 1


def test_a_fixed_verdict_equal_to_the_undecided_marker_is_not_a_transfer(emu):
    """an issue whose caller-supplied verdict byte is 0xFF (a failure, with the slot of a failure: past the table) is never
    compacted into a round, nor are its slots read"""
    none = 0xFFFFFFFF
    bad, verdicts, rounds, sets = run_header(emu, 2, [1, 0], [none, 0], [none, 1], [0xFF, 0], [0, 1])
    assert (bad, verdicts, rounds, sets) == (-1, [0xFF, 1], 1, [{1}])
    # the same between the failures of a chain: issue and destroy bytes 0xFF, 0x80 and 0 all fail and are passed through
    kind = [0, 1, 0, 2, 0, 1, 0]
    key_a = [0, none, 0, none, 0, 1, 0]
    key_b = [1, none, 1, none, 1, none, 1]
    fixed = [0, 0xFF, 0, 0x80, 0, 1, 0]
    intended = [1, 0, 0, 0, 1, 0, 1]
    bad, verdicts, rounds, sets = run_header(emu, 2, kind, key_a, key_b, fixed, intended)
    assert (bad, verdicts, rounds) == (-1, [1, 0xFF, 0, 0x80, 1, 1, 1], 2)
    assert sets == [{0, 2, 4, 6}, {4, 6}]
