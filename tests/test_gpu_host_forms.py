"""GPU tests of the host forms' in-and-out arrays: zk_balances_confidential_block's balance_after, zk_assets_block's
balance_after / event_ct / event_flags and zk_anonymous_calls_block's issued are written only for the applied
transactions, and the header promises the caller's bytes everywhere else.  Each call runs through ctypes with those
arrays preset, twice with different presets so that a stale device copy cannot pass for the caller's bytes, and its
outputs are compared with the _device form's on the same presets."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.jubjub_oracle import anon_issue_corpus
from tests.jubjub_oracle import assets_corpus
from tests.jubjub_oracle import bal_corpus
from zero_chain_b200 import _lib
from zero_chain_b200 import groth16 as zk

pytestmark = pytest.mark.gpu
PRESETS = (0x5C, 0xAB)


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def _u8(b):
    return np.frombuffer(bytes(b), np.uint8).copy()


def _u32(v):
    return np.ascontiguousarray(np.asarray(v, np.int64).reshape(-1).astype(np.uint32))


def _host(ctx, name, args):
    """the host form on copies of args (ints: sizes, arrays: the arrays); returns the arrays after the call"""
    arrs = [a.copy() if isinstance(a, np.ndarray) else a for a in args]
    zk._ck(getattr(_lib.lib(), name)(ctx._h, *[zk._p(a) if isinstance(a, np.ndarray) else a for a in arrs]))
    return [a for a in arrs if isinstance(a, np.ndarray)]


def _device(ctx, name, args):
    """the _device form on device copies of args; returns the arrays after the call"""
    ts = [torch.from_numpy(a.view(np.uint8).copy()).cuda() if isinstance(a, np.ndarray) else a for a in args]
    torch.cuda.synchronize()
    zk._ck(getattr(_lib.lib(), name + "_device")(ctx._h, *[C.c_void_p(t.data_ptr()) if isinstance(t, torch.Tensor) else t for t in ts]))
    ctx.sync()
    return [t.cpu().numpy() for t in ts if isinstance(t, torch.Tensor)]


def _check(ctx, name, make_args, preset_at, written):
    """make_args(preset) -> args; preset_at: the indices (among the arrays) of the in-and-out arrays, with their row sizes;
    written(host arrays) -> per in-and-out array, a mask of the rows the call writes"""
    for preset in PRESETS:
        args = make_args(preset)
        host, dev = _host(ctx, name, args), _device(ctx, name, args)
        assert len(host) == len(dev)
        for h, d in zip(host, dev):
            assert h.view(np.uint8).tobytes() == d.view(np.uint8).tobytes()
        masks = written(host)
        for (i, row), wrote in zip(preset_at, masks):
            rows = host[i].view(np.uint8).reshape(-1, row)
            assert 0 < wrote.sum() < len(wrote)
            assert (rows[~wrote] == preset).all()
            assert not (rows[wrote] == preset).all(axis=1).any()


def test_confidential_block_keeps_balance_after(ctx):
    b = bal_corpus.make(120, 1500, 31, skew=1.2, bad_points=20, bad_index=True, self_frac=0.05)
    n_acct, n_tx = len(b.flags), b.n_tx

    def args(preset):
        z = lambda n, v=0: np.full(n, v, np.uint8)
        return [n_acct, _u8(b.balances), _u8(b.pendings), _u8(b.flags), n_tx, _u32(b.sender), _u32(b.recipient), _u8(b.tx_points),
                _u8(b.applied), z(64 * n_tx), z(64 * n_tx, preset), z(n_tx), z(64 * n_acct), z(64 * n_acct), z(n_acct)]

    # arrays: balances, pendings, flags, sender, recipient, tx_points, applied, balance_sender, balance_after (8), status (9)
    _check(ctx, "zk_balances_confidential_block", args, [(8, 64)], lambda h: [h[9] == 0])


def test_assets_block_keeps_balance_after_and_events(ctx):
    b = assets_corpus.make(120, 1500, 32, skew=1.2, issue_frac=0.1, destroy_frac=0.05, bad_points=20, bad_index=True)
    n, n_tx = len(b.flags), b.n_tx
    kind = _u8(b.kind)

    def args(preset):
        z = lambda m, v=0: np.full(m, v, np.uint8)
        return [n, _u8(b.balances), _u8(b.pendings), _u8(b.flags), n_tx, kind, _u32(b.slot_a), _u32(b.slot_b), _u8(b.tx_points),
                _u8(b.applied), z(64 * n_tx), z(64 * n_tx, preset), z(128 * n_tx, preset), z(n_tx, preset), z(n_tx), z(64 * n), z(64 * n),
                z(n)]

    # arrays: ..., applied (7), balance_sender (8), balance_after (9), event_ct (10), event_flags (11), status (12)
    def written(h):
        ok = h[12] == 0
        return [ok & (kind == 0), ok & (kind != 0), ok & (kind != 0)]

    _check(ctx, "zk_assets_block", args, [(9, 64), (10, 128), (11, 1)], written)


def test_anonymous_calls_block_keeps_issued(ctx):
    b = anon_issue_corpus.make(120, 1200, 33, issue_frac=0.15, free=10, skew=1.2, bad_points=20, bad_index=True, bad_issue_points=8)
    n_acct = len(b.flags)
    kind = _u8(b.kind)
    n_tx = len(kind)

    def args(preset):
        z = lambda m, v=0: np.full(m, v, np.uint8)
        return [n_acct, _u8(b.keys), _u8(b.balances), _u8(b.pendings), _u8(b.flags), n_tx, kind, _u32(b.members), _u8(b.tx_points),
                _u8(b.tx_extra), _u8(b.g_epoch), _u8(b.applied), z(768 * n_tx), z(1664 * n_tx), z(64 * n_tx, preset), z(n_tx),
                z(64 * n_acct), z(64 * n_acct), z(n_acct)]

    # arrays: keys, ..., applied (9), enc_balances (10), verify_points (11), issued (12), status (13)
    _check(ctx, "zk_anonymous_calls_block", args, [(12, 64)], lambda h: [(kind == 1) & (h[13] == 0)])
