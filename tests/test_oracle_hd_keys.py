"""CPU checks of the two key-derivation oracles (tests/jubjub_oracle/hd_keys.py and the C oracle hd_keys_oracle.c): they
agree byte for byte on edge rows, random rows and every status; both satisfy the reference's own tests
(zface/src/derive/mod.rs:267-319: derive_nonhardened_child, derive_hardened_child, read_write) as properties over many
seeds; and what the reference pins is pinned here: hashlib for every hash, and the Alice literal for
SpendingKey::from_seed.  The reference has no literal for any derived key."""
import hashlib
import json
import os
import struct

import numpy as np
import pytest

from tests.jubjub_oracle import hd_coracle as hc
from tests.jubjub_oracle import hd_keys as hd
from tests.jubjub_oracle import pyref as jj
from tests.jubjub_oracle import redjubjub as rj

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tx_build.json")


def test_master_agrees_and_is_pinned():
    seeds = [b"", b"x", bytes(64)] + [np.random.default_rng(1).bytes(k) for k in (16, 32, 64, 129)]
    assert hc.master(seeds) == [hd.master_row(s) for s in seeds]
    for s in seeds:
        i = hashlib.blake2b(s, digest_size=64, person=b"Zerochain_Master").digest()
        x = hd.master(s)
        assert x[:9] == bytes(9) and x[9:41] == i[32:]
        assert x[41:] == rj.scalar_bytes(rj.spending_key(i[:32]))
    # SpendingKey::from_seed, which the master key applies to I_L, is pinned by the reference's Alice literal
    g = json.load(open(GOLDEN))
    assert rj.encryption_key(g["alice_seed"].encode()).hex() == g["alice_encryption_key"]["value"]


def test_tag_is_hashlibs():
    for pgk in (bytes(32), jj.encode(rj.P_G), hd.IDENTITY_SIGNED):
        assert hc.tag(pgk) == hashlib.blake2b(pgk, digest_size=32, person=b"ZerochainEFinger").digest()[:4]


def test_edge_rows_agree():
    parents = hd.edge_xsk_parents()
    pidx, cidx = hd.edge_rows(len(parents))
    want = hd.xsk_derive_rows(parents, pidx, cidx)
    assert hc.xsk_derive(parents, pidx, cidx) == want
    assert {w[4] for w in want} == {0, hd.BAD_INDEX, hd.DEPTH}
    assert [r[0] for r in hc.xsk_derive(parents, pidx, cidx, outputs=False)] == [w[0] for w in want]
    xp = hd.edge_xpgk_parents()
    pidx, cidx = hd.edge_rows(len(xp))
    want = hd.xpgk_derive_rows(xp, pidx, cidx)
    assert hc.xpgk_derive(xp, pidx, cidx) == want
    assert {w[3] for w in want} == {0, 1, 2, 3, hd.BAD_INDEX, hd.HARDENED_INDEX, hd.DEPTH}


def test_random_rows_agree():
    parents = hd.random_xsk_parents(16, seed=2)
    pidx, cidx = hd.random_rows(2000, 16, seed=3)
    assert hc.xsk_derive(parents, pidx, cidx) == hd.xsk_derive_rows(parents, pidx, cidx)
    xp = [hd.xpgk_from_xsk(x) for x in parents]
    pidx, cidx = hd.random_rows(2000, 16, seed=4)
    pidx = [p for p in pidx]
    cidx = [c & 0x7fffffff if k % 4 else c for k, c in enumerate(cidx)]     # mostly non-hardened, so most rows derive
    assert hc.xpgk_derive(xp, pidx, cidx) == hd.xpgk_derive_rows(xp, pidx, cidx)


def test_bad_named_parent_is_refused_by_both():
    parents = hd.random_xsk_parents(5, seed=6)
    parents[3] = parents[3][:41] + b"\xff" * 32
    parents[1] = parents[1][:41] + rj.scalar_bytes(rj.R_J)
    for f in (hd.xsk_derive_rows, hc.xsk_derive):
        with pytest.raises(hd.NotInField, match=r"parents\[1\]"):
            f(parents, [0, 3, 1], [0, 0, 0])
        assert f(parents, [0, 2, 4, 7], [0, 1, 2, 3])[3][4] == hd.BAD_INDEX        # unnamed bad parents are not read


# ---- the reference's tests (derive/mod.rs:267-319) as properties, in both oracles -------------------------------------------
def _seeds(n):
    rng = np.random.default_rng(11)
    return [rng.bytes(32) for _ in range(n)]


def test_derive_nonhardened_child_property():
    """From(xsk.derive(i)) == xpgk.derive(i) for non-hardened i"""
    seeds = _seeds(24)
    masters = [hd.master(s) for s in seeds]
    xpgks = [hd.xpgk_from_xsk(m) for m in masters]
    idx = [3] + [int(v) for v in np.random.default_rng(12).integers(0, 2 ** 31, len(seeds) - 1)]
    for m, x, i in zip(masters, xpgks, idx):
        st, child = hd.xpgk_derive_child(x, i)
        assert st == 0 and hd.xpgk_from_xsk(hd.xsk_derive_child(m, i)) == child
    rows = list(range(len(seeds)))
    cx = hc.xsk_derive(masters, rows, idx)
    cp = hc.xpgk_derive(xpgks, rows, idx)
    assert [r[1] for r in cx] == [r[0] for r in cp] and {r[3] for r in cp} == {0}
    assert [r[2:4] for r in cx] == [r[1:3] for r in cp]


def test_derive_hardened_child_property():
    """an xpgk refuses a hardened index; From(xsk.derive(h)).derive(n) == From(xsk.derive(h).derive(n))"""
    seeds = _seeds(16)
    rng = np.random.default_rng(13)
    for s in seeds:
        m = hd.master(s)
        h, nh = int(rng.integers(2 ** 31, 2 ** 32)), int(rng.integers(0, 2 ** 31))
        assert hd.xpgk_derive_child(hd.xpgk_from_xsk(m), h)[0] == hd.HARDENED_INDEX
        xh = hd.xsk_derive_child(m, h)
        st, child = hd.xpgk_derive_child(hd.xpgk_from_xsk(xh), nh)
        assert st == 0 and child == hd.xpgk_from_xsk(hd.xsk_derive_child(xh, nh))
        assert hc.xpgk_derive([hd.xpgk_from_xsk(m)], [0], [h])[0][3] == hd.HARDENED_INDEX
        c1 = hc.xsk_derive([m], [0], [h])[0]
        assert c1[0] == xh
        assert hc.xpgk_derive([c1[1]], [0], [nh])[0][0] == hc.xsk_derive([xh], [0], [nh])[0][1] == child


def test_read_write_property():
    """write then read gives the same value, for xsks and xpgks at every depth reached"""
    for s in _seeds(8):
        x = hd.master(s)
        for i in (0, 2 ** 31 + 1, 7):
            for k in (x, hd.xpgk_from_xsk(x)):
                if k is x:
                    assert hd.write(*hd.read_xsk(k)[:4], rj.scalar_bytes(hd.read_xsk(k)[4])) == k
                else:
                    st, f = hd.read_xpgk(k)
                    assert st == 0 and hd.write(*f[:4], jj.encode(f[4])) == k
            x = hd.xsk_derive_child(x, i)
            assert x[0] <= 3 and struct.unpack("<I", x[5:9])[0] == i
