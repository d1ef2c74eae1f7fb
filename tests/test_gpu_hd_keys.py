"""GPU tests of zk_xsk_master_batch, zk_xsk_derive_batch and zk_xpgk_derive_batch with their _device forms: every output
byte-equal to the C oracle on edge rows (indices 0, 2^31 - 1, 2^31, 2^32 - 1; parent depths 0, 254, 255; sk = 0 and
r_J - 1; an identity pgk; all-zero and all-0xff chain codes; out-of-range parents; pgks failing each way) and on 2^16 random
rows; a parent table with failing parents no row names; the reference's derive tests as properties over 10^4 rows; a
depth-3 path chained through the device forms; derived accounts that receive confidential transfers, decrypt them with the
watch-only dks and sign with the derived sks; and the argument errors."""
import numpy as np
import pytest

from tests.jubjub_oracle import hd_coracle as hc
from tests.jubjub_oracle import hd_keys as hd
from tests.jubjub_oracle import redjubjub as rj
from zero_chain_b200 import _lib
from zero_chain_b200 import groth16 as zk

pytestmark = pytest.mark.gpu
XK = hd.XK


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


def _t(b: bytes):
    import torch
    return torch.from_numpy(np.frombuffer(b if b else b"\0", np.uint8).copy()).cuda()


def _z(n: int):
    import torch
    return torch.full((max(n, 1),), 0xEE, dtype=torch.uint8, device="cuda")


def _u32(v):
    import torch
    return torch.from_numpy(np.ascontiguousarray(np.asarray(v, np.int64).reshape(-1).astype(np.uint32)).view(np.int32).copy()).cuda()


def _rows(t, size, n):
    b = t.cpu().numpy().tobytes()
    return [b[size * i:size * (i + 1)] for i in range(n)]


# ---- the three calls in both forms, as lists of row tuples in the C oracle's layout -----------------------------------------
def master_host(ctx, seeds):
    return list(zip(*zk.xsk_master(ctx, seeds)))


def master_device(ctx, seeds):
    import torch
    n = len(seeds)
    off = torch.from_numpy(zk.message_offsets(seeds).view(np.int64).copy()).cuda()
    sd = _t(b"".join(seeds))
    outs = [_z(XK * n), _z(XK * n), _z(32 * n), _z(32 * n)]
    torch.cuda.synchronize()                      # the fills above run on torch's stream, the call on the context's
    zk.xsk_master_device(ctx, n, sd.data_ptr(), off.data_ptr(), *(o.data_ptr() for o in outs))
    ctx.sync()
    return list(zip(_rows(outs[0], XK, n), _rows(outs[1], XK, n), _rows(outs[2], 32, n), _rows(outs[3], 32, n)))


def xsk_host(ctx, parents, pidx, cidx):
    return list(zip(*zk.xsk_derive(ctx, parents, pidx, cidx)))


def _launch_xsk(ctx, parents, pidx, cidx):
    import torch
    n = len(pidx)
    pb = _t(b"".join(parents)) if parents else None
    ins = [_u32(pidx), _u32(cidx)]
    outs = [_z(XK * n), _z(XK * n), _z(32 * n), _z(32 * n), _z(n)]
    torch.cuda.synchronize()                      # the fills above run on torch's stream, the call on the context's
    zk.xsk_derive_device(ctx, len(parents), pb.data_ptr() if pb is not None else 0, n, *(x.data_ptr() for x in ins + outs))
    return [pb] + ins + outs                      # alive until the context's stream is done with them


def _read_xsk(bufs, n):
    outs = bufs[3:]
    return list(zip(_rows(outs[0], XK, n), _rows(outs[1], XK, n), _rows(outs[2], 32, n), _rows(outs[3], 32, n),
                    [int(v) for v in outs[4].cpu().numpy()[:n]]))


def xsk_device(ctx, parents, pidx, cidx):
    bufs = _launch_xsk(ctx, parents, pidx, cidx)
    ctx.sync()
    return _read_xsk(bufs, len(pidx))


def xpgk_host(ctx, parents, pidx, cidx):
    return list(zip(*zk.xpgk_derive(ctx, parents, pidx, cidx)))


def xpgk_device(ctx, parents, pidx, cidx):
    import torch
    n = len(pidx)
    pb = _t(b"".join(parents)) if parents else None
    ins = [_u32(pidx), _u32(cidx)]
    outs = [_z(XK * n), _z(32 * n), _z(32 * n), _z(n)]
    torch.cuda.synchronize()
    zk.xpgk_derive_device(ctx, len(parents), pb.data_ptr() if pb is not None else 0, n, *(x.data_ptr() for x in ins + outs))
    ctx.sync()
    return list(zip(_rows(outs[0], XK, n), _rows(outs[1], 32, n), _rows(outs[2], 32, n), [int(v) for v in outs[3].cpu().numpy()[:n]]))


# ---- parity with the C oracle ---------------------------------------------------------------------------------------------
def test_master_matches_oracle_both_forms(ctx):
    rng = np.random.default_rng(1)
    seeds = [b"", b"Alice" + b" " * 27] + [rng.bytes(int(k)) for k in rng.integers(1, 300, 998)]
    want = hc.master(seeds)
    assert master_host(ctx, seeds) == want == master_device(ctx, seeds)
    xs, xp, d, e = zk.xsk_master(ctx, seeds[:5], xpgk=False, dk=False, ek=True)
    assert xs == [w[0] for w in want[:5]] and xp is None and d is None and e == [w[3] for w in want[:5]]


def test_edge_rows_match_oracle_both_forms(ctx):
    parents = hd.edge_xsk_parents()
    pidx, cidx = hd.edge_rows(len(parents))
    want = hc.xsk_derive(parents, pidx, cidx)
    assert want == hd.xsk_derive_rows(parents, pidx, cidx)
    assert {w[4] for w in want} == {0, zk.HD_BAD_INDEX, zk.HD_DEPTH}
    assert xsk_host(ctx, parents, pidx, cidx) == want == xsk_device(ctx, parents, pidx, cidx)
    xp = hd.edge_xpgk_parents()
    pidx, cidx = hd.edge_rows(len(xp))
    want = hc.xpgk_derive(xp, pidx, cidx)
    assert want == hd.xpgk_derive_rows(xp, pidx, cidx)
    assert {w[3] for w in want} == {0, 1, 2, 3, zk.HD_BAD_INDEX, zk.HD_HARDENED_INDEX, zk.HD_DEPTH}
    assert xpgk_host(ctx, xp, pidx, cidx) == want == xpgk_device(ctx, xp, pidx, cidx)


def test_random_rows_match_oracle_both_forms(ctx):
    n = 1 << 16
    parents = hd.random_xsk_parents(512, seed=2)
    pidx, cidx = hd.random_rows(n, 512, seed=3)
    want = hc.xsk_derive(parents, pidx, cidx)
    assert xsk_host(ctx, parents, pidx, cidx) == want
    assert xsk_device(ctx, parents, pidx, cidx) == want
    xs, xp, d, e, st = zk.xsk_derive(ctx, parents, pidx, cidx, xpgk=False, dk=False, ek=False)   # hashes and one addition
    assert xs == [w[0] for w in want] and st == [w[4] for w in want] and xp is d is e is None
    xpar = [hd.xpgk_from_xsk(x) for x in parents]
    cidx = [c & 0x7fffffff if k % 8 else c for k, c in enumerate(cidx)]
    want = hc.xpgk_derive(xpar, pidx, cidx)
    assert xpgk_host(ctx, xpar, pidx, cidx) == want
    assert xpgk_device(ctx, xpar, pidx, cidx) == want


def test_unnamed_failing_parents_are_not_read(ctx):
    """a 20000-parent table, every 7th parent failing (sk >= r_J, or a pgk failing each way); the rows name only good ones"""
    good = hd.random_xsk_parents(64, seed=4)
    bad_x = [g[:41] + rj.scalar_bytes(rj.R_J + k) for k, g in enumerate(good[:4])]
    bad_p = [hd.write(1, bytes(4), 0, good[0][9:41], k) for k, _ in hd.bad_pgks()]
    xs, xp, named = [], [], []
    for k in range(20000):
        if k % 7 == 3:
            xs.append(bad_x[k % 4]); xp.append(bad_p[k % 3])
        else:
            xs.append(good[k % 64]); xp.append(hd.xpgk_from_xsk(good[k % 64]))
            named.append(k)
    rng = np.random.default_rng(5)
    pidx = [named[int(v)] for v in rng.integers(0, len(named), 3000)]
    cidx = [int(v) for v in rng.integers(0, 2 ** 31, 3000)]
    want = hc.xsk_derive([xs[p] for p in pidx], list(range(3000)), cidx)
    assert {w[4] for w in want} <= {0, zk.HD_DEPTH}
    assert xsk_host(ctx, xs, pidx, cidx) == want == xsk_device(ctx, xs, pidx, cidx)
    want = hc.xpgk_derive([xp[p] for p in pidx], list(range(3000)), cidx)
    assert xpgk_host(ctx, xp, pidx, cidx) == want == xpgk_device(ctx, xp, pidx, cidx)


# ---- the reference's tests (zface/src/derive/mod.rs:267-319) as properties at scale ----------------------------------------
def test_reference_properties_at_scale(ctx):
    n = 10000
    rng = np.random.default_rng(6)
    seeds = [rng.bytes(32) for _ in range(100)]
    ms, mp, _, _ = zk.xsk_master(ctx, seeds, dk=False, ek=False)
    pidx = [int(v) for v in rng.integers(0, 100, n)]
    nh = [int(v) for v in rng.integers(0, 2 ** 31, n)]
    hard = [int(v) for v in rng.integers(2 ** 31, 2 ** 32, n, dtype=np.uint64)]
    # derive_nonhardened_child: From(xsk.derive(i)) == xpgk.derive(i)
    xs, xsp, xsd, xse, st = zk.xsk_derive(ctx, ms, pidx, nh)
    xp, xpd, xpe, st2 = zk.xpgk_derive(ctx, mp, pidx, nh)
    assert st == st2 == [0] * n and xsp == xp and xsd == xpd and xse == xpe
    # derive_hardened_child: an xpgk refuses a hardened index; below a hardened child the two paths agree again
    assert zk.xpgk_derive(ctx, mp, pidx, hard)[3] == [zk.HD_HARDENED_INDEX] * n
    hs, hp, _, _, st = zk.xsk_derive(ctx, ms, pidx, hard, dk=False, ek=False)
    assert st == [0] * n
    a = zk.xsk_derive(ctx, hs, list(range(n)), nh)
    b = zk.xpgk_derive(ctx, hp, list(range(n)), nh)
    assert a[1] == b[0] and a[2:4] == b[1:3]
    # read_write: the written keys read back (a parent table of written keys derives without error) and keep their fields
    assert all(hd.write(*hd.read_xsk(x)[:4], x[41:]) == x for x in xs)
    for x in xp[:200]:
        st, f = hd.read_xpgk(x)
        assert st == 0 and hd.write(*f[:4], hd.jj.encode(f[4])) == x
    assert [x[0] for x in xs] == [1] * n and [x[5:9] for x in xs] == [i.to_bytes(4, "little") for i in nh]
    assert hc.xsk_derive(ms, pidx[:500], nh[:500]) == list(zip(xs, xsp, xsd, xse, [0] * n))[:500]


def test_depth3_path_chained_on_the_device(ctx):
    """m / 44' / k / j for 8 masters, 4 accounts and 16 addresses: three device calls, each level's xsks the next level's
    parents, with no host round trip, equal three host calls"""
    import torch
    seeds = [b"path seed %d" % i for i in range(8)]
    ms = zk.xsk_master(ctx, seeds)[0]
    levels = [([i for i in range(8)], [2 ** 31 + 44] * 8), ([p for p in range(8) for _ in range(4)], [k for _ in range(8) for k in range(4)]),
              ([p for p in range(32) for _ in range(16)], [2 ** 31 - 1 - j if j % 2 else j for _ in range(32) for j in range(16)])]
    # host
    parents = ms
    for pidx, cidx in levels:
        out = zk.xsk_derive(ctx, parents, pidx, cidx)
        assert out[4] == [0] * len(pidx)
        parents = out[0]
    want = list(zip(*out))
    # device
    d_par = _t(b"".join(ms))
    n_par = 8
    keep = [d_par]                                # every level's buffers stay alive until the context's stream is done
    for pidx, cidx in levels:
        n = len(pidx)
        ins = [_u32(pidx), _u32(cidx)]
        outs = [_z(XK * n), _z(XK * n), _z(32 * n), _z(32 * n), _z(n)]
        torch.cuda.synchronize()                  # the fills run on torch's stream, the calls on the context's
        zk.xsk_derive_device(ctx, n_par, d_par.data_ptr(), n, *(x.data_ptr() for x in ins + outs))
        keep += ins + outs
        d_par, n_par = outs[0], n
    ctx.sync()
    got = list(zip(_rows(outs[0], XK, n), _rows(outs[1], XK, n), _rows(outs[2], 32, n), _rows(outs[3], 32, n),
                   [int(v) for v in outs[4].cpu().numpy()[:n]]))
    assert got == want
    assert {g[0][0] for g in got} == {3}
    torch.cuda.synchronize()


# ---- end to end: derived accounts send, receive, decrypt watch-only and sign -----------------------------------------------
def test_derived_accounts_transfer_decrypt_and_sign(ctx):
    rng = np.random.default_rng(7)
    m = zk.xsk_master(ctx, [b"exchange wallet seed"])
    n = 256
    xs, xp, dks, eks, st = zk.xsk_derive(ctx, m[0], [0] * n, list(range(n)))
    assert st == [0] * n
    # the watch-only holder derives the same accounts from the master xpgk alone
    wp, wdk, wek, wst = zk.xpgk_derive(ctx, m[1], [0] * n, list(range(n)))
    assert wst == [0] * n and wp == xp and wdk == dks and wek == eks
    sks = [x[41:] for x in xs]
    fs = lambda: int.from_bytes(rng.bytes(64), "little") % rj.R_J
    sender = [int(v) for v in rng.integers(0, n, 400)]
    recipient = [(s + 1 + int(v)) % n for s, v in zip(sender, rng.integers(0, n - 1, 400))]
    amounts = [int(v) for v in rng.integers(0, 10 ** 6, 400)]
    g = zk.g_epoch(ctx, [3])[0]
    fields, rsks, fdks, fst = zk.confidential_fields(ctx, [sks[s] for s in sender], [eks[r] for r in recipient], amounts, [1] * 400,
                                                     [fs() for _ in range(400)], [fs() for _ in range(400)], g)
    assert fst == [0] * 400 and fdks == [dks[s] for s in sender]
    cts = [f["amount_recipient"] + f["randomness"] for f in fields]
    assert zk.elgamal_decrypt(ctx, [wdk[r] for r in recipient], cts) == ([zk.ELGAMAL_OK] * 400, amounts)
    assert zk.elgamal_decrypt(ctx, [wdk[s] for s in sender], [f["amount_sender"] + f["randomness"] for f in fields]) == \
        ([zk.ELGAMAL_OK] * 400, amounts)
    msgs = [b"transfer %d" % i for i in range(400)]
    sigs = zk.redjubjub_sign(ctx, rsks, msgs, [rng.bytes(80) for _ in range(400)])
    assert zk.redjubjub_verify(ctx, [f["rvk"] for f in fields], sigs, msgs) == [zk.REDJUBJUB_OK] * 400
    # and a derived sk signs under its own public key, sk P_G, the key of its xpgk
    sigs = zk.redjubjub_sign(ctx, sks[:32], msgs[:32], [rng.bytes(80) for _ in range(32)])
    assert zk.redjubjub_verify(ctx, [x[41:] for x in wp[:32]], sigs, msgs[:32]) == [zk.REDJUBJUB_OK] * 32


# ---- the context's workspace --------------------------------------------------------------------------------------------
def test_destroy_releases_the_parent_workspace():
    """the derive calls keep a per-parent workspace in the context (about 134 B per parent for an xpgk table); destroying
    the context gives it back.  2^21 parents make it about 300 MB, and six contexts in turn would hold 1.8 GB if it were
    kept; the device's free memory is allowed a 600 MB drift for other work on the card."""
    import torch
    n_par = 1 << 21
    xp = hd.xpgk_from_xsk(hd.master(b"workspace"))
    parents = torch.zeros(XK * n_par, dtype=torch.uint8, device="cuda")
    parents[:XK] = torch.from_numpy(np.frombuffer(xp, np.uint8).copy()).cuda()
    bufs = [_u32([0]), _u32([5]), _z(XK), _z(32), _z(32), _z(1)]
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for k in range(6):
        c = zk.Context(0)
        zk.xpgk_derive_device(c, n_par, parents.data_ptr(), 1, *(b.data_ptr() for b in bufs))
        c.sync()
        if k == 0:
            assert free0 - torch.cuda.mem_get_info()[0] > 200 << 20      # the workspace is there while the context lives
        c.close()
    assert free0 - torch.cuda.mem_get_info()[0] < 600 << 20
    assert _rows(bufs[2], XK, 1)[0] == hc.xpgk_derive([xp], [0], [5])[0][0]


# ---- errors ---------------------------------------------------------------------------------------------------------------
def test_errors(ctx):
    parents = hd.random_xsk_parents(6, seed=8)
    parents = [bytes([min(p[0], 254)]) + p[1:] for p in parents]
    bad = list(parents)
    bad[4] = bad[4][:41] + rj.scalar_bytes(rj.R_J)
    with pytest.raises(zk.SynthesisError, match=r"parents\[4\]") as e:
        zk.xsk_derive(ctx, bad, [0, 4, 1], [1, 2, 3])
    assert e.value.code == -8
    assert zk.xsk_derive(ctx, bad, [0, 1, 5], [1, 2, 3])[4] == [0, 0, 0]           # not named: not read
    assert zk.xsk_derive(ctx, [], [0, 3], [1, 2])[4] == [zk.HD_BAD_INDEX] * 2
    assert zk.xsk_derive(ctx, parents, [], []) == ([], [], [], [], [])
    # the device form leaves the rows naming the bad parent unwritten, writes the others, and reports at the next sync
    bufs = _launch_xsk(ctx, bad, [0, 4, 1, 4], [1, 2, 3, 4])
    with pytest.raises((zk.SynthesisError, _lib.ZkError)) as e:
        ctx.sync()                                # synchronises the context's stream before it reports
    assert e.value.code == -8
    got = _read_xsk(bufs, 4)
    untouched = (b"\xee" * XK, b"\xee" * XK, b"\xee" * 32, b"\xee" * 32, 0xEE)
    assert got[1] == got[3] == untouched
    want = hc.xsk_derive(parents, [0, 1], [1, 3])
    assert [got[0], got[2]] == want
    assert xsk_device(ctx, parents, [0, 1], [1, 3]) == want                        # the context stays usable
