"""GPU tests of zk_import_block and its _device form (groth16.block_import / block_import_device): a block's extrinsic
signatures, then the confidential transfers, the encrypted-asset calls and the anonymous-balances calls in one call,
with the verifier launches shared across sections.

Every section's output is checked against its own call (confidential_import, asset_calls_import, anonymous_import) on
the same section, and against the corpora's C oracles.  All sections verify with one toy 11-point key and one 52-point
key (tests/import_corpus.py, import_anon_corpus.py); the signatures come from tests/jubjub_oracle/redjubjub.py."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from tests import import_anon_corpus as iac
from tests import import_corpus as ic
from tests.jubjub_oracle import redjubjub as rj
from zero_chain_b200 import _lib
from zero_chain_b200 import groth16 as zk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = zk.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def keys(ctx):
    conf, anon = iac.ForgeKey(zk.CONFIDENTIAL_POINTS, 171), iac.ForgeKey(zk.ANONYMOUS_POINTS, 71)
    conf.pvk = zk.PreparedVerifyingKey.prepare(ctx, conf.params_bytes)
    anon.pvk = zk.PreparedVerifyingKey.prepare(ctx, anon.params_bytes)
    yield conf, anon
    conf.pvk.free()
    anon.pvk.free()


def signatures(n, seed, bad=()):
    """n signed extrinsics; bad: {index: how} with how in "tamper", "vk", "rbar", "sbar" """
    vks, sigs, msgs = [], [], []
    for i in range(n):
        sk = rj.spending_key(b"block-%d-%d" % (seed, i))
        msg = b"extrinsic %d of block %d" % (i, seed)
        vk, sig = rj.public_key(sk), rj.sign(sk, msg, bytes([i % 256]) * 80)
        how = dict(bad).get(i)
        if how == "tamper":
            msg = msg + b"!"
        elif how == "vk":
            vk = (2).to_bytes(32, "little")                  # y = 2 is not on the curve
        elif how == "rbar":
            sig = (2).to_bytes(32, "little") + sig[32:]
        elif how == "sbar":
            sig = sig[:32] + b"\xff" * 32
        vks.append(vk)
        sigs.append(sig)
        msgs.append(msg)
    return vks, sigs, msgs, None


def sections(keys, seed, conf_fail=0.0, asset_fail=0.0, anon_fail=0.0, present=(True, True, True), n=(120, 90, 60)):
    conf, anon = keys
    c = ic.confidential(conf, 24, n[0], seed, fail_frac=conf_fail) if present[0] else None
    a = ic.assets(conf, 12, n[1], seed + 1, fail_frac=asset_fail, fixed_fail_frac=asset_fail) if present[1] else None
    b = iac.block(anon, conf, 40, n[2], seed + 2, issue_frac=0.2, fail_frac=anon_fail) if present[2] else None
    return c, a, b


def check(ctx, keys, c, a, b, n_sig=5, seed=0):
    """block_import against each section's own call and the oracles; returns (result, own rounds)"""
    conf, anon = keys
    got = zk.block_import(ctx, conf.pvk, anon.pvk, signatures(n_sig, seed), confidential=(c.accounts, c.txs, c.proofs) if c else None,
                          assets=a.args() if a else None, anonymous=b.args() if b else None)
    launches = 0
    if c:
        want = zk.confidential_import(ctx, conf.pvk, c.accounts, c.txs, c.proofs)
        assert got.confidential == want and want[0] == c.intended
        o = c.oracle(want[0])
        assert want[2] == o[0] and want[1] == tuple(o[2:])
        launches += want[3]
    else:
        assert got.confidential is None
    if a:
        want = zk.asset_calls_import(ctx, conf.pvk, *a.args())
        assert got.assets == want and want[0] == a.intended
        assert want[3][1:] == a.oracle(want[0])[5:]
        launches += want[4] + any(t.kind != zk.ASSET_TRANSFER for t in a.txs)
    else:
        assert got.assets is None
    if b:
        want = zk.anonymous_import(ctx, anon.pvk, conf.pvk, *b.args())
        assert got.anonymous == want and want[0] == b.intended
        o = b.oracle(want[0])
        assert want[2] == o[0] and want[1] == o[4:]
        launches += any(t.kind == zk.ANON_ISSUE for t in b.txs) + any(t.kind == zk.ANON_TRANSFER for t in b.txs)
    else:
        assert got.anonymous is None
    assert got.launches <= launches
    return got


def test_no_failures_take_three_launches(ctx, keys):
    got = check(ctx, keys, *sections(keys, 10))
    assert got.launches == 3
    assert got.confidential[3] == 1 and got.assets[4] == 1


@pytest.mark.parametrize("seed, rates", [(20, (0.1, 0.0, 0.1)), (30, (0.0, 0.15, 0.05)), (40, (0.3, 0.05, 0.2))])
def test_failures_in_every_kind_equal_the_own_calls(ctx, keys, seed, rates):
    c, a, b = sections(keys, seed, *rates)
    got = check(ctx, keys, c, a, b)
    r_conf, r_assets = got.confidential[3], got.assets[4]
    assert got.launches == max(r_conf, 1 + r_assets) + 1


@pytest.mark.parametrize("present", [p for p in itertools.product([False, True], repeat=3)])
def test_every_combination_of_sections(ctx, keys, present):
    got = check(ctx, keys, *sections(keys, 50, 0.05, 0.05, 0.05, present, n=(40, 30, 20)))
    if present == (True, False, False):
        assert got.launches == got.confidential[3]
    if not any(present):
        assert got.launches == 0


def test_asset_transfers_only_spend_no_launch_on_an_empty_l1(ctx, keys):
    conf, _ = keys
    a = ic.assets(conf, 12, 50, 61, fail_frac=0.1, issue_frac=0.0, destroy_frac=0.0)
    got = check(ctx, keys, None, a, None)
    assert got.launches == got.assets[4]


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_a_tampered_signature_rejects_the_block_and_writes_nothing(ctx, keys, where):
    conf, anon = keys
    n = 7
    i = {"first": 0, "middle": 3, "last": n - 1}[where]
    c, a, b = sections(keys, 70, 0.05, 0.05, 0.05, n=(20, 20, 20))
    with pytest.raises(zk.BadSignature) as e:
        zk.block_import(ctx, conf.pvk, anon.pvk, signatures(n, 70, {i: "tamper"}), (c.accounts, c.txs, c.proofs), a.args(), b.args())
    assert (e.value.index, e.value.verdict, e.value.code) == (i, 0, _lib.ZK_ERR_BAD_SIGNATURE)


@pytest.mark.parametrize("bad, want", [({4: "vk"}, (4, 2)), ({2: "rbar"}, (2, 3)), ({5: "sbar"}, (5, 4)),
                                       ({6: "vk", 1: "sbar", 3: "tamper"}, (1, 4))])
def test_rejected_encodings_name_the_lowest_extrinsic(ctx, keys, bad, want):
    conf, anon = keys
    c = ic.confidential(conf, 8, 10, 80)
    with pytest.raises(zk.BadSignature) as e:
        zk.block_import(ctx, conf.pvk, anon.pvk, signatures(8, 80, bad), (c.accounts, c.txs, c.proofs))
    assert (e.value.index, e.value.verdict) == want


def test_no_signatures_and_a_valid_set_pass(ctx, keys):
    c, a, b = sections(keys, 90, n=(10, 10, 10))
    conf, anon = keys
    args = dict(confidential=(c.accounts, c.txs, c.proofs), assets=a.args(), anonymous=b.args())
    assert zk.block_import(ctx, conf.pvk, anon.pvk, ([], [], [], None), **args) == \
        zk.block_import(ctx, conf.pvk, anon.pvk, signatures(30, 90), **args)


def test_an_index_error_names_its_section_before_a_bad_signature(ctx, keys):
    conf, anon = keys
    c = ic.confidential(conf, 8, 10, 100)
    c.txs[6].recipient = 8
    with pytest.raises(ValueError, match="block_import: confidential: .*transaction 6"):
        zk.block_import(ctx, conf.pvk, anon.pvk, signatures(3, 100, {0: "tamper"}), (c.accounts, c.txs, c.proofs))
    b = iac.block(anon, conf, 20, 12, 101, issue_frac=0.3)
    b.txs[4].members[3] = 20 if b.txs[4].kind == zk.ANON_TRANSFER else b.txs[4].members[3]
    b.txs[4].members[0] = 20
    with pytest.raises(ValueError, match="block_import: anonymous: .*transaction 4"):
        zk.block_import(ctx, conf.pvk, anon.pvk, signatures(3, 100, {1: "tamper"}), anonymous=b.args())


def test_swapped_keys_are_malformed(ctx, keys):
    conf, anon = keys
    c = ic.confidential(conf, 8, 10, 110)
    with pytest.raises(zk.SynthesisError):
        zk.block_import(ctx, anon.pvk, conf.pvk, signatures(2, 110), (c.accounts, c.txs, c.proofs))


# where each section's outputs start among its C arguments (after them come only the host pointers rounds / n_out)
OUT_FROM = (9, 13, 13)


class DeviceBlock:
    """block_import's arguments on the device: every array of each section's C arguments copied to its own device buffer
    (outputs prefilled with fill, when given); run() calls block_import_device and returns what block_import would"""

    def __init__(self, ctx, keys, signatures, c, a, b, fill=None):
        self.ctx, self.keys = ctx, keys
        vks, sigs, msgs, zs = signatures
        zs = zk.random_batch_scalars(len(msgs)) if zs is None else zs
        dev = lambda x: torch.tensor(list(x) or [0], dtype=torch.uint8, device="cuda")
        self.n_sig = len(msgs)
        self.sig = [dev(b"".join(vks)), dev(b"".join(sigs)), dev(b"".join(msgs)),
                    torch.tensor(zk.message_offsets(msgs).astype(np.int64), device="cuda"), dev(zs)]
        self.sections, self.outputs, self.copies, self.buffers = [], [], [], []
        for make, args, out_from in ((zk._conf_section, (c.accounts, c.txs, c.proofs) if c else None, OUT_FROM[0]),
                                     (zk._asset_section, a.args() if a else None, OUT_FROM[1]),
                                     (zk._anon_section, b.args() if b else None, OUT_FROM[2])):
            if args is None:
                self.sections.append(None)
                continue
            cargs, result, keep = make("t", *args)
            t = []
            for j, x in enumerate(cargs):
                if isinstance(x, C.c_void_p):
                    d = torch.from_numpy(x._arr.view(np.uint8).reshape(-1).copy()).to("cuda")
                    self.buffers.append(d)
                    if j >= out_from:
                        if fill is not None:
                            d.fill_(fill)
                        self.outputs.append(d)
                        self.copies.append((x._arr, d))
                    t.append(d.data_ptr())
                elif x is None:
                    t.append(0)
                elif isinstance(x, int):
                    t.append(x)
            self.sections.append((t, cargs, result, keep))
        torch.cuda.synchronize()

    def run(self):
        conf, anon = self.keys
        arg = lambda i: self.sections[i][0] if self.sections[i] else None
        c_rounds, (n_out, a_rounds), launches = zk.block_import_device(self.ctx, conf.pvk, anon.pvk, self.n_sig,
                                                                       *[t.data_ptr() for t in self.sig], arg(0), arg(1), arg(2))
        for arr, d in self.copies:
            arr.view(np.uint8).reshape(-1)[:] = d.cpu().numpy()
        if self.sections[0]:
            self.sections[0][1][-1]._obj.value = c_rounds
        if self.sections[1]:
            self.sections[1][1][-2]._obj.value = n_out
            self.sections[1][1][-1]._obj.value = a_rounds
        return zk.BlockImport(*[s[2]() if s else None for s in self.sections], launches)


@pytest.mark.parametrize("present", [(True, True, True), (False, True, True), (False, True, False), (False, False, True),
                                     (True, False, True), (False, False, False)])
def test_the_device_form_equals_the_host_form(ctx, keys, present):
    conf, anon = keys
    c, a, b = sections(keys, 130, 0.05, 0.05, 0.05, present, n=(30, 30, 20))
    vks, sigs, msgs, _ = signatures(4, 130)
    sig = (vks, sigs, msgs, zk.random_batch_scalars(4))
    host = zk.block_import(ctx, conf.pvk, anon.pvk, sig, confidential=(c.accounts, c.txs, c.proofs) if c else None,
                           assets=a.args() if a else None, anonymous=b.args() if b else None)
    assert DeviceBlock(ctx, keys, sig, c, a, b).run() == host


@pytest.mark.parametrize("bad", [{0: "tamper"}, {3: "vk"}, {5: "rbar"}, {6: "sbar"}])
def test_a_rejected_block_writes_no_output(ctx, keys, bad):
    """the device form on output buffers prefilled with a sentinel: a bad signature leaves every one unchanged"""
    c, a, b = sections(keys, 140, 0.05, 0.05, 0.05, n=(20, 20, 20))
    blk = DeviceBlock(ctx, keys, signatures(7, 140, bad), c, a, b, fill=0xA5)
    with pytest.raises(zk.BadSignature) as e:
        blk.run()
    assert e.value.index == min(bad)
    torch.cuda.synchronize()
    assert blk.outputs and all(bool((d == 0xA5).all()) for d in blk.outputs)


def test_a_z_above_r_j_is_not_canonical(ctx, keys):
    conf, anon = keys
    c = ic.confidential(conf, 8, 10, 145)
    vks, sigs, msgs, _ = signatures(4, 145, {1: "tamper"})
    zs = [bytes(32)] * 2 + [b"\xff" * 32] * 2
    with pytest.raises(zk.SynthesisError, match=r"z\[2\] >= r_J") as e:
        zk.block_import(ctx, conf.pvk, anon.pvk, (vks, sigs, msgs, zs), (c.accounts, c.txs, c.proofs))
    assert e.value.code == -8


def _asset_errors_agree(ctx, keys, a, sig):
    """the asset section's error in the block names the section and the same transaction or row as its own call"""
    conf, anon = keys
    with pytest.raises(Exception) as own:
        zk.asset_calls_import(ctx, conf.pvk, *a.args())
    with pytest.raises(type(own.value)) as blk:
        zk.block_import(ctx, conf.pvk, anon.pvk, sig, assets=a.args())
    tail = str(own.value).split("zk_import_asset_calls: ")[1]
    assert "zk_import_block: assets: " + tail in str(blk.value)
    if isinstance(own.value, ValueError):
        assert str(blk.value).startswith("block_import: assets: ")
    return tail


def test_asset_section_errors(ctx, keys):
    conf, _ = keys
    bad_sig, good_sig = signatures(3, 150, {0: "tamper"}), signatures(3, 150)
    a = ic.assets(conf, 12, 30, 151, issue_frac=0.2, destroy_frac=0.2)
    k = next(i for i, t in enumerate(a.txs) if t.kind == zk.ASSET_DESTROY)
    a.txs[k].kind = 3
    assert _asset_errors_agree(ctx, keys, a, bad_sig).startswith("transaction %d: an unknown kind" % k)
    a = ic.assets(conf, 12, 30, 152, issue_frac=0.2)
    slots = list(a.state[0])
    slots[5] = slots[2]
    a.state = (slots,) + tuple(a.state[1:])
    assert _asset_errors_agree(ctx, keys, a, bad_sig).startswith("slot row 5 repeats")
    a = ic.assets(conf, 12, 30, 153, issue_frac=0.2)
    a.next_asset_id = 2**32 - 1
    second = [i for i, t in enumerate(a.txs) if t.kind == zk.ASSET_ISSUE][1]
    assert _asset_errors_agree(ctx, keys, a, good_sig).startswith("transaction %d: the issue's asset id" % second)
