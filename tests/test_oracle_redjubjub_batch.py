"""CPU checks of the batch-verification oracles (tests/jubjub_oracle): the Python and C restatements of
redjubjub::batch_verify agree on mixed corpora under several z seeds; all-valid batches pass and one swapped message or
signature fails; the reference's test_batch_verify scenario with the Diversifier generator; a vk plus a point of order 8
still passes (as in the reference's cofactor_check); a bad entry with z_i = 0 passes, which pins the exact equation; the
"batch first, per-signature fallback" pattern gives the per-signature verdicts; and the oracle multiexp's closed form."""
import numpy as np

from tests.jubjub_oracle import pyref as jj
from tests.jubjub_oracle import redjubjub as rj
from tests.jubjub_oracle import rj_batch as rjb
from tests.jubjub_oracle import rjb_coracle as cjb
from tests.jubjub_oracle import rj_coracle as cj
from tests.jubjub_oracle import rj_corpus

R_J = rj.R_J


def _zs(n, seed):
    rng = np.random.default_rng(seed)
    return [int.from_bytes(rng.bytes(64), "little") % R_J for _ in range(n)]


def _both(vks, sigs, msgs, zs):
    py = rjb.batch_verify(vks, sigs, msgs, zs)
    c = cjb.redjubjub_batch_verify(b"".join(vks), b"".join(sigs), msgs, b"".join(z.to_bytes(32, "little") for z in zs))
    assert py == c
    return py


def test_python_and_c_agree_on_mixed_corpora():
    entries, _ = rj_corpus.mixed(64, seed=41)
    want = [rj_corpus.python_verdict(e) for e in entries]
    valid = [e for e, w in zip(entries, want) if w == rj.OK]
    seen = set()
    for seed in range(3):
        for lo in range(seed, len(entries), 3):
            batch = valid[:5] + entries[lo:lo + 3]
            vks, sigs, msgs = rj_corpus.columns(batch)
            got = _both([e[0] for e in batch], [e[1] for e in batch], msgs, _zs(len(batch), seed * 100 + lo))
            seen.add(got[0])
            per = [rj_corpus.python_verdict(e) for e in batch]
            first = next((i for i, v in enumerate(per) if v in (2, 3, 4)), None)
            if first is not None:
                assert got == (per[first], first)
            else:
                assert got == ((1, None) if all(v == 1 for v in per) else (0, None))
    assert seen == {0, 1, 2, 3, 4}


def test_valid_batch_and_swaps():
    entries, _ = rj_corpus.mixed(24, seed=42)
    valid = [e for e in entries if rj_corpus.python_verdict(e) == rj.OK][:12]
    vks, sigs, msgs = [e[0] for e in valid], [e[1] for e in valid], [e[2] for e in valid]
    zs = _zs(len(valid), 1)
    assert _both(vks, sigs, msgs, zs) == (1, None)
    assert _both(vks, sigs, msgs[:3] + [msgs[4]] + msgs[4:], zs) == (0, None)
    assert _both(vks, sigs[:5] + [sigs[6]] + sigs[6:], msgs, zs) == (0, None)


def test_reference_batch_scenario():
    """redjubjub.rs test_batch_verify with the Diversifier generator: two signatures over "Foo bar", then batch[0].sig = sig2."""
    rng = np.random.default_rng(43)
    sk1, sk2 = [int.from_bytes(rng.bytes(64), "little") % R_J for _ in range(2)]
    vk1, vk2 = rj.public_key(sk1), rj.public_key(sk2)
    msg = b"Foo bar"
    sig1, sig2 = rj.sign(sk1, msg, rng.bytes(80)), rj.sign(sk2, msg, rng.bytes(80))
    assert rj.verify(vk1, msg, sig1) == rj.verify(vk2, msg, sig2) == rj.OK
    assert _both([vk1, vk2], [sig1, sig2], [msg, msg], _zs(2, 2)) == (1, None)
    assert _both([vk1, vk2], [sig2, sig2], [msg, msg], _zs(2, 3)) == (0, None)


def test_torsion_vk_passes():
    rng = np.random.default_rng(44)
    sk = int.from_bytes(rng.bytes(64), "little") % R_J
    msg = b"Foo bar"
    sig = rj.sign(sk, msg, rng.bytes(80))
    _, a = jj.read(rj.public_key(sk))
    vk8 = jj.encode(jj.add(a, jj.torsion_point(8)))
    assert rj.verify(vk8, msg, sig) == rj.OK
    assert _both([vk8, rj.public_key(sk)], [sig, sig], [msg, msg], _zs(2, 4)) == (1, None)


def test_zero_randomizer_lets_a_bad_entry_pass():
    entries, _ = rj_corpus.mixed(16, seed=45)
    valid = [e for e in entries if rj_corpus.python_verdict(e) == rj.OK][:6]
    vks, sigs, msgs = [e[0] for e in valid], [e[1] for e in valid], [e[2] for e in valid]
    msgs[2] = msgs[2] + b"forged"
    zs = _zs(6, 5)
    assert _both(vks, sigs, msgs, zs) == (0, None)
    zs[2] = 0
    assert _both(vks, sigs, msgs, zs) == (1, None)


def test_batch_first_then_per_signature():
    """The pattern of groth16.redjubjub_verify_batched, on the oracles: per-signature verdicts whatever the batch holds."""
    entries, _ = rj_corpus.mixed(32, seed=46)
    for lo in range(0, len(entries), 7):
        batch = entries[lo:lo + 7]
        vks, sigs, msgs = rj_corpus.columns(batch)
        per = [rj_corpus.python_verdict(e) for e in batch]
        v, _ = cjb.redjubjub_batch_verify(vks, sigs, msgs, b"".join(z.to_bytes(32, "little") for z in _zs(len(batch), lo)))
        batched = [rj.OK] * len(batch) if v == rj.OK else [int(x) for x in cj.redjubjub_verify(vks, sigs, msgs)]
        assert batched == per


def test_multiexp_closed_form():
    rng = np.random.default_rng(47)
    n = 12
    ss = [int.from_bytes(rng.bytes(32), "little") % R_J for _ in range(n)] + [0, R_J - 1]
    bases = [jj.mul(rj.P_G, i) for i in range(1, len(ss) + 1)]
    want = jj.mul(rj.P_G, sum(s * i for i, s in enumerate(ss, 1)) % R_J)
    assert rjb.multiexp(bases, ss) == want
