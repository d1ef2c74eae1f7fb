#!/usr/bin/env python3
"""Generates tests/golden/elgamal.json: the numbers ElGamal balance decryption is pinned to, each with the file and line it
comes from, and the expected decryptions of the reference's own transaction literals.

Run with ZK_REFERENCE pointing at a checkout of the reference; the tests never read the reference itself.
  core/crypto/src/elgamal.rs:102                  the search bound 1_000_000
  src/chain_spec.rs:185, 189                      Alice's genesis balance 10_000, encrypted with randomness Fs::one()
  modules/encrypted-balances/src/lib.rs:295, 302  the module test's balance 100, also with Fs::one()
  core/crypto/src/elgamal.rs:203-332              the amounts of the reference's ElGamal tests
  modules/encrypted-balances/src/lib.rs:443-448   the transaction literals, named as in jubjub_points.json
The expected decryptions were computed with tests/jubjub_oracle/elgamal.py (the None by the C oracle's full walk); the
tests check every one of them again."""
import json
import os
import re
import sys

REF = os.environ.get("ZK_REFERENCE", "")


def number(path, ln, pattern):
    line = open(os.path.join(REF, path)).read().split("\n")[ln - 1]
    m = re.search(pattern, line)
    assert m, (path, ln, line)
    return {"value": int(m.group(1).replace("_", "")), "source": "%s:%d" % (path, ln)}


def check(path, ln, text):
    line = open(os.path.join(REF, path)).read().split("\n")[ln - 1]
    assert text in line, (path, ln, line)
    return "%s:%d" % (path, ln)


def main():
    if not os.path.isdir(REF):
        sys.exit("set ZK_REFERENCE to a checkout of LayerXcom/zero-chain")
    eg, mod, cs = "core/crypto/src/elgamal.rs", "modules/encrypted-balances/src/lib.rs", "src/chain_spec.rs"
    res = {
        "source": "LayerXcom/zero-chain",
        "bound": number(eg, 102, r"0\.\.([0-9_]+)"),
        "genesis": [
            dict(number(cs, 185, r"alice_value = ([0-9_]+)"), randomness="Fs::one()", randomness_source=check(cs, 189, "Fs::one()"),
                 account="alice"),
            dict(number(mod, 295, r"alice_amount = ([0-9_]+)"), randomness="Fs::one()", randomness_source=check(mod, 302, "Fs::one()"),
                 account="alice"),
        ],
        "test_amounts": {
            "enc_dec": number(eg, 203, r"amount = ([0-9]+)"),
            "enc_dec_ivk": number(eg, 223, r"alice_amount = ([0-9]+)"),
            "homomorphic_sub": [number(eg, 247 + k, r"= ([0-9]+)") for k in range(3)],
            "add_no_params": [number(eg, 273 + k, r"= ([0-9]+)") for k in range(3)],
            "read_write": number(eg, 332, r"amount = ([0-9]+)"),
        },
        "bob_seed": {
            "text": "Bob".ljust(32),
            "source": "no literal in the reference: this seed's EncryptionKey reproduces pkd_addr_bob (%s), which pins it"
                      % check(mod, 444, "45e66da531088b55dcb3b273ca825454d79d2d1d5c4fa2ba4a12c1fa1ccd6389"),
        },
        "literal_decryptions": [
            {"left": "enc10_by_alice", "right": "randomness", "key": "alice", "value": 10},
            {"left": "enc1_by_alice", "right": "randomness", "key": "alice", "value": 1},
            {"left": "enc10_by_bob", "right": "randomness", "key": "bob", "value": 10},
            {"left": "enc10_by_bob", "right": "randomness", "key": "alice", "value": None},
        ],
        "literal_decryptions_source": check(mod, 445, "enc10_by_alice") + "-448",
    }
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "elgamal.json")
    json.dump(res, open(out, "w"), indent=1)
    print("wrote", out)


if __name__ == "__main__":
    main()
