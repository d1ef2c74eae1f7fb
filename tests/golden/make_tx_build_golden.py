#!/usr/bin/env python3
"""Generates tests/golden/tx_build.json: the literals that building a confidential transfer must reproduce, each with the
file and line it comes from.

Run with ZK_REFERENCE pointing at a checkout of the reference; the tests never read the reference itself.
  modules/encrypted-balances/src/lib.rs:324   the Alice seed
  modules/encrypted-balances/src/lib.rs:443   pkd_addr_alice = EncryptionKey::from_seed(Alice seed)
  modules/encrypted-balances/src/lib.rs:407   the g_epoch "of block height one" = GEpoch::group_hash(0)
  modules/encrypted-balances/src/lib.rs:450   the nonce = Alice's dk * GEpoch::group_hash(0)
  modules/encrypted-balances/src/lib.rs:445, 448  enc10_by_alice | randomness: a ciphertext of 10 under Alice's key
GEpoch::group_hash(1) has no literal in the reference; its value comes from the Python oracle and is marked so, and
tests/test_oracle_tx_build.py checks it against the C oracle, an independent restatement.
tests/test_oracle_tx_build.py and tests/test_gpu_tx_build.py give each entry its meaning."""
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = os.environ.get("ZK_REFERENCE", "")


def literal(path, ln, pattern):
    line = open(os.path.join(REF, path)).read().split("\n")[ln - 1]
    m = re.search(pattern, line)
    assert m, (path, ln, line)
    return {"value": m.group(1), "source": "%s:%d" % (path, ln)}


def main():
    if not os.path.isdir(REF):
        sys.exit("set ZK_REFERENCE to a checkout of LayerXcom/zero-chain")
    from tests.jubjub_oracle import tx_build as tb
    lib = "modules/encrypted-balances/src/lib.rs"
    hex32 = lambda name: r'%s: \[u8; 32\] = hex!\("([0-9a-f]{64})"\)' % name
    seed = literal(lib, 324, r'alice_seed = b"(Alice +)"')
    res = {
        "source": "LayerXcom/zero-chain",
        "alice_seed": seed["value"],
        "alice_seed_source": seed["source"],
        "alice_encryption_key": literal(lib, 443, hex32("pkd_addr_alice")),
        "g_epoch_0": literal(lib, 407, hex32("g_epoch_vec")),
        "g_epoch_1": {"value": tb.g_epoch(1)[0].hex(), "source": "the Python oracle (no literal in the reference)"},
        "alice_nonce": literal(lib, 450, hex32("nonce")),
        "enc10_by_alice": literal(lib, 445, hex32("enc10_by_alice")),
        "randomness": literal(lib, 448, hex32("randomness")),
    }
    assert len(res["alice_seed"]) == 32
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tx_build.json")
    with open(out, "w") as f:
        json.dump(res, f, indent=1)
        f.write("\n")
    print("wrote", out)


if __name__ == "__main__":
    main()
