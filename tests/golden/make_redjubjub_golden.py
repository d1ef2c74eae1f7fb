#!/usr/bin/env python3
"""Generates tests/golden/redjubjub.json: the byte-string literals RedJubjub verification and the Alice key derivation
depend on, each with the file and line it comes from.

Run with ZK_REFERENCE pointing at a checkout of the reference; the tests never read the reference itself.
  core/jubjub/src/constants.rs:6              GH_FIRST_BLOCK (BLAKE2s prefix of group_hash)
  core/jubjub/src/constants.rs:20             "Zcash_PH" (find_group_hash personalization of the Diversifier generator)
  core/jubjub/src/redjubjub.rs:25             "Zcash_RedJubjubH" (H*)
  core/keys/src/lib.rs:40-41                  "zech_ExpandSeed_" (SpendingKey::from_seed), "zech_bdk" (into_decryption_key)
  modules/encrypted-balances/src/lib.rs:382   the Alice seed, whose EncryptionKey is pkd_addr_alice in jubjub_points.json
  core/jubjub/src/redjubjub.rs:321-322        the messages of the reference's random_signatures test
tests/test_oracle_redjubjub.py and tests/test_gpu_redjubjub.py give each entry its meaning."""
import json
import os
import re
import sys

REF = os.environ.get("ZK_REFERENCE", "")


def literal(path, ln, pattern):
    line = open(os.path.join(REF, path)).read().split("\n")[ln - 1]
    m = re.search(pattern, line)
    assert m, (path, ln, line)
    return {"text": m.group(1), "source": "%s:%d" % (path, ln)}


def main():
    if not os.path.isdir(REF):
        sys.exit("set ZK_REFERENCE to a checkout of LayerXcom/zero-chain")
    c, rj, keys = "core/jubjub/src/constants.rs", "core/jubjub/src/redjubjub.rs", "core/keys/src/lib.rs"
    res = {
        "source": "LayerXcom/zero-chain",
        "gh_first_block": literal(c, 6, r'b"([0-9a-f]{64})"'),
        "personalizations": {
            "pedersen_hash_generators": literal(c, 20, r'b"(Zcash_PH)"'),
            "h_star": literal(rj, 25, r'b"(Zcash_RedJubjubH)"'),
            "prf_expand": literal(keys, 40, r'b"(zech_ExpandSeed_)"'),
            "crh_bdk": literal(keys, 41, r'b"(zech_bdk)"'),
        },
        "alice_seed": literal("modules/encrypted-balances/src/lib.rs", 382, r'b"(Alice *)"'),
        "messages": [literal(rj, 321, r'b"(Foo bar)"'), literal(rj, 322, r'b"(Spam eggs)"')],
    }
    assert len(res["alice_seed"]["text"]) == 32
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "redjubjub.json")
    json.dump(res, open(out, "w"), indent=1)
    print("wrote", out)


if __name__ == "__main__":
    main()
