#!/usr/bin/env python3
"""Generates tests/golden/jubjub_points.json: the Jubjub point encodings the reference's own sources hold as literals.

Run with ZK_REFERENCE pointing at a checkout of the reference; the tests never read the reference itself.  Only the hex /
decimal literals are extracted, each with the file and line it comes from:
  - modules/encrypted-balances/src/lib.rs:407, 443-450   g_epoch and the public-input points of a confidential transfer
  - core/jubjub/src/curve/mod.rs:424-444                  the two Point::read vectors of test_jubjub_bls12 (same y, both
                                                          signs) and the y they must decode to (decimal, line 428)
tests/test_oracle_jubjub.py and tests/test_gpu_jubjub.py give each entry its meaning."""
import json
import os
import re
import sys

REF = os.environ.get("ZK_REFERENCE", "")
EB = "modules/encrypted-balances/src/lib.rs"
MOD = "core/jubjub/src/curve/mod.rs"


def lines(path):
    return open(os.path.join(REF, path)).read().split("\n")


def hex32(line):
    m = re.findall(r'hex!\("([0-9a-f]{64})"\)', line)
    assert len(m) == 1, line
    return m[0]


def main():
    if not os.path.isdir(REF):
        sys.exit("set ZK_REFERENCE to a checkout of LayerXcom/zero-chain")
    src = lines(EB)
    tx = []
    for ln in [407] + list(range(443, 451)):
        m = re.search(r"let (\w+): \[u8; 32\]", src[ln - 1])
        assert m, ln
        tx.append({"name": m.group(1), "hex": hex32(src[ln - 1]), "source": "%s:%d" % (EB, ln)})
    src = lines(MOD)
    reads = []
    for ln in range(424, 445):
        if "hex!(" in src[ln - 1]:
            reads.append({"hex": hex32(src[ln - 1]), "source": "%s:%d" % (MOD, ln)})
    assert len(reads) == 2
    m = re.search(r'Fr::from_str\("(\d+)"\)', src[427])
    assert m
    res = {"source": "LayerXcom/zero-chain", "transaction_points": tx, "read_vectors": reads,
           "read_vectors_y": {"decimal": m.group(1), "source": "%s:428" % MOD}}
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "jubjub_points.json")
    json.dump(res, open(out, "w"), indent=1)
    print("wrote", out, len(tx), "transaction points,", len(reads), "read vectors")


if __name__ == "__main__":
    main()
