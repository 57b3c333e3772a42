"""Extracts the reference's own BLS12-381 pairing vectors into tests/golden/bls12_pairing_kats.json.

    python tests/golden/make_bls12_pairing_kats.py        (needs /root/reference; run in the build container only)

Source: /root/reference/test/tests/levm/bls12_tests.rs:10-48 -- the EIP-2537 vectors "bls_pairing_non-degeneracy"
(result 0), the same calldata with an (infinity, G2) pair appended (still 0), and "bls_pairing_e(G1,-G2)=e(-G1,G2)",
whose full calldata (G1, G2) . (G1, -G2) checks to 1.  Only the test DATA is copied (hex strings); nothing under
/root/reference is read at test time.
"""
import json
import os
import re

SRC = "/root/reference/test/tests/levm/bls12_tests.rs"
HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    src = open(SRC).read()
    hexes = re.findall(r'hex::decode\("([0-9a-f]+)"\)', src)
    assert len(hexes) == 2
    degenerate, valid = hexes
    assert len(degenerate) == 2 * 384 and len(valid) == 2 * 768
    with_infinity = degenerate + "00" * 128 + valid[2 * 128:2 * 384]  # bls12_tests.rs:31-36: G1 infinity, then valid[128..384]
    out = {"source": "lambdaclass/ethrex test/tests/levm/bls12_tests.rs:10-48 (EIP-2537 pairing_check_bls.json)",
           "vectors": [{"name": "bls_pairing_non-degeneracy", "calldata": degenerate, "expected": 0},
                       {"name": "bls_pairing_non-degeneracy_with_infinity_pair", "calldata": with_infinity, "expected": 0},
                       {"name": "bls_pairing_e(G1,-G2)=e(-G1,G2)", "calldata": valid, "expected": 1}]}
    json.dump(out, open(os.path.join(HERE, "bls12_pairing_kats.json"), "w"), indent=1)
    print("wrote", len(out["vectors"]), "vectors")


if __name__ == "__main__":
    main()
