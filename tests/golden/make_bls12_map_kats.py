"""Extracts the reference's one map-to-curve vector into tests/golden/bls12_map_kats.json.

    python tests/golden/make_bls12_map_kats.py        (needs /root/reference; run in the build container only)

Source: /root/reference/crates/vm/levm/src/precompiles.rs:44-60 -- FP2_ZERO_MAPPED_TO_G2, the padded 256-byte output of
MAP_FP2_TO_G2 (precompile 0x11) for the input (0, 0), which levm returns directly because the bls12_381 crate's
map_to_curve mishandles it.  Only the test DATA is copied (the byte list, as hex); nothing under /root/reference is read
at test time.
"""
import json
import os
import re

SRC = "/root/reference/crates/vm/levm/src/precompiles.rs"
HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    src = open(SRC).read()
    m = re.search(r"const FP2_ZERO_MAPPED_TO_G2: \[u8; 256\] = \[([^\]]*)\];", src)
    data = bytes(int(v) for v in m.group(1).replace("\n", " ").split(",") if v.strip())
    assert len(data) == 256
    out = {"source": "lambdaclass/ethrex crates/vm/levm/src/precompiles.rs:44-60 (FP2_ZERO_MAPPED_TO_G2)",
           "vectors": [{"name": "map_fp2_to_g2(0, 0)", "group": "G2", "input": "00" * 128, "expected": data.hex()}]}
    json.dump(out, open(os.path.join(HERE, "bls12_map_kats.json"), "w"), indent=1)
    print("wrote", len(out["vectors"]), "vector")


if __name__ == "__main__":
    main()
