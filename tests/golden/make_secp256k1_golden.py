"""Extracts the ethrex L1 development keys into tests/golden/secp256k1_l1_keys.json.

    python tests/golden/make_secp256k1_golden.py <ethrex checkout>

Source: fixtures/keys/private_keys_l1.txt (192 private keys, one per line) and fixtures/genesis/l1.json of lambdaclass/ethrex.
Each key's address is derived here (public key with the `cryptography` package, then the oracle's keccak256) and must be in
the genesis alloc, so the JSON pairs are the genesis's own accounts.  Only this data is copied; the tests read the JSON.
"""
import json
import os
import sys

from cryptography.hazmat.primitives.asymmetric import ec

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import secp256k1_ref as ref  # noqa: E402


def main(src):
    keys = [k.strip() for k in open(os.path.join(src, "fixtures", "keys", "private_keys_l1.txt")) if k.strip()]
    alloc = {a.lower().removeprefix("0x") for a in json.load(open(os.path.join(src, "fixtures", "genesis", "l1.json")))["alloc"]}
    pairs = []
    for k in keys:
        pub = ec.derive_private_key(int(k, 16), ec.SECP256K1()).public_key().public_numbers()
        addr = ref.address((pub.x, pub.y)).hex()
        assert addr in alloc, f"{k}: derived address {addr} is not in the genesis alloc"
        pairs.append({"private_key": k.lower().removeprefix("0x"), "address": addr})
    assert len(pairs) == 192
    out = {"source": "lambdaclass/ethrex fixtures/keys/private_keys_l1.txt and fixtures/genesis/l1.json (alloc)", "keys": pairs}
    json.dump(out, open(os.path.join(HERE, "secp256k1_l1_keys.json"), "w"), indent=1)
    print("wrote", len(pairs), "keys")


if __name__ == "__main__":
    main(sys.argv[1])
