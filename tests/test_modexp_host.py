"""CPU tests of the MODEXP reference (tests/modexp_ref.py): the two EIP-198 examples and each rule of Crypto::modexp
that b200zk_modexp_batch reproduces."""
import random

import modexp_ref as ref
import secp256k1_ref as k1


def test_eip198_fermat_example():
    """3^(p-1) mod p = 1 for the secp256k1 prime, the first example of EIP-198"""
    out = ref.modexp(ref.be(3, 1), ref.be(k1.P - 1, 32), ref.be(k1.P, 32))
    assert out == ref.be(1, 32)


def test_eip198_empty_base_example():
    """a 0-length base over a 32-byte modulus gives 32 zero bytes, the second example of EIP-198"""
    assert ref.modexp(b"", ref.be(k1.P - 1, 32), ref.be(k1.P, 32)) == bytes(32)


def test_zero_modulus_is_all_zero_bytes():
    assert ref.modexp(b"\x05", b"\x03", bytes(7)) == bytes(7)
    assert ref.modexp(b"\x05", b"", bytes(3)) == bytes(3)  # m = 0 outranks e = 0
    assert ref.modexp(b"\x05", b"\x03", b"") == b""


def test_zero_exponent_is_one_mod_m():
    assert ref.modexp(b"\x07", b"", b"\x05") == b"\x01"
    assert ref.modexp(b"", bytes(4), b"\x00\x09") == b"\x00\x01"  # 0^0 = 1, zero-padded exponent
    assert ref.modexp(b"\x07", b"\x00", b"\x01") == b"\x00"         # 1 mod 1 = 0
    assert ref.modexp(b"\x07", b"", bytes(5) + b"\x01") == bytes(6)


def test_base_is_reduced_first_and_output_is_padded():
    assert ref.modexp(ref.be(1000, 2), b"\x01", b"\x07") == ref.be(1000 % 7, 1)
    assert ref.modexp(b"\x02", b"\x0a", bytes(3) + b"\x03\xe8") == ref.be(1024 % 1000, 5)
    # leading zeros of any operand change nothing but the output length
    assert ref.modexp(bytes(9) + b"\x03", bytes(2) + b"\x05", bytes(4) + b"\x65") == bytes(4) + ref.be(pow(3, 5, 101), 1)


def test_bound_is_on_the_declared_length():
    ok = (bytes(1024), b"\x01", b"\x07")
    assert ref.expected(ok) == (b"\x00", 0)
    for j in range(3):
        item = list(ok)
        item[j] = bytes(1025) if j != 2 else bytes(1024) + b"\x07"
        out, st = ref.expected(tuple(item))
        assert st == ref.OVER_BOUND and out == bytes(len(item[2]))


def test_generators_cover_what_they_promise():
    rng = random.Random(1)
    for ml in ref.CLASS_EDGES:
        b, e, m = ref.rand_item(rng, ml, odd=False)
        assert len(m) == ml and m[0] != 0 and m[-1] % 2 == 0 and len(e) == 32
    items = ref.mixed_items(rng, 256)
    assert all(max(len(x) for x in it) <= ref.MAX_BYTES for it in items)
    assert any(int.from_bytes(e, "big") == 0 for _, e, _ in items)
    assert any(m[0] == 0 for _, _, m in items)
