"""MODEXP in Python: the rules of Crypto::modexp (/root/reference/crates/common/crypto/provider.rs:334-380 and its
pad_modexp_output, :705-716) with EIP-7823's 1024-byte bound as b200zk_modexp_batch reports it (include/b200zk.h), and
the item generators the GPU tests and tools/modexp_latency.py share.  Python's `pow` is exact for every input."""
import random

MAX_BYTES = 1024  # EIP-7823
OVER_BOUND = 2    # per-item status of an item with an operand over the bound

# modulus lengths in bytes at the edges of the device's size classes (8, 32, 64, 128, 256 limbs of 32 bits)
CLASS_EDGES = (1, 31, 32, 33, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024)


def modexp(base: bytes, exp: bytes, mod: bytes) -> bytes:
    """len(mod) bytes: all zero for m = 0, 1 mod m for e = 0, else (b mod m)^e mod m, big-endian and left-padded"""
    b, e, m = (int.from_bytes(x, "big") for x in (base, exp, mod))
    if m == 0:
        r = 0
    elif e == 0:
        r = 1 % m
    else:
        r = pow(b % m, e, m)
    return r.to_bytes(len(mod), "big") if mod else b""


def expected(item):
    """(output, status) the device call gives for one (base, exp, mod) item"""
    if any(len(x) > MAX_BYTES for x in item):
        return bytes(len(item[2])), OVER_BOUND
    return modexp(*item), 0


def be(x: int, n: int) -> bytes:
    return x.to_bytes(n, "big")


def rand_bytes(rng: random.Random, n: int, top: bool = True) -> bytes:
    """n random bytes; top: the first byte nonzero, so the value has exactly n significant bytes"""
    if n == 0:
        return b""
    b = bytearray(rng.randbytes(n))
    if top and b[0] == 0:
        b[0] = 1
    return bytes(b)


def rand_item(rng: random.Random, mod_len: int, base_len: int = None, exp_len: int = 32, odd: bool = None):
    """a random item with a modulus of exactly mod_len significant bytes; odd = None leaves its parity to chance"""
    m = bytearray(rand_bytes(rng, mod_len))
    if odd is not None and mod_len:
        m[-1] = (m[-1] | 1) if odd else (m[-1] & 0xfe) or 2
    base_len = mod_len if base_len is None else base_len
    return rand_bytes(rng, base_len, top=False), rand_bytes(rng, exp_len), bytes(m)


def mixed_items(rng: random.Random, n: int):
    """n items across every class: random operand lengths up to 1024 bytes with short exponents (at most 64 bytes, so a
    call stays short), odd and even moduli, leading zero bytes, and the trivial operands"""
    items = []
    for i in range(n):
        kind = i % 8
        ml = rng.choice(CLASS_EDGES) if kind < 4 else rng.randrange(1, MAX_BYTES + 1)
        bl = rng.randrange(0, MAX_BYTES + 1) if kind == 5 else ml
        base, exp, mod = rand_item(rng, ml, bl, rng.randrange(1, 65), odd=None)
        if kind == 6:
            mod = bytes(rng.randrange(0, 8)) + mod  # leading zeros: a longer output, the same class
        if kind == 7:
            exp = bytes(rng.randrange(0, 4)) + exp[:rng.randrange(0, 3)]  # e = 0 or tiny, maybe zero-padded
        items.append((base, exp, mod))
    return items


def rsa_items(rng: random.Random, bits: int, n: int):
    """n RSA signatures s over random digests with e = 65537 (made by the `cryptography` package): the items
    (s, 65537, N) and the values s^e mod N should give (the PKCS #1 v1.5 encoded digests)"""
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import padding, rsa, utils
    key = rsa.generate_private_key(public_exponent=65537, key_size=bits)
    nn = key.public_key().public_numbers().n
    k = bits // 8
    items, want = [], []
    for _ in range(n):
        digest = rng.randbytes(32)
        sig = key.sign(digest, padding.PKCS1v15(), utils.Prehashed(hashes.SHA256()))
        items.append((sig, be(65537, 3), be(nn, k)))
        want.append(pow(int.from_bytes(sig, "big"), 65537, nn).to_bytes(k, "big"))
    return items, want
