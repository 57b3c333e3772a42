"""CPU checks of the Groth16 batch verification's statement (tests/groth16_batch_ref.py): the combined equation of
b200zk_groth16_verify_batch over the oracle's pairing, its Fiat-Shamir coefficients, and why they must be random."""
import groth16_batch_ref as g
import pyref as o

R, P = g.R, g.P


def _batch(key, n):
    items = [key.proof(with_logs=True) for _ in range(n)]
    return [p for p, _, _ in items], [x for _, x, _ in items], [lg for _, _, lg in items]


def _tampers(key, proofs, xs):
    """(name, proofs, public inputs) with proof 1 of 3 made bad, each well-formed unless the name says otherwise"""
    other = g.SimKey(key.n_pub, seed=99)
    foreign, fx = other.proof()
    p1 = proofs[1]
    out = [("wrong input", proofs, [xs[0], [(xs[1][0] + 1) % R] + xs[1][1:], xs[2]]),
           ("A from proof 0", [proofs[0], proofs[0][:64] + p1[64:], proofs[2]], xs),
           ("B from proof 0", [proofs[0], p1[:64] + proofs[0][64:192] + p1[192:], proofs[2]], xs),
           ("C from proof 0", [proofs[0], p1[:192] + proofs[0][192:], proofs[2]], xs),
           ("A = identity", [proofs[0], bytes(64) + p1[64:], proofs[2]], xs),
           ("another key", [proofs[0], foreign, proofs[2]], [xs[0], fx, xs[2]])]
    return out


def test_valid_batches_pass_the_combined_check():
    for n_pub in (0, 1, 3):
        key = g.SimKey(n_pub, seed=n_pub + 5)
        proofs, xs, logs = _batch(key, 3)
        assert g.combined_check(key.vk, proofs, xs)
        assert g.combined_exponent(key, logs, xs, g.batch_rhos(key.vk, proofs, xs)) == 0
        assert all(g.single_check(key.vk, p, x) for p, x in zip(proofs, xs))


def test_each_tamper_fails_the_combined_check_and_agrees_with_the_per_proof_check():
    key = g.SimKey(2, seed=7)
    proofs, xs, _ = _batch(key, 3)
    for name, ps, x in _tampers(key, proofs, xs):
        per_proof = [g.single_check(key.vk, p, xx) for p, xx in zip(ps, x)]
        assert per_proof == [True, False, True], name
        assert not g.combined_check(key.vk, ps, x), name


def test_malformed_proofs_are_left_out_of_the_combined_check():
    key = g.SimKey(1, seed=8)
    proofs, xs, _ = _batch(key, 2)
    a = proofs[1]
    p_coord = P.to_bytes(32, "big")
    off_curve = (1).to_bytes(32, "big") + (3).to_bytes(32, "big")
    cases = [(a[:32] + p_coord + a[64:], xs[1], 2),                 # a coordinate = p
             (a, [R], 2),                                           # a public input = r
             (off_curve + a[64:], xs[1], 3),                        # A off the curve
             (a[:192] + off_curve, xs[1], 3)]                       # C off the curve
    for bad, bx, status in cases:
        assert g.proof_status(bad, bx) == status
        assert g.combined_check(key.vk, [proofs[0], bad], [xs[0], bx])
        assert not g.single_check(key.vk, bad, bx)


def test_cancelling_tamper_passes_all_ones_but_not_the_derived_coefficients():
    key = g.SimKey(1, seed=9)
    items = [key.proof(with_logs=True) for _ in range(3)]
    xs = [x for _, x, _ in items]
    d = 123456789
    logs = [lg for _, _, lg in items]
    logs[0] = (logs[0][0], logs[0][1], (logs[0][2] + d) % R)
    logs[1] = (logs[1][0], logs[1][1], (logs[1][2] - d) % R)
    proofs = [p[:192] + g.g1(c) for (p, _, _), (_, _, c) in zip(items, logs)]
    assert not g.single_check(key.vk, proofs[0], xs[0]) and not g.single_check(key.vk, proofs[1], xs[1])
    ones = [1, 1, 1]
    assert g.combined_exponent(key, logs, xs, ones) == 0
    assert g.combined_check(key.vk, proofs, xs, ones)
    rhos = g.batch_rhos(key.vk, proofs, xs)
    assert g.combined_exponent(key, logs, xs, rhos) != 0
    assert not g.combined_check(key.vk, proofs, xs, rhos)


def test_coefficients_are_128_bit_nonzero_distinct_and_bind_every_byte():
    key = g.SimKey(2, seed=10)
    proofs, xs, _ = _batch(key, 4)
    rhos = g.batch_rhos(key.vk, proofs, xs)
    assert all(0 < r < 1 << 128 for r in rhos) and len(set(rhos)) == len(rhos)
    assert max(rhos).bit_length() > 120
    flips = []
    for k in range(0, len(key.vk), 97):
        vk = bytearray(key.vk)
        vk[k] ^= 1
        flips.append((bytes(vk), proofs, xs))
    for k in range(0, 256, 31):
        ps = list(proofs)
        ps[2] = ps[2][:k] + bytes([ps[2][k] ^ 0x80]) + ps[2][k + 1:]
        flips.append((key.vk, ps, xs))
    flips.append((key.vk, proofs, [xs[0], xs[1], [xs[2][0] ^ 1, xs[2][1]], xs[3]]))
    flips.append((key.vk, proofs[:3], xs[:3]))
    for vk, ps, x in flips:
        new = g.batch_rhos(vk, ps, x)
        assert all(a != b for a, b in zip(new, rhos))
