"""PLONK from circom artifacts on the device (b200zk_plonk_zkey_*, ethrex_b200.zkey.PlonkProver): snarkjs-0.7-layout files
of tests/plonk_ref.py proved bit-exactly against the Python prover (snarkjs's own root-domain route), verified by
PlonkVerifier on the device and by the Python verifier, then every refusal, each followed by a good proof."""
import pytest

import plonk_ref as pr
import zkey_ref as zr

from ethrex_b200 import _ffi as F
from ethrex_b200.errors import B200Error
from ethrex_b200.zkey import PlonkProver, PlonkVerifier, ZkeyProver

pytestmark = pytest.mark.gpu

R = pr.R
BLINDINGS = {"zero": [0] * 11, "random": [(0x5DEECE66D * (k + 7) ** 9) % R for k in range(11)], "order_minus_1": [R - 1] * 11}
# (n_gates, n_public, n_additions, log_n)
SHAPES = [(5, 1, 2, 3), (21, 0, 6, 5), (100, 3, 30, 7), (700, 2, 150, 10)]
_CIRCUITS = {}


def _circuit(shape):
    if shape not in _CIRCUITS:
        g, npub, na, log_n = shape
        c = pr.PlonkCircuit(n_gates=g, n_public=npub, n_private=4, n_additions=na, seed=0x9100 + g, log_n=log_n)
        _CIRCUITS[shape] = (c, c.zkey())
    return _CIRCUITS[shape]


def _witness(c):
    return c.assign([0x1234567 + 11 * i for i in range(c.n_public)])


@pytest.mark.parametrize("case", sorted(BLINDINGS))
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("precompute", [False, True])
def test_proof_equals_the_oracle(ctx, shape, case, precompute):
    c, zkey = _circuit(shape)
    prover = PlonkProver(ctx, zkey, precompute=precompute)
    try:
        assert (prover.n_vars, prover.n_public, prover.log_n) == (c.n_vars, c.n_public, c.log_n)
        assert prover.vk() == c.vk()
        wt = _witness(c)
        want, _ = c.prove(wt, BLINDINGS[case])
        assert prover.prove(c.wtns(wt), BLINDINGS[case]) == want
    finally:
        prover.close()


@pytest.mark.parametrize("shape", SHAPES)
def test_proofs_verify_and_tampering_fails(ctx, shape):
    c, zkey = _circuit(shape)
    prover = PlonkProver(ctx, zkey)
    try:
        ver = prover.verifier()
        wt = _witness(c)
        pub = c.public(wt)
        proof = prover.prove(c.wtns(wt))  # random blinding
        assert ver.verify(proof, pub)
        assert c.verify(proof, pub, tau=c.tau)
        if shape == SHAPES[0]:
            assert c.verify(proof, pub)  # the Python pairing
        bad = proof[:64 * 3] + pr._g1(77) + proof[64 * 4:]
        assert not ver.verify(bad, pub) and not c.verify(bad, pub, tau=c.tau)
        bad = proof[:700] + bytes([proof[700] ^ 1]) + proof[701:]
        assert not ver.verify(bad, pub)
        if pub:
            assert not ver.verify(proof, [(pub[0] + 1) % R] + pub[1:])
        # two proves of the same inputs are the same bytes
        b = BLINDINGS["random"]
        assert prover.prove(c.wtns(wt), b) == prover.prove(c.wtns(wt), b)
    finally:
        prover.close()


def _refused(ctx, fn, status, fragment):
    with pytest.raises(B200Error) as ei:
        fn()
    assert ei.value.status == status and fragment in str(ei.value), (ei.value.status, str(ei.value))


def test_refusals_each_followed_by_a_good_proof(ctx):
    c, zkey = _circuit(SHAPES[2])
    prover = PlonkProver(ctx, zkey)
    wt = _witness(c)
    good, _ = c.prove(wt, BLINDINGS["random"])
    blinding = BLINDINGS["random"]

    def ok():
        assert prover.prove(c.wtns(wt), blinding) == good
    try:
        ok()
        _refused(ctx, lambda: prover.prove(c.wtns(wt[:-1]), blinding), F.ERR_INVALID_ARG, "nWitness")
        ok()
        big = list(wt)
        big[5] = R + 3
        _refused(ctx, lambda: prover.prove(c.wtns(big), blinding), F.ERR_NOT_IN_FIELD, "value 5 is >= r")
        ok()
        # one copy constraint broken: a key whose C map sends one gate row to another signal than its sigma cycles
        # assume (a witness alone cannot do it: every place of a signal reads the same value)
        secs = dict(c.sections())
        row = c.n_public + 1
        other = next(s for s in range(c.n_wtns) if wt[s] != c.full(wt)[c.map_c[row]])
        bad_map = secs[6][:4 * row] + other.to_bytes(4, "little") + secs[6][4 * row + 4:]
        bad_key = PlonkProver(ctx, zr.container(b"zkey", 1, [(k, bad_map if k == 6 else v) for k, v in c.sections()]), precompute=False)
        try:
            _refused(ctx, lambda: bad_key.prove(c.wtns(wt), blinding), F.ERR_INVALID_ARG, "copy constraints")
        finally:
            bad_key.close()
        ok()
        used = {s for m in (c.map_a, c.map_b) for s in m[c.n_public:]}
        outs = [1 + c.n_public + 4 + j for j in range(len(c.gates))]
        lone = next(s for s in outs if s not in used and all(a[0] != s and a[1] != s for a in c.adds))
        broken = list(wt)
        broken[lone] = (broken[lone] + 1) % R
        _refused(ctx, lambda: prover.prove(c.wtns(broken), blinding), F.ERR_INVALID_ARG, "gates")
        ok()
        _refused(ctx, lambda: prover.prove(c.wtns(wt), blinding[:4] + [R] + blinding[5:]), F.ERR_NOT_IN_FIELD, "b5 is >= r")
        ok()
        ctx.set_ntt_root(ctx.ntt_root_preset(ctx.NTT_ROOT_HALO2))
        try:
            _refused(ctx, lambda: prover.prove(c.wtns(wt), blinding), F.ERR_INVALID_ARG, "preset 0")
        finally:
            ctx.set_ntt_root(None)
        ok()
        key = prover.key
        for fn in (lambda: F.lib.b200zk_plonk_zkey_free(ctx._h, key + 1000), lambda: F.lib.b200zk_plonk_zkey_info(ctx._h, 0, None, None, None, None, 0)):
            assert fn() == F.ERR_INVALID_ARG
        ok()
        # a Groth16 key is not a PLONK key, and the reverse
        g16 = ZkeyProver(ctx, zr.ZkeyCircuit(11, 2, seed=3).zkey(), precompute=False)
        try:
            assert F.lib.b200zk_plonk_zkey_info(ctx._h, g16.key, None, None, None, None, 0) == F.ERR_INVALID_ARG
            assert F.lib.b200zk_groth16_zkey_info(ctx._h, prover.key, None, None, None, None, 0) == F.ERR_INVALID_ARG
            pg = PlonkProver.__new__(PlonkProver)
            pg.ctx, pg.key = ctx, g16.key
            _refused(ctx, lambda: pg.prove(c.wtns(wt), blinding), F.ERR_INVALID_ARG, "unknown key")
        finally:
            g16.close()
        ok()
        # a PLONK key is refused by the Groth16 loader, and the reverse
        _refused(ctx, lambda: ZkeyProver(ctx, zkey), F.ERR_UNSUPPORTED, "not Groth16")
        _refused(ctx, lambda: PlonkProver(ctx, zr.ZkeyCircuit(11, 2, seed=3).zkey()), F.ERR_UNSUPPORTED, "not PLONK")
        ok()
    finally:
        prover.close()


def test_device_verifier_matches_python_on_oracle_proofs(ctx):
    c, zkey = _circuit(SHAPES[1])
    wt = _witness(c)
    proof, _ = c.prove(wt, BLINDINGS["random"])
    ver = PlonkVerifier(ctx, c.vk(), c.n_public, c.log_n)
    assert ver.verify(proof, c.public(wt))
    assert not ver.verify(proof[:576] + proof[608:640] + proof[576:608] + proof[640:], c.public(wt))


# ---- at circuit sizes: 2^16 (the scans' carry CTA walks several chunks per thread, several evaluation blocks, more
# public inputs than plonk_eval_finish has threads), 2^20, and 2^21 (the scans' chunks grow past 32 values, and the Z
# scan has more chunks than the openings' scans).  The key's polynomial sections come from the C++ oracle's
# NTTs and PTau from the device's batched scalar multiplication; the Python prover is too slow here, so the proofs are
# checked by both verifiers (the device's PlonkVerifier and the Python one with the trapdoor) and tampering must fail.
@pytest.mark.parametrize("log_n,n_public", [(16, 300), (20, 2), (21, 2)])
def test_large_domains_verify_and_tampering_fails(ctx, log_n, n_public):
    n = 1 << log_n
    c = pr.PlonkCircuit(n_gates=n - n // 8 - n_public, n_public=n_public, n_private=64, n_additions=n // 16, seed=log_n, log_n=log_n)
    prover = PlonkProver(ctx, c.zkey(ctx), precompute=True)
    try:
        assert (prover.log_n, prover.n_public) == (log_n, n_public)
        wt = _witness(c)
        pub = c.public(wt)
        proof = prover.prove(c.wtns(wt))
        ver = prover.verifier()
        assert ver.verify(proof, pub)
        assert pr.plonk_verify(prover.vk(), n_public, log_n, proof, pub, tau=c.tau)
        for bad in (proof[:64 * 7] + pr._g1(5) + proof[64 * 8:], proof[:600] + bytes([proof[600] ^ 4]) + proof[601:]):
            assert not ver.verify(bad, pub)
            assert not pr.plonk_verify(prover.vk(), n_public, log_n, bad, pub, tau=c.tau)
        assert not ver.verify(proof, [(pub[0] + 1) % R] + pub[1:])
    finally:
        prover.close()
