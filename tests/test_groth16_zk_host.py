"""CPU tests of the zero-knowledge Groth16 prove: the blinded expected proof the GPU tests compare against verifies
under the pairing the reference's KATs pin, the blinding sampler is uniform below r by rejection, and the ctypes twin
of struct b200zk_groth16_zk has the header's size."""
import ctypes

import pyref as o
from groth16_toy import ToyGroth16
from groth16_toy_zk import expected_zk_proof


def test_blinded_toy_proof_satisfies_the_verification_equation():
    """e(-A, B) e(alpha, beta) e(IC(x), gamma) e(C, delta) == 1 under pyref's pairing (the one
    tests/test_oracle.py replays the reference's 14 ecpairing vectors on), for blinded proofs; a proof with
    C from a different s does not verify."""
    toy = ToyGroth16(3)
    x = 0x1234567
    z = toy.assign(x)

    def pairs(proof):
        cd = toy.verifier_calldata(proof, x)
        return [(o.g1_from_be(cd[i:i + 64]), o.g2_from_be(cd[i + 64:i + 192])) for i in range(0, len(cd), 192)]

    r, s = 0x1F2E3D4C5B6A79881726354453627180, o.R - 1
    proof = expected_zk_proof(toy, z, r, s)
    assert o.pairing_check(pairs(proof))
    wrong_c = proof[:192] + expected_zk_proof(toy, z, r, s - 1)[192:]
    assert not o.pairing_check(pairs(wrong_c))


def test_rejection_sampler_stays_below_r():
    """random_scalar draws 254 bits and retries while the value is >= r: fed values at and above r first, it skips
    them and returns the first one below r, unchanged (no reduction)."""
    from ethrex_b200.groth16 import R_MOD, random_scalar
    draws = iter([R_MOD, (1 << 254) - 1, R_MOD + 5, R_MOD - 1])
    seen = []

    def bits(k):
        assert k == 254
        v = next(draws)
        seen.append(v)
        return v

    assert random_scalar(bits) == R_MOD - 1
    assert len(seen) == 4
    draws = iter([0])
    assert random_scalar(lambda k: next(draws)) == 0
    assert all(0 <= random_scalar() < R_MOD for _ in range(2000))


def test_zk_assembly_kernel_does_not_spill():
    """groth16_assemble_zk holds G2 formulas in one thread: ptxas must fit it in registers (the build keeps the
    `-Xptxas -v` report of every translation unit)."""
    import os
    import re
    import pytest
    log = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ethrex_b200", "csrc", "build", "msm.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("msm.ptxas.log not built")
    txt = open(log).read()
    m = re.search(r"Function properties for \w*groth16_assemble_zk\w*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", txt)
    assert m, "no ptxas report for groth16_assemble_zk"
    assert m.group(2) == "0" and m.group(3) == "0", m.group(0)


def test_zk_struct_layout():
    from ethrex_b200 import _ffi
    assert ctypes.sizeof(_ffi.Groth16Zk) == 80
    assert _ffi.Groth16Zk.r.offset == 16 and _ffi.Groth16Zk.s.offset == 48
