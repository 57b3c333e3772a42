"""CPU checks of the EIP-2537 map-to-curve oracle (tests/bls12_map_ref.py) the device tests compare against: the
reference's FP2_ZERO_MAPPED_TO_G2, the constant checks of tests/golden/make_bls12_map_constants.py and the tables
bls_map.cu embeds, the psi form of G2's cofactor clearing against h_eff, the group properties of every output, SSWU's
exceptional inputs, and the ptxas report of the new kernels."""
import json
import os
import random
import re
import sys

import pytest

import bls12_map_ref as M
import bls_pairing_ref as B
import bls_ref as bls

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "ethrex_b200", "csrc")
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_bls12_map_constants as K  # noqa: E402

P = M.P
KAT = json.load(open(os.path.join(HERE, "golden", "bls12_map_kats.json")))["vectors"][0]


def g1_exceptional():
    """u with Z^2 u^4 + Z u^2 = 0: u = 0 and u = +-sqrt(-1/Z)"""
    r = M.Fp.sqrt(-pow(M.G1_Z, -1, P) % P)
    assert r is not None
    return [0, r, P - r]


def g2_exceptional():
    r = M.Fp2.sqrt(B.f2_neg(B.f2_inv(M.G2_Z)))
    return [(0, 0)] + ([] if r is None else [r, B.f2_neg(r)])


def test_zero_fp2_gives_the_reference_vector():
    assert M.map_fp2_to_g2_bytes(bytes.fromhex(KAT["input"])) == (bytes.fromhex(KAT["expected"]), 0)


def test_g1_constants_checked_against_the_curves():
    K.check_g1_point_count(n=2)
    K.check_g1_iso_on_curve()
    K.check_g1_iso_additive()
    assert K.find_z_sswu_g1() == 11


def test_g2_isogeny_rederived_from_the_vector():
    K.check_g2_against_vector()


def test_cu_tables_equal_the_generator():
    src = open(os.path.join(CSRC, "bls_map.cu")).read()
    for name, vals in K.tables().items():
        m = re.search(r"__constant__ uint32_t " + name + r"\[[^=]*= \{(.*?)\n\};", src, re.S)
        assert m, name
        got = [int(h, 16) for h in re.findall(r"0x([0-9a-f]{8})u", m.group(1))]
        assert got == K.table_limbs(vals), name


def test_psi_cofactor_clearing_equals_h_eff():
    for seed in range(3):
        q = B.g2_random_point(0x9380 + seed)
        assert B.g2_on_curve(q) and not B.g2_in_subgroup(q)
        assert M.clear_cofactor_g2_psi(q) == M.clear_cofactor_g2_scalar(q)


def _g1_ok(pt):
    return pt is not None and bls.on_curve(pt) and B.g1_in_subgroup(pt)


def _g2_ok(pt):
    return pt is not None and B.g2_on_curve(pt) and B.g2_in_subgroup(pt)


def test_outputs_are_subgroup_points_and_odd():
    rng = random.Random(9380)
    for u in [1, P - 1, 2, 11] + [rng.randrange(P) for _ in range(3)]:
        pt = M.map_to_g1(u)
        assert _g1_ok(pt), u
        assert M.map_to_g1(P - u) == (pt[0], -pt[1] % P), u
    for u in [(1, 0), (0, 1), (P - 1, 5), (5, P - 1)] + [(rng.randrange(P), rng.randrange(P)) for _ in range(2)]:
        pt = M.map_to_g2(u)
        assert _g2_ok(pt), u
        assert M.map_to_g2(B.f2_neg(u)) == B.g2_neg(pt), u


def test_exceptional_inputs_give_valid_points():
    for u in g1_exceptional():
        assert _g1_ok(M.map_to_g1(u)), u
    ex = g2_exceptional()
    assert len(ex) in (1, 3)
    for u in ex:
        assert _g2_ok(M.map_to_g2(u)), u


def test_byte_interface_statuses():
    good = M.fp64(5)
    assert M.map_fp_to_g1_bytes(good)[1] == 0
    for bad in (bytes([1]) + good[1:], good[:15] + bytes([1]) + good[16:], M.fp64(P), bytes(16) + b"\xff" * 48):
        assert M.map_fp_to_g1_bytes(bad) == (bytes(128), 2)
        assert M.map_fp2_to_g2_bytes(good + bad) == (bytes(256), 2)
        assert M.map_fp2_to_g2_bytes(bad + good) == (bytes(256), 2)


@pytest.mark.parametrize("field", ["FeBigINS_8Fp381Cfg", "Fp2_381"])
def test_ptxas_lists_the_new_kernels(field):
    log = os.path.join(CSRC, "build", "bls_map.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("bls_map.ptxas.log not built")
    m = re.search(r"Function properties for \w*bls_mapINS_\d+" + field + r"\w*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\nptxas info\s*: Used (\d+) registers", open(log).read())
    assert m, f"no ptxas report for bls_map<{field}>"
