"""CPU checks of the EIP-2537 addition and MSM oracle (tests/bls12_ops_ref.py) the device tests compare against: addition
and MSM against closed forms on chain bases P_i = (a + i d) G, the scalar edge cases, the off-subgroup points the device
tests use, the EIP-2537 encodings, and the ptxas report of the new kernels."""
import os
import re

import pytest

import bls12_ops_ref as ops

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "ethrex_b200", "csrc")
P, R = ops.P, ops.R
GROUPS = [ops.G1, ops.G2]


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.name)
def test_add_closed_forms(g):
    a, b = 0x1234567890ABCDEF1234, R - 5
    pa, pb = g.mul(a, g.gen), g.mul(b, g.gen)
    assert g.on_curve(pa) and g.on_curve(pb)
    assert g.add(pa, pb) == g.mul((a + b) % R, g.gen)
    assert g.add(pa, pa) == g.mul(2 * a, g.gen)
    assert g.add(pa, g.neg(pa)) is None
    assert g.add(None, pa) == pa and g.add(pa, None) == pa and g.add(None, None) is None
    assert g.mul(R, g.gen) is None and g.in_subgroup(g.gen)


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.name)
def test_msm_chain_closed_form(g):
    a, d = 0xA11CE, 0xB0B
    ks = [0, 1, R - 1, R, R + 1, (1 << 256) - 1, 7, 0xDEADBEEF << 200]
    bases = g.chain(len(ks), a, d)
    assert all(g.on_curve(p) for p in bases)
    assert bases[3] == g.mul(a + 3 * d, g.gen)
    assert g.msm(list(zip(bases, ks))) == g.chain_msm(ks, a, d)
    assert g.msm([(bases[0], k) for k in (R - 1, 1)]) is None  # terms that cancel
    assert g.msm([]) is None


def test_off_subgroup_points():
    p0 = ops.G1_OFF_SUBGROUP
    assert ops.G1.on_curve(p0) and not ops.G1.in_subgroup(p0)
    assert ops.G1.mul(3, p0) is None  # order 3
    for g in GROUPS:
        q = g.random_point(2537)
        assert g.on_curve(q) and not g.in_subgroup(q)
        # the group law holds outside the subgroup: (q + q) + q = 3 q by double-and-add
        assert g.add(g.add(q, q), q) == g.mul(3, q)


@pytest.mark.parametrize("g", GROUPS, ids=lambda g: g.name)
def test_eip2537_encoding(g):
    q = g.mul(0xC0FFEE, g.gen)
    enc = g.encode(q)
    assert len(enc) == g.size and all(enc[i:i + 16] == bytes(16) for i in range(0, g.size, 64))
    assert g.encode(None) == bytes(g.size)
    data = g.calldata([(q, 5), (None, (1 << 256) - 1)])
    assert len(data) == 2 * g.pair and data[g.pair - 32:g.pair] == (5).to_bytes(32, "big")


@pytest.mark.parametrize("field", ["FeBigINS_8Fp381Cfg", "Fp2_381"])
@pytest.mark.parametrize("kernel", ["bls_add", "bls_msm_terms", "bls_msm_fold"])
def test_ptxas_lists_the_new_kernels(kernel, field):
    log = os.path.join(CSRC, "build", "bls_ops.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("bls_ops.ptxas.log not built")
    m = re.search(r"Function properties for \w*" + kernel + r"INS_\d+" + field + r"\w*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\nptxas info\s*: Used (\d+) registers", open(log).read())
    assert m, f"no ptxas report for {kernel}<{field}>"
