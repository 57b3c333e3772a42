"""CPU checks of the EIP-4844 proof path: the Fr381 constants of bls381.cuh recomputed from their definitions, the reference
quotient (tests/kzg_ref.py) against the spec's direct formulas, the library's host SHA-256 against hashlib, KzgSettings'
bookkeeping over a stand-in context, and the ptxas report of the new kernels."""
import os
import re
import subprocess

import numpy as np
import pytest

import bls_ref as bls
import kzg_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ethrex_b200", "csrc")


def _limbs(cfg: str, name: str) -> int:
    """the 8 x u32 little-endian array `name` of struct `cfg` in bls381.cuh, as an integer"""
    txt = open(os.path.join(CSRC, "bls381.cuh")).read()
    body = txt[txt.index(f"struct {cfg}"):]
    body = body[:body.index("\n};")]
    m = re.search(name + r"\(int i\) \{[^{]*\{([^}]*)\}", body)
    words = [int(w.strip().rstrip("u"), 16) for w in m.group(1).split(",")]
    return sum(w << (32 * i) for i, w in enumerate(words))


def test_fr381_constants_from_their_definitions():
    txt = open(os.path.join(CSRC, "bls381.cuh")).read()
    r = bls.R
    limbs = re.search(r"bls_r_limb\(int i\) \{[^{]*\{([^}]*)\}", txt).group(1).split(",")
    assert sum(int(w.strip().rstrip("u"), 16) << (32 * i) for i, w in enumerate(limbs)) == r
    assert _limbs("Fr381Cfg", "r1") == (1 << 256) % r
    assert _limbs("Fr381Cfg", "r2") == (1 << 512) % r
    inv = int(re.search(r"struct Fr381Cfg.*?INV = (0x[0-9a-f]+)u", txt, re.S).group(1), 16)
    assert inv == (-pow(r, -1, 1 << 32)) % (1 << 32)
    assert 2 * r < 1 << 256  # FeBig::add and mul need no carry limb
    # the root of unity and 1/4096 the device derives: w = 7^((r-1)/4096) has order exactly 4096
    w = pow(7, (r - 1) // 4096, r)
    assert w == bls.ROOT_4096 and pow(w, 4096, r) == 1 and pow(w, 2048, r) == r - 1
    assert w == 0x564C0A11A0F704F4FC3E8ACFE0F8245F0AD1347B378FBF96E206DA11A5D36306
    assert (r - (r - 1) // 4096) * 4096 % r == 1
    roots = ref.roots_brp()
    assert roots[0] == 1 and roots[1] == r - 1 and len(set(roots)) == 4096


def _direct(poly, z):
    """the spec's formulas, written out for one z: y = p(z) through the Lagrange basis, q_i = (p_i - y)/(w_i - z) and the
    in-domain q_m = sum_{i != m} (p_i - y) w_i / (z (z - w_i))"""
    r, roots = bls.R, ref.roots_brp()
    y = ref.evaluate_direct(poly, z)
    q = []
    for i, w in enumerate(roots):
        if w == z:
            q.append(sum((poly[j] - y) * roots[j] * pow(z * (z - roots[j]) % r, -1, r) for j in range(4096) if j != i) % r)
        else:
            q.append((poly[i] - y) * pow((w - z) % r, -1, r) % r)
    return q, y


@pytest.mark.parametrize("case", ["random", "ones", "single", "in_domain_0", "in_domain_77", "zero_z"])
def test_reference_quotient_matches_the_spec(case):
    rng = np.random.default_rng(11)
    poly = [int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]
    z = int.from_bytes(rng.bytes(32), "big") % bls.R
    if case == "ones":
        poly = [1] * 4096
    if case == "single":
        poly = [0] * 4096
        poly[4095] = bls.R - 1
    if case.startswith("in_domain"):
        z = ref.roots_brp()[int(case.rsplit("_", 1)[1])]
    if case == "zero_z":
        z = 0
    q, y = ref.quotient(poly, z)
    assert (q, y) == _direct(poly, z)
    if case == "ones":
        assert y == 1 and q == [0] * 4096


def test_host_sha256_matches_hashlib(tmp_path):
    """ethrex_b200/csrc/sha256.h (the challenge hash of b200zk_kzg_blob_to_commitment_and_proof), compiled on its own"""
    src = tmp_path / "sha.cpp"
    src.write_text('#include "sha256.h"\n#include <cstdio>\n#include <cstdlib>\n#include <vector>\n'
                   "int main(int argc, char** argv) {\n"
                   "  size_t n = strtoul(argv[1], 0, 10), split = strtoul(argv[2], 0, 10);\n"
                   "  std::vector<uint8_t> m(n + 1);\n"
                   "  for (size_t i = 0; i < n; ++i) m[i] = (uint8_t)(i * 131 + 7);\n"
                   "  b200zk::Sha256 h;\n"
                   "  h.update(m.data(), split);\n"
                   "  h.update(m.data() + split, n - split);\n"
                   "  uint8_t d[32];\n"
                   "  h.final(d);\n"
                   '  for (int i = 0; i < 32; ++i) printf("%02x", d[i]);\n'
                   "}\n")
    exe = tmp_path / "sha"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", CSRC, str(src), "-o", str(exe)])
    import hashlib
    for n in (0, 1, 55, 56, 63, 64, 65, 119, 120, 128, 16 + 16 + 131072 + 48):
        for split in sorted({0, min(1, n), min(63, n), min(64, n), n // 2, n}):
            msg = bytes((i * 131 + 7) & 255 for i in range(n))
            got = subprocess.run([str(exe), str(n), str(split)], capture_output=True, text=True, check=True).stdout
            assert got == hashlib.sha256(msg).hexdigest(), (n, split)


def test_kzg_settings_over_the_one_call_entry_points_without_a_gpu():
    """ethrex_b200/kzg.py around the device calls (challenge, z encoding, y decoding, exception types), with the two KZG
    calls served in the exponent by a stand-in context built on the reference quotient: the commitment must be p(tau) G and
    the proof ((p(tau) - p(z)) / (tau - z)) G for a synthetic Lagrange setup (device half: tests/test_gpu_kzg_proof.py)."""
    import ethrex_b200 as eb
    from ethrex_b200.kzg import KzgSettings, roots_of_unity_brp
    tau = 0x123456789ABCDEF0FEDCBA9876543210 % bls.R
    lag = bls.lagrange_setup_scalars(tau)

    def at_tau(vals):
        return sum(v * l for v, l in zip(vals, lag)) % bls.R

    class ExponentCtx:
        def bls12_381_g1_bases_upload(self, pts, n, flags=0): return 1
        def bases_precompute(self, h, c): pass
        def bases_free(self, h): pass

        def _blobs(self, raw):
            vals = [ref.blob_values(raw[k * 131072:(k + 1) * 131072]) for k in range(len(raw) // 131072)]
            if any(v >= bls.R for b in vals for v in b):
                raise eb.B200Error.serialization("element >= r", 2)
            return vals

        def _proof(self, vals, z):
            q, y = ref.quotient(vals, z)
            return bls.compress(bls.mul(at_tau(q), bls.G1)), y.to_bytes(32, "big")

        def kzg_blob_to_commitment_and_proof(self, h, raw):
            cs, ps = [], []
            for vals in self._blobs(raw):
                cs.append(bls.compress(bls.mul(at_tau(vals), bls.G1)))
                ps.append(self._proof(vals, ref.challenge(ref.to_blob(vals), cs[-1]))[0])
            return cs, ps

        def kzg_compute_proof(self, h, raw, zs):
            out = [self._proof(vals, int.from_bytes(zs[32 * k:32 * k + 32], "big")) for k, vals in enumerate(self._blobs(raw))]
            return [p for p, _ in out], [y for _, y in out]

    st = KzgSettings(ExponentCtx(), bytes(48 * 4096), precompute=True)
    rng = np.random.default_rng(7)
    vals = [int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(4096)]
    blob = ref.to_blob(vals)
    p_tau = at_tau(vals)
    c, proof = st.blob_to_kzg_commitment_and_proof(blob)
    assert c == bls.compress(bls.mul(p_tau, bls.G1))
    z = st.compute_challenge(blob, c)
    assert z == ref.challenge(blob, c)
    proof_z, y = st.compute_kzg_proof(blob, z)
    assert proof_z == proof == st.compute_blob_kzg_proof(blob, c)
    assert y == ref.evaluate_direct(vals, z)
    assert proof == bls.compress(bls.mul((p_tau - y) * pow((tau - z) % bls.R, -1, bls.R) % bls.R, bls.G1))
    zr = roots_of_unity_brp()[1234]
    proof_r, yr = st.compute_kzg_proof(blob, zr)
    assert yr == vals[1234]
    assert proof_r == bls.compress(bls.mul((p_tau - yr) * pow((tau - zr) % bls.R, -1, bls.R) % bls.R, bls.G1))
    with pytest.raises(ValueError):
        st.compute_kzg_proof(bls.R.to_bytes(32, "big") + blob[32:], 5)
    with pytest.raises(ValueError):
        st.compute_kzg_proof(blob, bls.R)
    with pytest.raises(eb.B200Error):
        st.blob_to_kzg_commitment_and_proof(bls.R.to_bytes(32, "big") + blob[32:])


@pytest.mark.parametrize("kernel", ["kzg_eval_quotient", "kzg_roots_build"])
def test_kzg_kernels_do_not_spill(kernel):
    log = os.path.join(CSRC, "build", "bls381.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("bls381.ptxas.log not built")
    m = re.search(r"Function properties for \w*" + kernel + r"\w*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                  open(log).read())
    assert m, f"no ptxas report for {kernel}"
    assert m.group(2) == "0" and m.group(3) == "0", m.group(0)
