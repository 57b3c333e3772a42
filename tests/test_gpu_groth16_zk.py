"""Zero-knowledge Groth16 on the device (b200zk_groth16_prove / b200zk_groth16_fold_zk): the toy instance of
tests/groth16_toy.py over a key in the ark-groth16 / gnark layout (tests/groth16_toy_zk.py), blinded with r and s,
bit-exact against the proof computed in the exponent and accepted by the GPU pairing check."""
import ctypes as C

import numpy as np
import pytest

import bls_ref as bls
from groth16_toy import N_PUBLIC, R, ToyGroth16, _g1
from groth16_toy_zk import ArkKey, expected_zk_proof

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200 import _ffi as F
from ethrex_b200.groth16 import Groth16Prover, Groth16Verifier, Groth16ZkProver, quotient_on_device

pytestmark = pytest.mark.gpu

X = 0x1234567
R_CASES = {"zero": (0, 0), "s_only": (0, 0x5A5A5A5A5A5A5A5A5A5A5A5A5A5A5A5A5A5A5A5A), "r_only": (0xC3C3C3C3C3C3C3C3C3C3C3C3, 0),
           "random": (0x2B1E4D7F9A3C6E8B0D2F4A6C8E0B3D5F7A9C1E3B5D7F9A2C4E6B8D0F2A4C6E8, 0x1D3F5B7E9A2C4E6B8D0F2A4C6E8B1D3F5A7C9E0B2D4F6A8C0E2B4D6F8A1C3E5),
           "order_minus_1": (R - 1, R - 1)}

_TOYS = {}


def _toy(log_n):
    if log_n not in _TOYS:
        toy = ToyGroth16(log_n)
        _TOYS[log_n] = (toy, ArkKey(toy))
    return _TOYS[log_n]


def _prover(ctx, log_n):
    toy, key = _toy(log_n)
    return toy, Groth16ZkProver(ctx, log_n, *key.columns(), N_PUBLIC, *key.terms())


def _host_inputs(prover, toy, z):
    return prover._host_inputs(z, *toy.evaluations(z))


def _dev(buf):
    import torch
    return torch.from_numpy(np.frombuffer(bytes(buf), dtype=np.int64).copy()).cuda()


@pytest.mark.parametrize("case", sorted(R_CASES))
@pytest.mark.parametrize("log_n", [3, 4, 5])
def test_blinded_proof_is_bit_exact(ctx, log_n, case):
    r, s = R_CASES[case]
    toy, prover = _prover(ctx, log_n)
    try:
        z = toy.assign(X)
        assert prover.prove(z, *toy.evaluations(z), r=r, s=s) == expected_zk_proof(toy, z, r, s)
    finally:
        prover.close()


@pytest.mark.parametrize("log_n", [3, 4])
def test_unblinded_ark_key_equals_the_folded_key_path(ctx, log_n):
    """r = s = 0 over the ark-layout key == b200zk_groth16_commit over the toy's key with alpha / beta folded in"""
    toy, prover = _prover(ctx, log_n)
    plain = Groth16Prover(ctx, log_n, toy.a_g1, toy.b_g1, toy.b_g2, toy.l_g1, toy.h_g1, N_PUBLIC)
    try:
        for x in (X, 0, R - 1):
            z = toy.assign(x)
            assert prover.prove(z, *toy.evaluations(z), r=0, s=0) == plain.prove(z, *toy.evaluations(z)) == toy.expected_proof(z)
    finally:
        prover.close()
        plain.close()


def test_blinded_proofs_verify_and_are_reproducible(ctx):
    toy, prover = _prover(ctx, 4)
    ver = Groth16Verifier(ctx, toy.vk_alpha_g1, toy.vk_beta_g2, toy.vk_gamma_g2, toy.vk_delta_g2, [_g1(k) for k in toy.ic])
    try:
        z = toy.assign(X)
        ev = toy.evaluations(z)
        proofs = [prover.prove(z, *ev, r=r, s=s) for r, s in R_CASES.values()]
        drawn = [prover.prove(z, *ev) for _ in range(2)]  # fresh random r, s
        assert all(ver.verify_batch(proofs + drawn, [[X]] * (len(proofs) + len(drawn))))
        assert not any(ver.verify_batch(proofs, [[X + 1]] * len(proofs)))
        assert len(set(proofs + drawn)) == len(proofs) + len(drawn)  # different (r, s), different proofs
        r, s = R_CASES["random"]
        assert prover.prove(z, *ev, r=r, s=s) == prover.prove(z, *ev, r=r, s=s) == proofs[list(R_CASES).index("random")]
    finally:
        prover.close()


def test_host_and_device_inputs_agree(ctx):
    """host buffers, device buffers (G16_INPUTS_DEVICE) and device quotient coefficients (G16_H_COEFFS): same bytes"""
    log_n = 4
    toy, prover = _prover(ctx, log_n)
    try:
        z = toy.assign(X)
        r, s = R_CASES["random"]
        zk = ctx.groth16_zk(prover.h["terms_g1"], prover.h["terms_g2"], r, s)
        wb, ab, bb, cb = _host_inputs(prover, toy, z)
        host = ctx.groth16_prove(prover.pk, zk, wb, ab, bb, cb)
        assert host == expected_zk_proof(toy, z, r, s)
        dev = ctx.groth16_prove(prover.pk, zk, _dev(wb), _dev(ab), _dev(bb), _dev(cb), F.G16_INPUTS_DEVICE)
        assert dev == host
        a, b, c = _dev(ab), _dev(bb), _dev(cb)
        h = quotient_on_device(ctx, log_n, a, b, c, prover.zinv)
        assert ctx.groth16_prove(prover.pk, zk, _dev(wb), h, None, None, F.G16_INPUTS_DEVICE | F.G16_H_COEFFS) == host
    finally:
        prover.close()


def test_point_split_fold_zk_equals_one_call(ctx):
    """three uneven shards of every column on one GPU, commit_partial each, ONE fold_zk over the three blocks"""
    import torch
    log_n = 4
    toy, key = _toy(log_n)
    prover = Groth16ZkProver(ctx, log_n, *key.columns(), N_PUBLIC, *key.terms())
    handles = []
    try:
        z = toy.assign(X)
        wb, ab, bb, cb = _host_inputs(prover, toy, z)
        r, s = R_CASES["random"]
        zk = ctx.groth16_zk(prover.h["terms_g1"], prover.h["terms_g2"], r, s)
        whole = ctx.groth16_prove(prover.pk, zk, wb, ab, bb, cb)
        assert whole == expected_zk_proof(toy, z, r, s)
        w = _dev(wb)
        h = quotient_on_device(ctx, log_n, _dev(ab), _dev(bb), _dev(cb), prover.zinv)
        m, n = toy.m, toy.n
        cols = [(key.a_g1, 64, m, 0), (key.b_g1, 64, m, 0), (key.b_g2, 128, m, 0), (key.l_g1, 64, m - N_PUBLIC, N_PUBLIC), (key.h_g1, 64, n - 1, 0)]
        blocks = torch.zeros(96 * 3, dtype=torch.int64, device="cuda")
        for j, (f0, f1) in enumerate(((0.0, 0.15), (0.15, 0.7), (0.7, 1.0))):
            hs, counts, offs = [], [], []
            for k, (col, width, total, base) in enumerate(cols):
                lo, hi = int(total * f0), int(total * f1)
                up = ctx.g2_bases_upload if width == 128 else ctx.g1_bases_upload
                hd = up(col[width * lo:width * hi], hi - lo, F.POINTS_BE)
                handles.append(hd)
                hs.append(hd); counts.append(hi - lo); offs.append(base + lo)
            pk = ctx.groth16_pk(log_n, hs, counts, offs)
            ctx.groth16_commit_partial(pk, w, h, None, None, blocks[96 * j:96 * (j + 1)], F.G16_INPUTS_DEVICE | F.G16_H_COEFFS)
        assert ctx.groth16_fold_zk(zk, blocks, 3) == whole
    finally:
        for hd in handles:
            ctx.bases_free(hd)
        prover.close()


def _status_prove(ctx, pk, zk, inputs):
    wb, ab, bb, cb = inputs
    keep = [np.frombuffer(bytes(x), dtype=np.uint8).copy() for x in (wb, ab, bb, cb)]
    ptrs = [k.ctypes.data_as(C.c_void_p) for k in keep]
    out = C.create_string_buffer(256)
    return F.lib.b200zk_groth16_prove(ctx._h, C.byref(pk), C.byref(zk) if zk is not None else None, *ptrs, 0, None, out)


def _status_fold(ctx, zk, blocks):
    out = C.create_string_buffer(256)
    return F.lib.b200zk_groth16_fold_zk(ctx._h, C.byref(zk) if zk is not None else None, C.c_void_p(blocks.data_ptr()), 1, None, out)


def test_refusals(ctx):
    import torch
    toy, prover = _prover(ctx, 3)
    extra = []
    try:
        z = toy.assign(X)
        inputs = _host_inputs(prover, toy, z)
        t1, t2 = prover.h["terms_g1"], prover.h["terms_g2"]
        blocks = torch.zeros(96, dtype=torch.int64, device="cuda")
        ok = ctx.groth16_zk(t1, t2, 1, 2)
        assert _status_prove(ctx, prover.pk, ok, inputs) == F.OK
        assert _status_fold(ctx, ok, blocks) == F.OK
        # r or s not below the group order: status 2, never reduced
        for r, s in ((R, 0), (0, R), (R + 1, 5), (1 << 255, 1), (3, (1 << 256) - 1)):
            zk = ctx.groth16_zk(t1, t2, r, s)
            assert _status_prove(ctx, prover.pk, zk, inputs) == F.ERR_NOT_IN_FIELD
            assert _status_fold(ctx, zk, blocks) == F.ERR_NOT_IN_FIELD
        # NULL zk
        assert _status_prove(ctx, prover.pk, None, inputs) == F.ERR_INVALID_ARG
        assert _status_fold(ctx, None, blocks) == F.ERR_INVALID_ARG
        # term handles: wrong count, wrong group, BLS12-381, precomputed, unknown
        key = _toy(3)[1]
        two_g1 = ctx.g1_bases_upload(key.alpha_g1 + key.beta_g1, 2, F.POINTS_BE)
        four_g1 = ctx.g1_bases_upload(key.alpha_g1 + key.beta_g1 + key.delta_g1 + key.delta_g1, 4, F.POINTS_BE)
        three_g2 = ctx.g2_bases_upload(key.beta_g2 + key.delta_g2 + key.delta_g2, 3, F.POINTS_BE)
        bls_h = ctx.bls12_381_g1_bases_upload(bls.G1_COMPRESSED * 3, 3)
        pre_g1 = ctx.g1_bases_upload(key.alpha_g1 + key.beta_g1 + key.delta_g1, 3, F.POINTS_BE)
        ctx.bases_precompute(pre_g1, 0)
        pre_g2 = ctx.g2_bases_upload(key.beta_g2 + key.delta_g2, 2, F.POINTS_BE)
        ctx.bases_precompute(pre_g2, 0)
        extra += [two_g1, four_g1, three_g2, bls_h, pre_g1, pre_g2]
        bad = [(two_g1, t2), (four_g1, t2), (t1, three_g2), (t2, t2), (t1, t1), (t2, t1), (bls_h, t2), (pre_g1, t2), (t1, pre_g2),
               (0, t2), (t1, 0), (t1 + 1000, t2)]
        for g1, g2 in bad:
            zk = ctx.groth16_zk(g1, g2, 1, 2)
            assert _status_prove(ctx, prover.pk, zk, inputs) == F.ERR_INVALID_ARG, (g1, g2)
            assert _status_fold(ctx, zk, blocks) == F.ERR_INVALID_ARG, (g1, g2)
        # r != 0 needs the B_g1 column; r = 0 does not (and gives the same proof)
        pk = prover.pk
        no_b1 = ctx.groth16_pk(pk.log_n, [pk.handle[0], 0, pk.handle[2], pk.handle[3], pk.handle[4]], list(pk.count), list(pk.offset))
        assert _status_prove(ctx, no_b1, ok, inputs) == F.ERR_INVALID_ARG
        zero_r = ctx.groth16_zk(t1, t2, 0, 7)
        assert ctx.groth16_prove(no_b1, zero_r, *inputs) == ctx.groth16_prove(pk, zero_r, *inputs) == expected_zk_proof(toy, z, 0, 7)
        # the Python wrapper raises on the same statuses
        with pytest.raises(eb.B200Error):
            ctx.groth16_prove(pk, ctx.groth16_zk(t1, t2, R, 0), *inputs)
    finally:
        for hd in extra:
            ctx.bases_free(hd)
        prover.close()
