"""Groth16 batch verification on the device (b200zk_groth16_verify_batch, Context.groth16_verify_batch,
Groth16Verifier.verify_batch): valid batches of every size decided by the one combined check, every single bad proof
decided as the per-proof route decides it (calldata() + bn254_pairing_check_batch), statuses, stability, a launch count
independent of the batch size, and the refusals."""
import pytest

import groth16_batch_ref as g
import pyref as o
import zkey_ref as zr
from ethrex_b200.errors import B200Error
from ethrex_b200.groth16 import Groth16Verifier
from ethrex_b200.zkey import ZkeyProver
from test_gpu_parity import _twist_point_outside_subgroup

pytestmark = pytest.mark.gpu

R, P = g.R, g.P
_KEYS, _PROOFS = {}, {}


def _key(n_pub):
    if n_pub not in _KEYS:
        _KEYS[n_pub] = g.SimKey(n_pub, seed=0xB47C + n_pub)
    return _KEYS[n_pub]


def _proofs(n_pub, n):
    """n valid proofs under _key(n_pub), cached and grown on demand"""
    have = _PROOFS.setdefault(n_pub, [])
    while len(have) < n:
        have.append(_key(n_pub).proof())
    return [p for p, _ in have[:n]], [x for _, x in have[:n]]


def _per_proof(ctx, key, proofs, xs):
    """the per-proof route: each proof's ecpairing calldata, then bn254_pairing_check_batch"""
    ver = Groth16Verifier(ctx, *key.elements())
    cds = [ver.calldata(p, x) for p, x in zip(proofs, xs)]
    live = [cd for cd in cds if cd is not None]
    res, st = ctx.bn254_pairing_check_batch(live) if live else ([], [])
    it = iter(zip(res, st))
    out = []
    for cd in cds:
        if cd is None:
            out.append(False)
        else:
            r, s = next(it)
            out.append(bool(r) and s == 0)
    return out


@pytest.mark.parametrize("n_pub,n", [(1, 1), (1, 2), (0, 31), (2, 32), (1, 33), (3, 1000), (1, 4096)])
def test_valid_batches_are_decided_by_the_combined_check(ctx, n_pub, n):
    key = _key(n_pub)
    proofs, xs = _proofs(n_pub, n)
    valid, status, ok = ctx.groth16_verify_batch(key.vk, proofs, xs_bytes(xs))
    assert valid == [True] * n and status == [0] * n and ok


def xs_bytes(xs):
    return b"".join(int(v).to_bytes(32, "big") for x in xs for v in x)


def test_zkey_proofs_verify_in_batches(ctx):
    for shape in ((11, 2), (27, 3)):
        c = zr.ZkeyCircuit(*shape, seed=0x5EED + shape[0])
        prover = ZkeyProver(ctx, c.zkey())
        try:
            ver = prover.verifier()
            pubs = [[7 + 3 * i + j for j in range(c.n_public)] for i in range(5)]
            proofs = [prover.prove(c.wtns(c.assign(p))) for p in pubs]
            assert ver.verify_batch(proofs, pubs) == [True] * 5
            vk = prover.vk
            valid, status, ok = ctx.groth16_verify_batch(vk, proofs, xs_bytes(pubs))
            assert valid == [True] * 5 and ok
            bad = [list(p) for p in pubs]
            bad[2][0] += 1
            assert ver.verify_batch(proofs, bad) == [True, True, False, True, True]
        finally:
            prover.close()


def _outside_subgroup_b() -> bytes:
    return o.g2_to_be(_twist_point_outside_subgroup())


def _tampers(key, proofs, xs, k):
    """(name, bad proof, its inputs, expected status, well-formed) for position k"""
    pf, x = proofs[k], xs[k]
    j = (k + 1) % len(proofs)
    other = g.SimKey(key.n_pub, seed=0xF00D)
    foreign, fx = other.proof()
    off = (1).to_bytes(32, "big") + (3).to_bytes(32, "big")
    return [("wrong input", pf, [(x[0] + 1) % R] + x[1:], 0, True),
            ("input = r", pf, [R] + x[1:], 2, False),
            ("A swapped", proofs[j][:64] + pf[64:], x, 0, True),
            ("B swapped", pf[:64] + proofs[j][64:192] + pf[192:], x, 0, True),
            ("C swapped", pf[:192] + proofs[j][192:], x, 0, True),
            ("coordinate = p", pf[:32] + P.to_bytes(32, "big") + pf[64:], x, 2, False),
            ("B coordinate = p", pf[:64] + P.to_bytes(32, "big") + pf[96:], x, 2, False),
            ("A off the curve", off + pf[64:], x, 3, False),
            ("C off the curve", pf[:192] + off, x, 3, False),
            ("B outside the subgroup", pf[:64] + _outside_subgroup_b() + pf[192:], x, 3, False),
            ("A = identity", bytes(64) + pf[64:], x, 0, True),
            ("another key", foreign, fx, 0, True)]


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_one_bad_proof_gets_the_per_proof_verdicts(ctx, where):
    key = _key(2)
    n = 33
    proofs, xs = _proofs(2, n)
    k = {"first": 0, "middle": n // 2, "last": n - 1}[where]
    for name, bad, bx, want_status, well_formed in _tampers(key, proofs, xs, k):
        ps, xx = list(proofs), [list(x) for x in xs]
        ps[k], xx[k] = bad, bx
        valid, status, ok = ctx.groth16_verify_batch(key.vk, ps, xs_bytes(xx))
        assert valid == _per_proof(ctx, key, ps, xx), name
        assert valid == [i != k for i in range(n)], name
        assert status == [want_status if i == k else 0 for i in range(n)], name
        assert ok == (not well_formed), name
        ver = Groth16Verifier(ctx, *key.elements())
        assert ver.verify_batch(ps, xx) == valid, name


def test_python_side_rejections(ctx):
    key = _key(1)
    proofs, xs = _proofs(1, 4)
    ver = Groth16Verifier(ctx, *key.elements())
    assert ver.verify_batch(proofs, [xs[0], [-1], [R], xs[3]]) == [True, False, False, True]
    assert ver.verify_batch(proofs, [xs[0], [R + 5], ["1"], xs[3]]) == [True, False, False, True]
    with pytest.raises(ValueError):
        ver.verify_batch([proofs[0][:255]], [xs[0]])
    with pytest.raises(ValueError):
        ver.verify_batch([proofs[0]], [xs[0] + [1]])


def test_cancelling_tamper_is_caught(ctx):
    key = _key(1)
    items = [key.proof(with_logs=True) for _ in range(4)]
    d = 987654321
    logs = [lg for _, _, lg in items]
    logs[1] = (logs[1][0], logs[1][1], (logs[1][2] + d) % R)
    logs[2] = (logs[2][0], logs[2][1], (logs[2][2] - d) % R)
    proofs = [p[:192] + g.g1(c) for (p, _, _), (_, _, c) in zip(items, logs)]
    xs = [x for _, x, _ in items]
    valid, status, ok = ctx.groth16_verify_batch(key.vk, proofs, xs_bytes(xs))
    assert valid == [True, False, False, True] and not ok and status == [0] * 4


def test_stability(ctx):
    key = _key(2)
    proofs, xs = _proofs(2, 40)
    first = ctx.groth16_verify_batch(key.vk, proofs, xs_bytes(xs))
    assert first == ctx.groth16_verify_batch(key.vk, proofs, xs_bytes(xs))
    bad = list(proofs)
    bad[5] = bad[5][:192] + bad[6][192:]
    valid, _, ok = ctx.groth16_verify_batch(key.vk, bad, xs_bytes(xs))
    assert not ok and valid == [i != 5 for i in range(40)]
    assert ctx.groth16_verify_batch(key.vk, proofs, xs_bytes(xs)) == first == ([True] * 40, [0] * 40, True)


def test_launch_count_does_not_grow_with_the_batch(ctx):
    key = _key(1)
    counts = []
    for n in (16, 1024):
        proofs, xs = _proofs(1, n)
        before = ctx.launch_count
        valid, _, ok = ctx.groth16_verify_batch(key.vk, proofs, xs_bytes(xs))
        counts.append(ctx.launch_count - before)
        assert ok and all(valid)
    assert counts[0] == counts[1]


def test_refused_keys_and_buffers(ctx):
    key = _key(1)
    proofs, xs = _proofs(1, 3)
    xb = xs_bytes(xs)
    vk = key.vk
    p_bytes = P.to_bytes(32, "big")
    off = (1).to_bytes(32, "big") + (3).to_bytes(32, "big")
    outside = _outside_subgroup_b()
    refused = [(p_bytes + vk[32:], 2, "alpha1"),
               (vk[:64] + p_bytes + vk[96:], 2, "beta2"),
               (vk[:448 + 64] + vk[448 + 64:448 + 96] + p_bytes, 2, "IC[1]"),
               (off + vk[64:], 3, "alpha1"),
               (vk[:448] + off + vk[512:], 3, "IC[0]"),
               (vk[:64] + outside + vk[192:], 3, "beta2"),
               (vk[:192] + outside + vk[320:], 3, "gamma2"),
               (vk[:320] + outside + vk[448:], 3, "delta2"),
               (vk[:320] + outside + vk[448:480] + p_bytes + vk[512:], 2, "IC[0]")]  # a range error outranks a curve error
    for bad_vk, status, name in refused:
        with pytest.raises(B200Error) as e:
            ctx.groth16_verify_batch(bad_vk, proofs, xb)
        assert e.value.status == status and name in str(e.value), name
        ver = Groth16Verifier(ctx, bad_vk[:64], bad_vk[64:192], bad_vk[192:320], bad_vk[320:448],
                              [bad_vk[448 + 64 * j: 512 + 64 * j] for j in range(2)])
        assert ver.verify_batch(proofs, xs) == [False] * 3, name
        assert ctx.groth16_verify_batch(vk, proofs, xb) == ([True] * 3, [0] * 3, True)
    with pytest.raises(B200Error):  # not 448 + 64 (n_pub + 1) bytes
        ctx.groth16_verify_batch(vk[:-1], proofs, xb)
    with pytest.raises(B200Error):
        ctx.groth16_verify_batch(vk[:448], [], b"")
    assert ctx.groth16_verify_batch(vk, [], b"")[:2] == ([], [])
    with pytest.raises(B200Error):  # short public inputs
        ctx.groth16_verify_batch(vk, proofs, xb[:-1])
    with pytest.raises(B200Error):  # a partial proof
        ctx.groth16_verify_batch(vk, b"".join(proofs)[:-1], xb)
