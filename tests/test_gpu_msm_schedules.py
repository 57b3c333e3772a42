"""The MSM schedules that the other parity files do not reach: BLS12-381 (msm_run<Fp381>, 256 scalar bits) through the
two-level sort, dense bucket totals, pair-sum rounds, the chunk-pipelined schedule, window tables and forced windows; the
BN254 partial-sum entry points over resident bases; the profiled schedule; and the refusal of B200ZK_SCALARS_RAW by every
BN254 MSM entry point.

Every case first asks a host-side mirror of the planner (below) which branch it takes and asserts that it is the one the
case is meant to cover, so that a later change of defaults cannot silently move a test off its branch.  Results are
compared bytes-for-bytes with a closed form: every base is a known multiple of the generator, so the MSM is one scalar
multiplication, evaluated by the CPU oracle (BN254) or by oracle/bls_ref.py (BLS12-381)."""
import math
from dataclasses import dataclass

import numpy as np
import pytest

import bls_ref as bls
import cpu_oracle as orc
import pyref
from helpers import chain_kd, dev_empty, expected_chain_msm_g1, expected_chain_msm_g2, scalars_special, to_dev, to_host

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402
from ethrex_b200 import _ffi as F  # noqa: E402


# ------------------------------------------------------------------------------------------ planner mirror
@dataclass(frozen=True)
class Plan:
    c: int
    W: int
    G: int            # buckets to reduce: W * 2^(c-1), or 2^(c-1) on a window table
    merged: bool      # window table: all windows share one bucket set
    two_level: bool   # two-level digit sort instead of the legacy hist / scan / scatter one
    dense: bool       # one-shot schedule: dense bucket totals instead of the fused bucket_chunk
    bitsums: bool     # bucket reduction by bit-sums (T >= 64) instead of the pairwise tree

    @property
    def top_bit(self):  # bit at which the top window ends
        return self.c * self.W


def table_window(n_bases: int) -> int:
    """precompute_window (msm.cu:44-52): the window b200zk_bases_precompute(handle, 0) picks"""
    lg = (n_bases - 1).bit_length()
    return 20 if lg >= 20 else (6 if lg <= 6 else lg)


def msm_plan(n: int, forced_c: int = 0, scalar_bits: int = 255, table_c: int = 0) -> Plan:
    """make_plan (msm.cu:56-79), make_sort_plan (msm.cu:270-287) and the reduction choices of msm_run (dense totals
    msm.cu:1514, bit-sums msm.cu:1631).  scalar_bits: 255 for BN254, 256 for BLS12-381 (ScalarBits<F>)."""
    lg = (n - 1).bit_length()
    forced = table_c or forced_c       # a window table fixes c; set_msm_window does not apply to it
    c = forced if forced else (lg - 4 if lg > 8 else 4)
    if not forced and c > 16:
        c = 17 if lg >= 23 else 16
    c = min(max(c, 2), 24)
    W = -(-scalar_bits // c)
    B = 1 << (c - 1)
    T = B // min(B, 16)
    G = (1 if table_c else W) * B
    kb = (G - 1).bit_length()
    cb = 10 if kb > 19 else 9
    two_level = W <= 16 and kb >= 12 and n >= (1 << 16) and kb - cb <= 11
    return Plan(c, W, G, bool(table_c), two_level, G >= (1 << 14), T >= 64)


def pipelined(n: int, chunks: int = 0, host_scalars: bool = False, profiling: bool = False, pair_rounds: int = -1, g2: bool = False) -> bool:
    """msm_run's choice of the chunk-pipelined schedule (msm.cu:1499-1502).  BLS12-381 calls stage their scalars
    themselves and reach msm_run with device scalars (host_scalars=False)."""
    K = chunks or ((2 if g2 else 3) if host_scalars and n >= (1 << 22) else 1)
    return (K > 1 or host_scalars) and not profiling and pair_rounds <= 0 and n >= 4096


def test_plan_mirror_matches_the_documented_defaults():
    """the mirror itself, on the numbers msm.cu's comments state: c = lg(n) - 4 up to 16, 16 for 2^20..2^22 points, 17 from
    2^23; 20 for a window table from 2^20; the BLS12-381 top window at c = 16 ends exactly at bit 256"""
    assert msm_plan(1 << 18).c == 14 and msm_plan(1 << 20).c == 16 and msm_plan(1 << 22).c == 16 and msm_plan(1 << 23).c == 17
    assert table_window(1 << 24) == 20 and table_window(3000) == 12 and table_window(10) == 6
    p = msm_plan((1 << 20) + 1, scalar_bits=256)
    assert (p.c, p.W, p.top_bit, p.two_level) == (16, 16, 256, True)
    assert msm_plan(1 << 24, table_c=20).two_level and not msm_plan(1 << 24, forced_c=12).two_level


# ------------------------------------------------------------------------------------------ BLS12-381 helpers
BLS_K = 0x2C1F6D8A9B3E4F5061728394A5B6C7D8E9F00112233445566778899AABBCCDD % bls.R
BLS_D = 0x1B2C3D4E5F60718293A4B5C6D7E8F9012345678987654321FEDCBA9876543210 % bls.R
N_MID = (1 << 16) + 12345


def bls_logs(n, start=0):
    """discrete logs of bls.chain(n, BLS_K, BLS_D) (offset by `start`)"""
    return [(BLS_K + (start + i) * BLS_D) % bls.R for i in range(n)]


def bls_expected(vals, logs) -> bytes:
    """closed form of sum_i vals[i] * (logs[i] * G), compressed"""
    return bls.compress(bls.mul(sum(v * l for v, l in zip(vals, logs)) % bls.R, bls.G1))


def bls_random(n, seed):
    rng = np.random.default_rng(seed)
    vals = [int.from_bytes(rng.bytes(32), "big") % bls.R for _ in range(n)]
    # bit 254 set (r > 2^254), r - 1 and the top-window neighbours, tiny values
    for i, v in enumerate((0, 1, 2, bls.R - 1, bls.R - 2, 1 << 254, (1 << 254) + (1 << 253), (1 << 240) - 1, 0xFFFF)):
        if i < n:
            vals[(i * 7919) % n] = v
    return vals


def be(vals) -> bytes:
    return b"".join(v.to_bytes(32, "big") for v in vals)


def le(vals) -> bytes:
    return b"".join(v.to_bytes(32, "little") for v in vals)


@pytest.fixture(scope="module")
def bls_mid():
    """bls.chain over N_MID = 2^16 + 12345 points (a prefix of it serves the smaller cases)"""
    return bls.chain(N_MID, BLS_K, BLS_D), bls_logs(N_MID)


def _bls_handle(ctx, raw, n, table_c=None):
    h = ctx.bls12_381_g1_bases_upload(raw[:96 * n], n, 0)
    if table_c is not None:
        ctx.bases_precompute(h, table_c)
    return h


# ------------------------------------------------------------------------------------------ BLS12-381: plain bases
@pytest.mark.parametrize("n", [(1 << 16) - 1, N_MID])
def test_bls_plain_bases_legacy_sort_dense_totals(ctx, bls_mid, n):
    """22 / 20 windows of c = 12 / 13: too many windows for the two-level sort, enough buckets for dense totals"""
    p = msm_plan(n, scalar_bits=256)
    assert not p.two_level and p.dense and p.bitsums and not pipelined(n)
    raw, logs = bls_mid
    vals = bls_random(n, seed=n)
    exp = bls_expected(vals, logs[:n])
    h = _bls_handle(ctx, raw, n)
    try:
        assert ctx.bls12_381_g1_msm_resident(h, be(vals), n) == exp
        assert ctx.bls12_381_g1_msm_resident(h, le(vals), n, 0) == exp
    finally:
        ctx.bases_free(h)


def test_bls_plain_bases_two_level_sort_at_2_20(ctx):
    """2^20 + 1 points at the default c = 16: the two-level sort over 16 windows, the top one ending at bit 256"""
    n = (1 << 20) + 1
    p = msm_plan(n, scalar_bits=256)
    assert (p.c, p.top_bit) == (16, 256) and p.two_level and p.dense and p.bitsums
    raw = bls.chain(n, BLS_K, BLS_D)
    vals = bls_random(n, seed=20)
    exp = bls_expected(vals, bls_logs(n))
    h = _bls_handle(ctx, raw, n)
    del raw
    try:
        assert ctx.bls12_381_g1_msm_resident(h, be(vals), n) == exp
        assert ctx.bls12_381_g1_msm_resident(h, le(vals), n, 0) == exp
    finally:
        ctx.bases_free(h)


def test_bls_window_sweep(ctx, bls_mid):
    """forced windows from 2 to 20 at n = 3000 (c = 2, 4, 8, 16 divide 256: the top window ends at bit 256), and at
    n = 257 against the affine double-and-add of bls_ref.msm"""
    raw, logs = bls_mid
    n, small = 3000, 257
    vals = bls_random(n, seed=3000)
    exp = bls_expected(vals, logs[:n])
    exp_small = bls.compress(bls.msm(vals[:small], [bls.mul(l, bls.G1) for l in logs[:small]]))
    assert exp_small == bls_expected(vals[:small], logs[:small])
    sweep = (2, 3, 4, 5, 7, 8, 11, 12, 13, 16, 17, 20)
    plans = [msm_plan(n, c, 256) for c in sweep]
    assert {p.dense for p in plans} == {True, False} and {p.bitsums for p in plans} == {True, False}
    assert {p.top_bit for p in plans if 256 % p.c == 0} == {256}
    h = _bls_handle(ctx, raw, n)
    try:
        for c in sweep:
            ctx.set_msm_window(c)
            assert ctx.bls12_381_g1_msm_resident(h, be(vals), n) == exp, c
            assert ctx.bls12_381_g1_msm_resident(h, be(vals[:small]), small) == exp_small, c
    finally:
        ctx.set_msm_window(0)
        ctx.bases_free(h)


# ------------------------------------------------------------------------------------------ BLS12-381: window tables
@pytest.mark.parametrize("c", [0, 6, 11, 16, 20])
def test_bls_window_tables(ctx, bls_mid, c):
    """merged tables at c = 17 (automatic), 6, 11, 16, 20: W <= 16 takes the two-level sort, 43 and 24 windows the legacy
    one; a prefix of the table (n < 2^16) always the legacy sort"""
    raw, logs = bls_mid
    n = N_MID
    tc = c or table_window(n)
    p = msm_plan(n, scalar_bits=256, table_c=tc)
    assert p.merged and p.two_level == (c in (0, 16, 20)) and tc == (17 if c == 0 else c)
    m = 10007
    assert not msm_plan(m, scalar_bits=256, table_c=tc).two_level
    vals = bls_random(n, seed=100 + c)
    h = _bls_handle(ctx, raw, n, c)
    try:
        assert ctx.bls12_381_g1_msm_resident(h, be(vals), n) == bls_expected(vals, logs)
        assert ctx.bls12_381_g1_msm_resident(h, le(vals[:m]), m, 0) == bls_expected(vals[:m], logs[:m])
    finally:
        ctx.bases_free(h)


@pytest.mark.parametrize("table", [False, True])
def test_bls_two_level_sort_on_skewed_scalars(ctx, bls_mid, table):
    """the BLS12-381 twin of test_two_level_sort_on_skewed_scalars: plain bases at a forced c = 16, and the automatic
    window table (c = 17), under all-equal, half-zero, tiny, all-(r - 1) and Zipf-like scalars"""
    raw, logs = bls_mid
    n = N_MID
    p = msm_plan(n, scalar_bits=256, table_c=table_window(n)) if table else msm_plan(n, 16, 256)
    assert p.two_level
    rnd = bls_random(n, seed=77)
    cases = {
        "all equal": [rnd[5]] * n,
        "half zeros": [0 if i % 2 == 0 else v for i, v in enumerate(rnd)],
        "below 2^16": [v & 0xFFFF for v in rnd],
        "all r - 1": [bls.R - 1] * n,
        "zipf-like": [rnd[7]] * (n // 2) + [rnd[11]] * (n // 4) + rnd[n // 2 + n // 4:],
    }
    h = _bls_handle(ctx, raw, n, 0 if table else None)
    try:
        if not table:
            ctx.set_msm_window(16)
        for name, vals in cases.items():
            assert len(vals) == n
            assert ctx.bls12_381_g1_msm_resident(h, be(vals), n) == bls_expected(vals, logs), name
    finally:
        ctx.set_msm_window(0)
        ctx.bases_free(h)


# ------------------------------------------------------------------------------------------ BLS12-381: pair sums, chunks
def test_bls_pair_sum_rounds_edge_bases(ctx, bls_mid):
    """batched-affine pair-sum rounds 1..4 over Fp381 at c = 6 and 11: repeated bases (tangent case), P and -P (identity),
    identity bases, with one heavy bucket, one value everywhere and neighbours that share every digit"""
    raw, logs = bls_mid
    n = 4096
    pts = bytearray(raw[:96 * n])
    logs = list(logs[:n])

    def put(i, rec, log):
        pts[96 * i:96 * i + 96] = rec
        logs[i] = log % bls.R

    for dst, src in ((1, 0), (3, 2), (9, 8)):                                       # repeated bases
        put(dst, bytes(pts[96 * src:96 * src + 96]), logs[src])
    x, y = int.from_bytes(pts[96 * 4:96 * 4 + 48], "big"), int.from_bytes(pts[96 * 4 + 48:96 * 5], "big")
    put(5, x.to_bytes(48, "big") + (bls.P - y).to_bytes(48, "big"), -logs[4])       # P and -P
    for i in (7, 11):
        put(i, bls.uncompressed(None), 0)                                          # identity bases
    cases = {
        "all_one": [1] * n,
        "all_same": [0x1234567] * n,
        "pairs": [(i // 2) * 7919 + 1 for i in range(n)],
    }
    h = ctx.bls12_381_g1_bases_upload(bytes(pts), n, 0)
    try:
        for c in (6, 11):
            ctx.set_msm_window(c)
            for rounds in (1, 2, 3, 4):
                assert not pipelined(n, pair_rounds=rounds)
                ctx.set_msm_pair_rounds(rounds)
                for name, vals in cases.items():
                    assert ctx.bls12_381_g1_msm_resident(h, be(vals), n) == bls_expected(vals, logs), (c, rounds, name)
    finally:
        ctx.set_msm_window(0)
        ctx.set_msm_pair_rounds(-1)
        ctx.bases_free(h)


@pytest.mark.parametrize("n", [10007, N_MID])
def test_bls_pipelined_chunks_match_one_shot(ctx, bls_mid, n):
    """set_msm_chunks 2 / 3 / 7 on plain bases and on the automatic window table: the chunk-pipelined schedule (each
    chunk's totals folded into dense totals) returns the one-shot bytes"""
    raw, logs = bls_mid
    assert not pipelined(n) and all(pipelined(n, chunks=k) for k in (2, 3, 7))
    vals = bls_random(n, seed=7 + n)
    exp = bls_expected(vals, logs[:n])
    hp, ht = _bls_handle(ctx, raw, n), _bls_handle(ctx, raw, n, 0)
    try:
        one_shot = {h: ctx.bls12_381_g1_msm_resident(h, be(vals), n) for h in (hp, ht)}
        assert list(one_shot.values()) == [exp, exp]
        for chunks in (2, 3, 7):
            ctx.set_msm_chunks(chunks)
            for h in (hp, ht):
                assert ctx.bls12_381_g1_msm_resident(h, be(vals), n) == one_shot[h], (chunks, h == ht)
    finally:
        ctx.set_msm_chunks(0)
        ctx.bases_free(hp)
        ctx.bases_free(ht)


@pytest.mark.parametrize("c", [0, 16])
def test_bls_scalar_encodings_and_range_check(ctx, bls_mid, c):
    """big- and little-endian scalars give the same bytes; in either order a scalar >= r is refused with status 2 -- at
    c = 8 (the default for 4096 points, top window bits 248..255) and c = 16 (bits 240..255) a value >= 2^255 would not
    fit the top window.  r - 1 is the largest scalar accepted."""
    raw, logs = bls_mid
    n = 4096
    assert msm_plan(n, c, 256).top_bit == 256
    vals = bls_random(n, seed=4096)
    exp = bls_expected(vals, logs[:n])
    h = _bls_handle(ctx, raw, n)
    try:
        ctx.set_msm_window(c)
        assert ctx.bls12_381_g1_msm_resident(h, be(vals), n) == exp
        assert ctx.bls12_381_g1_msm_resident(h, le(vals), n, 0) == exp
        top = list(vals)
        top[1234] = bls.R - 1
        assert ctx.bls12_381_g1_msm_resident(h, le(top), n, 0) == bls_expected(top, logs[:n])
        for bad in (bls.R, 1 << 255, (1 << 256) - 1):
            wrong = list(vals)
            wrong[2345] = bad
            for order, flags in (("little", 0), ("big", eb.SCALARS_BE)):
                with pytest.raises(eb.B200Error) as e:
                    ctx.bls12_381_g1_msm_resident(h, b"".join(v.to_bytes(32, order) for v in wrong), n, flags)
                assert e.value.status == 2, (hex(bad), order)
        assert ctx.bls12_381_g1_msm_resident(h, le(vals), n, 0) == exp  # the context is still usable
    finally:
        ctx.set_msm_window(0)
        ctx.bases_free(h)


# ------------------------------------------------------------------------------------------ BN254: partial sums
def _cuts(n):
    """three uneven shards; only the first is below the 4096 points the pipelined schedule needs"""
    a = 1500
    b = a + (n - a) // 2 - 53
    return [(0, a), (a, b), (b, n)]


@pytest.mark.parametrize("g2", [False, True], ids=["g1", "g2"])
@pytest.mark.parametrize("table", [False, True], ids=["plain", "table"])
@pytest.mark.parametrize("n", [10007, (1 << 18) + 777])
def test_partial_resident_shards_fold_to_the_whole(ctx, g2, table, n):
    """b200zk_g{1,2}_msm_partial_resident (host scalars: the pipelined schedule, or the staged one-shot path below 4096
    points) and _partial_resident_device (device scalars: one shot): every shard on its own resident handle, the partials
    folded -- equal to the unsharded call and to the closed form"""
    import torch
    k, d = chain_kd()
    w, pw = (16, 32) if g2 else (8, 16)
    cuts = _cuts(n)
    assert [pipelined(hi - lo, host_scalars=True, g2=g2) for lo, hi in cuts] == [False, True, True]
    dp = dev_empty(w * n)
    (ctx.g2_chain_device if g2 else ctx.g1_chain_device)(dp, 0, n, k, d)
    s = np.ascontiguousarray(scalars_special(n, seed=n))
    ds = to_dev(s)
    exp = (expected_chain_msm_g2 if g2 else expected_chain_msm_g1)(s, k, d)
    assert (ctx.g2_msm_device if g2 else ctx.g1_msm_device)(dp, ds, n) == exp
    handles = []
    try:
        for lo, hi in cuts:
            handles.append((ctx.g2_bases_from_device if g2 else ctx.g1_bases_from_device)(dp[w * lo:w * hi], hi - lo))
            if table:
                ctx.bases_precompute(handles[-1], 0)
        fold = ctx.g2_fold_partials_device if g2 else ctx.g1_fold_partials_device
        parts = torch.zeros(pw * len(cuts), dtype=torch.int64, device="cuda")
        for r, (h, (lo, hi)) in enumerate(zip(handles, cuts)):
            fn = ctx.g2_msm_partial_resident if g2 else ctx.g1_msm_partial_resident
            fn(h, np.ascontiguousarray(s[lo:hi]), hi - lo, parts[pw * r:pw * (r + 1)])
        assert fold(parts, len(cuts)) == exp, "host scalars"
        parts.zero_()
        for r, (h, (lo, hi)) in enumerate(zip(handles, cuts)):
            fn = ctx.g2_msm_partial_resident_device if g2 else ctx.g1_msm_partial_resident_device
            fn(h, ds[lo:hi], hi - lo, parts[pw * r:pw * (r + 1)])  # ds: one row of four limbs per scalar
        assert fold(parts, len(cuts)) == exp, "device scalars"
    finally:
        for h in handles:
            ctx.bases_free(h)


def test_profiled_partial_resident_device_at_2_20(ctx):
    """bench.py's kernel-time call: g1_msm_partial_resident_device over a c = 20 window table at 2^20.  Profiling must not
    change the folded bytes, and last_msm_phase_ms must then report six finite, non-negative phase times"""
    import torch
    n = 1 << 20
    p = msm_plan(n, table_c=20)
    assert p.merged and p.two_level and not pipelined(n) and not pipelined(n, profiling=True)
    k, d = chain_kd()
    dp, ds = dev_empty(8 * n), dev_empty(4 * n)
    ctx.g1_chain_device(dp, 0, n, k, d)
    ctx.fr_random_device(ds, n, pyref.SEED_SCALARS, 0)
    exp = expected_chain_msm_g1(to_host(ds).reshape(n, 4), k, d)
    h = ctx.g1_bases_from_device(dp, n)
    del dp
    part = torch.zeros(16, dtype=torch.int64, device="cuda")
    try:
        ctx.bases_precompute(h, 20)
        ctx.g1_msm_partial_resident_device(h, ds, n, part)
        assert ctx.g1_fold_partials_device(part, 1) == exp
        part.zero_()
        ctx.set_profiling(True)
        ctx.g1_msm_partial_resident_device(h, ds, n, part)
        phases = ctx.last_msm_phase_ms()
        assert ctx.g1_fold_partials_device(part, 1) == exp
    finally:
        ctx.set_profiling(False)
        ctx.bases_free(h)
    assert len(phases) == 6 and all(math.isfinite(v) and v >= 0 for v in phases.values()), phases
    assert phases["accumulate"] > 0, phases


@pytest.mark.parametrize("g2", [False, True], ids=["g1", "g2"])
def test_profiled_host_scalar_msm_equals_the_pipelined_one(ctx, g2):
    """with profiling on, host scalars skip the pipeline and take the staged one-shot path: same bytes"""
    n = N_MID if not g2 else 20011
    assert pipelined(n, host_scalars=True, g2=g2) and not pipelined(n, host_scalars=True, profiling=True, g2=g2)
    k, d = chain_kd()
    w = 16 if g2 else 8
    dp = dev_empty(w * n)
    (ctx.g2_chain_device if g2 else ctx.g1_chain_device)(dp, 0, n, k, d)
    s = np.ascontiguousarray(scalars_special(n, seed=5))
    exp = (expected_chain_msm_g2 if g2 else expected_chain_msm_g1)(s, k, d)
    h = (ctx.g2_bases_from_device if g2 else ctx.g1_bases_from_device)(dp, n)
    fn = ctx.g2_msm_resident if g2 else ctx.g1_msm_resident
    try:
        assert fn(h, s, n) == exp
        ctx.set_profiling(True)
        assert fn(h, s, n) == exp
        assert ctx.last_msm_phase_ms()["accumulate"] > 0
    finally:
        ctx.set_profiling(False)
        ctx.bases_free(h)


# ------------------------------------------------------------------------------------------ BN254: SCALARS_RAW
def test_bn254_entry_points_refuse_scalars_raw(ctx):
    """B200ZK_SCALARS_RAW skips the reduction mod r, which BN254's signed-digit recoding needs: every BN254 MSM family
    refuses it with status 4 (host, device, async, resident, resident_device, partial, partial_resident in both scalar
    residencies, multi_resident), and the same calls without it succeed"""
    import torch
    n = 8
    k, d = chain_kd()
    s = np.ascontiguousarray(scalars_special(n))
    ds = to_dev(s)
    raw = F.SCALARS_RAW
    for g2 in (False, True):
        size = 128 if g2 else 64
        pts = (orc.g2_chain if g2 else orc.g1_chain)(n, k, d)
        exp = (orc.g2_msm if g2 else orc.g1_msm)(pts, s)
        dp = to_dev(pts)
        h = (ctx.g2_bases_upload if g2 else ctx.g1_bases_upload)(pts, n)
        out = torch.zeros(size // 8 + 1, dtype=torch.int64, device="cuda")
        part = torch.zeros(size // 4, dtype=torch.int64, device="cuda")
        pre = "g2_" if g2 else "g1_"
        calls = {
            "host": lambda f: getattr(ctx, pre + "msm")(pts, s, n, f),
            "device": lambda f: getattr(ctx, pre + "msm_device")(dp, ds, n, f),
            "async": lambda f: getattr(ctx, pre + "msm_device_async")(dp, ds, n, out, f),
            "resident": lambda f: getattr(ctx, pre + "msm_resident")(h, s, n, f),
            "resident_device": lambda f: getattr(ctx, pre + "msm_resident_device")(h, ds, n, f),
            "partial": lambda f: getattr(ctx, pre + "msm_partial_device")(dp, ds, n, part, f),
            "partial_resident": lambda f: getattr(ctx, pre + "msm_partial_resident")(h, s, n, part, f),
            "partial_resident_device": lambda f: getattr(ctx, pre + "msm_partial_resident_device")(h, ds, n, part, f),
            "multi_resident": lambda f: ctx.msm_multi_resident_device([h], [g2], ds, n, f)[0],
        }
        try:
            for name, call in calls.items():
                for flags in (raw, raw | eb.SCALARS_BE, raw | eb.SCALARS_MONT):
                    with pytest.raises(eb.B200Error) as e:
                        call(flags)
                    assert e.value.status == 4, (g2, name, flags)
            assert calls["device"](0) == exp and calls["host"](0) == exp and calls["multi_resident"](0) == exp
            calls["partial_resident"](0)
            assert (ctx.g2_fold_partials_device if g2 else ctx.g1_fold_partials_device)(part, 1) == exp
        finally:
            ctx.bases_free(h)
