"""The Fr NTT at every size from 2^0 to 2^28 in every mode, and the Groth16 quotient chain at the prover's domain sizes.

The transform's plan changes with the size: one pass up to 2^12, two up to 2^20, three above; the last pass's inter-pass
twiddles come from the 2^16-entry table (2^13..2^16), the direct N-entry table (2^17..2^26, unless B200ZK_NTT_FULL_TW says
otherwise) or the two-level tables (2^27, 2^28, where n^-1 rides on lo_n); stage counts per pass are odd or even, the tile
width changes, and the coset tables gain a high part above 2^12.  Running every size is the only way to reach every
combination, now and after the next schedule change.

Up to 2^24 every output is compared with the CPU oracle's transform.  From 2^25 the oracle's O(n) whole-vector identity
(cpu_oracle.NttIdentity) checks the output chunk by chunk against the input the host regenerates, so no vector is ever
held whole on the host.  Every size also gets a bit-exact round trip on the device and three outputs of the forward
transform evaluated from the definition.

From 2^23 each size runs in a Context of its own, closed afterwards: the twiddle cache never evicts, and one direct table
at 2^26 is 2 GiB."""
import contextlib

import numpy as np
import pytest

import cpu_oracle as orc
import pyref
from helpers import dev_empty, to_dev, to_host

pytestmark = pytest.mark.gpu

import ethrex_b200 as eb  # noqa: E402

HALO2_ROOT = pow(7, (pyref.R - 1) >> 28, pyref.R)
SEED = pyref.SEED_NTT
CHUNK = 1 << 22          # host chunk of the whole-vector checks (128 MiB of input and of output)
ELEMENTWISE_MAX = 24     # above this, the oracle's own transform is too slow: the identity checks instead
OWN_CONTEXT_FROM = 23
# (device flags, coset generator): forward, inverse, coset and inverse coset with the default generator 5, then both coset
# directions with a caller's generator
MODES = [(0, None), (eb.NTT_INVERSE, None), (eb.NTT_COSET, None), (eb.NTT_INVERSE | eb.NTT_COSET, None),
         (eb.NTT_COSET, 7), (eb.NTT_INVERSE | eb.NTT_COSET, pyref.R - 3)]
_PEAK = {"used": 0}


def _oflags(flags):
    return (orc.NTT_INVERSE if flags & eb.NTT_INVERSE else 0) | (orc.NTT_COSET if flags & eb.NTT_COSET else 0)


def _gen(gen, big_endian=False):
    return None if gen is None else gen.to_bytes(32, "big" if big_endian else "little")


def _sample_memory():
    import torch
    free, total = torch.cuda.mem_get_info()
    _PEAK["used"] = max(_PEAK["used"], total - free)


@pytest.fixture(scope="module", autouse=True)
def _report_peak_memory():
    yield
    if _PEAK["used"]:
        print(f"\ntest_gpu_ntt_sweep: peak device memory in use (mem_get_info, whole device) {_PEAK['used'] / 2**30:.2f} GiB")


@contextlib.contextmanager
def _context(ctx, log_n):
    """the session context below 2^23, a context of its own (closed afterwards) from there up"""
    import torch
    if log_n < OWN_CONTEXT_FROM:
        yield ctx
        return
    c = eb.Context(0)
    try:
        yield c
    finally:
        c.close()
        torch.cuda.empty_cache()


@contextlib.contextmanager
def _root(c, root):
    if root is None:
        yield
        return
    c.set_ntt_root(root.to_bytes(32, "little"))
    try:
        yield
    finally:
        c.set_ntt_root(None)


def _set_knob(monkeypatch, knob):
    if knob is None:
        monkeypatch.delenv("B200ZK_NTT_FULL_TW", raising=False)
    else:
        monkeypatch.setenv("B200ZK_NTT_FULL_TW", knob)


def _need_free_device_memory(nbytes, what):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"{what} needs {nbytes / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB are free")


def _eval_points(n):
    return sorted({1 % n, n - 1, (0x9E3779B97F4A7C15 >> 3) % n})


def _to_int(row_mont):
    return orc.limbs_to_int(orc.fr_from_mont(row_mont.reshape(1, 4))[0])


def _sweep_elementwise(c, log_n, root, knobs, monkeypatch):
    n = 1 << log_n
    a = orc.fr_to_mont(orc.rand_fr(SEED, 0, n))
    for flags, gen in MODES:
        exp = orc.fr_ntt(a, log_n, _oflags(flags), coset_gen=gen, root_2_28=root)
        for knob in knobs:
            _set_knob(monkeypatch, knob)
            what = f"log_n={log_n} flags={flags} gen={gen} root={root} B200ZK_NTT_FULL_TW={knob}"
            d = to_dev(a)
            c.fr_ntt_device(d, log_n, flags, _gen(gen))
            got = to_host(d).reshape(n, 4)
            assert (got == exp).all(), what
            if root is None and flags == 0 and knob == knobs[0]:
                for k in _eval_points(n):
                    assert (orc.fr_ntt_eval_output(a, log_n, k) == got[k]).all(), (what, k)
            if not flags & eb.NTT_INVERSE:
                c.fr_ntt_device(d, log_n, flags | eb.NTT_INVERSE, _gen(gen))
                assert (to_host(d).reshape(n, 4) == a).all(), (what, "round trip")
            del d


def _sweep_by_identity(c, log_n, root, knobs, monkeypatch):
    import torch
    n = 1 << log_n
    # data and workspace, plus up to three direct tables (forward, inverse with n^-1 folded, inverse without) up to 2^26
    tables = 3 * n * 32 if log_n <= 26 else 0
    _need_free_device_memory(2 * n * 32 + tables + (2 << 30), f"the 2^{log_n} NTT")
    d, ref = dev_empty(4 * n), dev_empty(4 * CHUNK)
    for flags, gen in MODES:
        for knob in knobs:
            _set_knob(monkeypatch, knob)
            what = f"log_n={log_n} flags={flags} gen={gen} root={root} B200ZK_NTT_FULL_TW={knob}"
            c.fr_random_device(d, n, SEED, 0, eb.SCALARS_MONT)
            c.fr_ntt_device(d, log_n, flags, _gen(gen))
            chk = orc.NttIdentity(log_n, _oflags(flags), gen, root)
            ks = _eval_points(n) if root is None and flags == 0 and knob == knobs[0] else []
            sums, outs = dict.fromkeys(ks, 0), {}
            for s in range(0, n, CHUNK):
                a = orc.fr_to_mont(orc.rand_fr(SEED, s, CHUNK))  # the input fr_random_device wrote, chunk by chunk
                y = to_host(d[4 * s:4 * (s + CHUNK)]).reshape(CHUNK, 4)
                chk.update(a, y, s)
                for k in ks:
                    sums[k] += orc.fr_ntt_eval_output_chunk(a, s, log_n, k)
                    if s <= k < s + CHUNK:
                        outs[k] = _to_int(y[k - s])
            _sample_memory()
            assert chk.ok(), what
            for k in ks:
                assert sums[k] % pyref.R == outs[k], (what, k)
            if not flags & eb.NTT_INVERSE:
                c.fr_ntt_device(d, log_n, flags | eb.NTT_INVERSE, _gen(gen))
                for s in range(0, n, CHUNK):
                    c.fr_random_device(ref, CHUNK, SEED, s, eb.SCALARS_MONT)
                    assert torch.equal(d[4 * s:4 * (s + CHUNK)], ref), (what, "round trip", s)
    del d, ref


def _sweep(ctx, log_n, root, knobs, monkeypatch):
    with _context(ctx, log_n) as c, _root(c, root):
        if log_n <= ELEMENTWISE_MAX:
            _sweep_elementwise(c, log_n, root, knobs, monkeypatch)
        else:
            _sweep_by_identity(c, log_n, root, knobs, monkeypatch)
        _sample_memory()


# ------------------------------------------------------------------------------------------ every size, every mode
@pytest.mark.parametrize("log_n", list(range(0, 29)))
def test_ntt_every_size_every_mode(ctx, log_n, monkeypatch):
    """Six modes at 2^log_n under the default root.  Sizes with a direct last-pass table (2^17..2^26) also run with it
    turned off (B200ZK_NTT_FULL_TW=0), so both last-pass twiddle sources are checked at each."""
    knobs = (None, "0") if 17 <= log_n <= 26 else (None,)
    _sweep(ctx, log_n, None, knobs, monkeypatch)


@pytest.mark.parametrize("log_n", [11, 12, 13, 16, 17, 21, 24, 27])
def test_ntt_halo2_root_every_plan_shape(ctx, log_n, monkeypatch):
    """halo2curves' root 7^((r-1)/2^28) in six modes at one size per plan shape: one pass; one pass with the largest
    stage; two passes on the 2^16 table; two passes with a direct table; three passes with a direct table; 2^24, the
    prover's size; three passes on the two-level tables."""
    _sweep(ctx, log_n, HALO2_ROOT, (None,), monkeypatch)


# ------------------------------------------------------------------------------------------ canonical and big-endian data
def _canonical_input_with_edges(log_n):
    n = 1 << log_n
    vals = orc.rand_fr(SEED ^ 0xCA, 0, n)
    low192, low224 = pyref.R & ((1 << 192) - 1), pyref.R & ((1 << 224) - 1)
    rnd = orc.array_to_ints(orc.rand_fr(SEED ^ 0xED, 0, 4))
    # 0, 1, r - 1, r - 2; values whose top 64-bit limb (and top 32-bit word) equals r's
    edges = [0, 1, pyref.R - 1, pyref.R - 2, pyref.R - low192, pyref.R - 1 - rnd[0] % low192, pyref.R - 1 - rnd[1] % low192,
             pyref.R - 1 - rnd[2] % low224, pyref.R - low224]
    # at the front, in the middle, and at the end (the second turn of the grid-stride conversion from 2^21 up)
    for i, v in enumerate(edges):
        for pos in (i, n // 2 + i, n - 1 - i):
            vals[pos] = orc.int_to_limbs(v)
    assert all(v < pyref.R for v in orc.array_to_ints(vals[:len(edges)]))
    return vals


def _be_bytes(canon):
    return np.ascontiguousarray(canon[:, ::-1]).astype(">u8").tobytes()


@pytest.mark.parametrize("log_n", [13, 21, 22])
def test_ntt_canonical_and_big_endian_data(ctx, log_n):
    """NTT_CANONICAL (little-endian limbs) and NTT_BE (32-byte big-endian values) in six modes, with the custom coset
    generator given big-endian under NTT_BE: the outputs must be the oracle's canonical bytes.  The conversions run a
    grid capped at 32 CTAs per SM, so from 2^21 up their grid-stride loop takes a second turn."""
    n = 1 << log_n
    canon = _canonical_input_with_edges(log_n)
    mont = orc.fr_to_mont(canon)
    be_in = np.frombuffer(_be_bytes(canon), dtype=np.uint64)
    for flags, gen in MODES:
        exp = orc.fr_from_mont(orc.fr_ntt(mont, log_n, _oflags(flags), coset_gen=gen))
        d = to_dev(canon)
        ctx.fr_ntt_device(d, log_n, flags | eb.NTT_CANONICAL, _gen(gen))
        assert (to_host(d).reshape(n, 4) == exp).all(), (log_n, flags, gen, "canonical")
        d = to_dev(be_in)
        ctx.fr_ntt_device(d, log_n, flags | eb.NTT_BE, _gen(gen, big_endian=True))
        assert to_host(d).tobytes() == _be_bytes(exp), (log_n, flags, gen, "big-endian")


# ------------------------------------------------------------------------------------------ buffer offsets
@pytest.mark.parametrize("log_n", [12, 13, 21])
def test_ntt_on_a_buffer_offset_inside_a_larger_allocation(ctx, log_n):
    """Data 16, 32 and 4096 bytes into an allocation: 16-byte aligned but not 256-byte aligned, the bulk copies' smallest
    legal alignment.  2^12 loads each tile with one bulk copy, 2^13 and 2^21 with one per row.  The sentinel words on both
    sides must come out untouched."""
    import torch
    n = 1 << log_n
    a = orc.fr_to_mont(orc.rand_fr(SEED ^ 0x0F, 0, n))
    sentinel = 0x5A5A_A5A5_0F0F_F0F0
    pad = 4096 // 8 + 64
    for flags, gen in MODES:
        exp = orc.fr_ntt(a, log_n, _oflags(flags), coset_gen=gen)
        for off in (16, 32, 4096):
            w = off // 8
            buf = torch.full((pad + 4 * n + pad,), sentinel, dtype=torch.int64, device="cuda")
            view = buf[w:w + 4 * n]
            view.copy_(to_dev(a).reshape(-1))
            assert view.data_ptr() % 256 == off % 256
            ctx.fr_ntt_device(view, log_n, flags, _gen(gen))
            assert (to_host(view).reshape(n, 4) == exp).all(), (log_n, flags, gen, off)
            assert bool((buf[:w] == sentinel).all()) and bool((buf[w + 4 * n:] == sentinel).all()), (log_n, flags, gen, off)


# ------------------------------------------------------------------------------------------ table caches
@pytest.mark.parametrize("log_n", [20, 24])
def test_ntt_table_caches_interleaved_without_synchronising(ctx, log_n):
    """Cached twiddle and coset tables are keyed by size, direction, root and generator: default root, halo2's root,
    default root again, and coset generator 5, 7, 5 again, each in both directions and enqueued back to back, must each
    use their own tables."""
    n = 1 << log_n
    a = orc.fr_to_mont(orc.rand_fr(SEED ^ 0xCC, 0, n))
    with _context(ctx, log_n) as c:
        for direction in (0, eb.NTT_INVERSE):
            bufs = [to_dev(a) for _ in range(3)]
            try:
                c.fr_ntt_device(bufs[0], log_n, direction)
                c.set_ntt_root(HALO2_ROOT.to_bytes(32, "little"))
                c.fr_ntt_device(bufs[1], log_n, direction)
            finally:
                c.set_ntt_root(None)
            c.fr_ntt_device(bufs[2], log_n, direction)
            exp_default = orc.fr_ntt(a, log_n, _oflags(direction))
            exp_halo2 = orc.fr_ntt(a, log_n, _oflags(direction), root_2_28=HALO2_ROOT)
            for b, exp, name in ((bufs[0], exp_default, "default"), (bufs[1], exp_halo2, "halo2"), (bufs[2], exp_default, "default again")):
                assert (to_host(b).reshape(n, 4) == exp).all(), (log_n, direction, name)
            del bufs
        for direction in (eb.NTT_COSET, eb.NTT_COSET | eb.NTT_INVERSE):
            bufs = [to_dev(a) for _ in range(3)]
            for b, g in zip(bufs, (5, 7, 5)):
                c.fr_ntt_device(b, log_n, direction, _gen(g))
            for b, g in zip(bufs, (5, 7, 5)):
                assert (to_host(b).reshape(n, 4) == orc.fr_ntt(a, log_n, _oflags(direction), coset_gen=g)).all(), (log_n, direction, g)
            del bufs
        _sample_memory()


def test_ntt_tables_built_on_one_stream_are_waited_for_on_another(ctx):
    """A table built on first use on one stream carries a build event: a transform enqueued at once on another stream
    must wait for it.  2^12 runs in one pass in place, so the two streams share no scratch buffer; a fresh context builds
    every table (twiddles per direction, coset powers per direction and generator) on first use."""
    import torch
    log_n, n = 12, 1 << 12
    a = orc.fr_to_mont(orc.rand_fr(SEED ^ 0x5E, 0, n))
    with eb.Context(0) as c:
        builder, consumer = torch.cuda.Stream(), torch.cuda.Stream()
        bufs = [(to_dev(a), to_dev(a)) for _ in MODES]
        builder.wait_stream(torch.cuda.current_stream())
        consumer.wait_stream(torch.cuda.current_stream())
        for (b1, b2), (flags, gen) in zip(bufs, MODES):
            with torch.cuda.stream(builder):
                c.fr_ntt_device(b1, log_n, flags, _gen(gen))
            with torch.cuda.stream(consumer):
                c.fr_ntt_device(b2, log_n, flags, _gen(gen))
        torch.cuda.synchronize()
        for (b1, b2), (flags, gen) in zip(bufs, MODES):
            exp = orc.fr_ntt(a, log_n, _oflags(flags), coset_gen=gen)
            assert (to_host(b1).reshape(n, 4) == exp).all(), (flags, gen, "builder")
            assert (to_host(b2).reshape(n, 4) == exp).all(), (flags, gen, "consumer")


# ------------------------------------------------------------------------------------------ Groth16 quotient chain
def _quotient_chain(c, log_n, evals, zinv):
    """the prover's quotient: 3 x (iNTT, coset NTT with generator 5), (a*b - c) * zinv in place over a, coset iNTT"""
    d = [to_dev(x) for x in evals]
    for p in d:
        c.fr_ntt_device(p, log_n, eb.NTT_INVERSE)
        c.fr_ntt_device(p, log_n, eb.NTT_COSET)
    c.fr_quotient_device(d[0], d[1], d[2], d[0], 1 << log_n, zinv)
    c.fr_ntt_device(d[0], log_n, eb.NTT_INVERSE | eb.NTT_COSET)
    return to_host(d[0]).reshape(-1, 4)


@pytest.mark.parametrize("log_n", [22, 24])
def test_groth16_quotient_chain_at_prover_sizes(ctx, log_n):
    """With random a, b, c the chain equals the oracle's element for element; with c = a * b pointwise the quotient is
    exact, of degree at most n - 2, so its top coefficient is zero."""
    n = 1 << log_n
    zinv = pow((pow(5, n, pyref.R) - 1) % pyref.R, -1, pyref.R)
    a, b, cc = (orc.fr_to_mont(orc.rand_fr(SEED ^ (0x9A + i), 0, n)) for i in range(3))
    with _context(ctx, log_n) as c:
        got = _quotient_chain(c, log_n, (a, b, cc), zinv)
        _sample_memory()
        co = [orc.fr_ntt(orc.fr_ntt(x, log_n, orc.NTT_INVERSE), log_n, orc.NTT_COSET) for x in (a, b, cc)]
        exp = orc.fr_ntt(orc.fr_quotient(co[0], co[1], co[2], zinv), log_n, orc.NTT_INVERSE | orc.NTT_COSET)
        del co
        assert (got == exp).all()
        h = _quotient_chain(c, log_n, (a, b, orc.field_mul("fr", a, b)), zinv)
        assert not h[n - 1].any(), "h[n - 1] != 0: the quotient of a satisfied system is not exact"
        assert h.any()
