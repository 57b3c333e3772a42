"""Every primitive of bigmod.cuh on the device against Python integers, at every width modexp.cu instantiates and at the
lane edges where carries and borrows cross lanes.

tests/csrc/bigmod_conformance.cu runs one item per group of TPI = N / 8 lanes in blocks of 64 threads, as modexp.cu does;
tests/bigmod_ref.py holds the integer model, the edge values and the documented domain of each op.  Each (op, width)
compares bit for bit: binary ops over the full cross product of their edges, wider ops over edge tuples (every edge
modulus with its edge operands), plus 2^12 random tuples.  Each item carries its own op id, so one launch can give the
groups of a warp different primitives with different shuffle sequences under their own masks; and item counts that end
inside a warp leave trailing groups to return early, as in modexp_kernel.  Every op that returns a scalar must return it
on every lane of the group.  A failure names the width, the op and the operands in hex."""
import ctypes
import os
import random

import numpy as np
import pytest

import bigmod_ref as ref

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "build", "libb200zk_conformance.so")
N_RANDOM = 1 << 12
SENTINEL = 0xa5a5a5a5  # the output rows past the last item, which no group may write
MULTI_LANE = [N for N in ref.WIDTHS if N > 8]


def pack(vals, words):
    """ints -> uint32 array (len(vals), words), little-endian limbs"""
    return np.frombuffer(b"".join(v.to_bytes(4 * words, "little") for v in vals), dtype="<u4").reshape(len(vals), words)


def unpack(arr):
    arr = np.ascontiguousarray(arr, dtype="<u4")
    step = 4 * arr.shape[1]
    buf = arr.tobytes()
    return [int.from_bytes(buf[i:i + step], "little") for i in range(0, len(buf), step)]


@pytest.fixture(scope="module")
def harness():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    assert os.path.exists(LIB), f"{LIB} is missing: run __graft_entry__.build() first"
    torch.cuda.set_device(0)
    fn = ctypes.CDLL(LIB).b200zk_bigmod_conformance_run
    fn.argtypes = [ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64]
    fn.restype = ctypes.c_int

    def run(N, items, extra=0):
        """items: (op, operands) pairs of width N; returns uint32 (n, N + 2): the number, the scalar, the lanes whose
        scalar differs from lane 0's.  `extra` sentinel rows past the last item must come back untouched."""
        n = len(items)
        arr = np.zeros((n, 1 + 3 * N), dtype=np.uint32)
        arr[:, 0] = [ref.OP[op] for op, _ in items]
        for k in range(3):
            arr[:, 1 + k * N:1 + (k + 1) * N] = pack([xs[k] if k < len(xs) else 0 for _, xs in items], N)
        out = np.zeros((n + extra, N + 2), dtype=np.uint32)
        out[n:] = SENTINEL
        d_in = torch.from_numpy(arr.view(np.int32)).cuda()
        d_out = torch.from_numpy(out.view(np.int32)).cuda()
        rc = fn(N, d_in.data_ptr(), d_out.data_ptr(), n)
        assert rc == 0, f"b200zk_bigmod_conformance_run(N = {N}, n = {n}) returned {rc}"
        got = d_out.cpu().numpy().view(np.uint32)
        assert (got[n:] == SENTINEL).all(), f"N = {N}, n = {n}: a group wrote past the last item"
        return got[:n]
    return run


def check(harness, N, items, what, extra=0):
    """runs (op, operands) items and compares each with the integer model: the number, the scalar, and that every lane
    of the group holds the same scalar"""
    for op, xs in items:
        assert ref.in_domain(N, op, xs), (N, op, [hex(x) for x in xs])
    out = harness(N, items, extra)
    got = list(zip(unpack(out[:, :N]), (int(v) for v in out[:, N]), (int(v) for v in out[:, N + 1])))
    exp = [ref.expect(N, op, xs) + (0,) for op, xs in items]
    bad = [i for i, (g, e) in enumerate(zip(got, exp)) if g != e]
    if bad:
        lines = [f"  {items[i][0]}({', '.join(hex(x) for x in items[i][1])}): got {hex(got[i][0])}, scalar "
                 f"{hex(got[i][1])} ({got[i][2]} lanes disagree), expected {hex(exp[i][0])}, scalar {hex(exp[i][1])}"
                 for i in bad[:5]]
        raise AssertionError(f"N = {N} ({N // 8} lanes) {what}: {len(bad)} of {len(items)} results differ\n" + "\n".join(lines))


CASES = [(N, op) for N in ref.WIDTHS for op in ref.OPS]


@pytest.mark.parametrize("N,op", CASES, ids=[f"{N // 8}lanes-{op}" for N, op in CASES])
def test_op(harness, N, op):
    rng = random.Random(f"bigmod/{N}/{op}")
    items = ref.edge_items(N, op) + ref.random_items(N, op, rng, N_RANDOM)
    check(harness, N, [(op, xs) for xs in items], op)


def mixed_items(N, rng, per_op):
    """per_op items of every op, random and edge, shuffled so that neighbouring groups run different primitives"""
    items = []
    for op in ref.OPS:
        edges = ref.edge_items(N, op)
        picked = ref.random_items(N, op, rng, per_op // 2) + rng.sample(edges, min(len(edges), per_op - per_op // 2))
        items += [(op, xs) for xs in picked]
    rng.shuffle(items)
    return items


@pytest.mark.parametrize("N", MULTI_LANE, ids=[f"{N // 8}lanes" for N in MULTI_LANE])
def test_mixed_ops_in_one_launch(harness, N):
    items = mixed_items(N, random.Random(f"bigmod/mixed/{N}"), 64)
    assert sum(a[0] != b[0] for a, b in zip(items, items[1:])) > len(items) * 3 // 4
    check(harness, N, items, "mixed-op launch")


@pytest.mark.parametrize("N", MULTI_LANE, ids=[f"{N // 8}lanes" for N in MULTI_LANE])
def test_partial_warps(harness, N):
    """item counts that end inside a warp (inside a block at 32 lanes), with every op before the last groups and the
    products that fold carries through every lane in them"""
    tpi = N // 8
    per_warp, per_block = 32 // tpi, 64 // tpi
    partial = (lambda c: c * tpi % 32 != 0) if tpi < 32 else (lambda c: c % 2 == 1)
    counts = (1, 3, per_warp - 1, per_warp + 1, per_block + 1, 5 * per_block - 1, 5 * per_block + per_warp + 1)
    counts = [c for c in dict.fromkeys(counts) if c > 0 and partial(c)]
    assert len(counts) >= 3
    rng = random.Random(f"bigmod/partial/{N}")
    pool = mixed_items(N, rng, 8)
    tail = [("mont_mul", it) for it in ref.probe_tuples(N)]
    for c in counts:
        items = ([pool[(c + i) % len(pool)] for i in range(c)] + tail)[-c:]
        check(harness, N, items, f"{c} items", extra=per_block + 1)
