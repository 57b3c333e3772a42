"""CPU checks of the bigmod.cuh suite (tests/test_gpu_bigmod_conformance.py) and of the carry machinery it tests.

The limb-exact model of tests/bigmod_ref.py (per-lane rows, pending words, the final fold, the generate / propagate
`resolve`, cond_sub) must equal the integer model on the edge values and on random inputs, and must stay inside the
header's bounds on every input: a pending word below 4, t < 2m before cond_sub.  The edge values must reach every carry
event the header's mechanisms exist for, which random operands almost never reach: a test per event names the one a later
edit stops reaching.  Each named mutant of the model (one mechanism broken) must be caught by the edge values; the
final-resolve mutant is also shown to pass every random product, which is why the edge values exist.  Last, the device
harness must list a kernel for every width in its ptxas report and use the op ids of the model."""
import functools
import os
import random
import re
import subprocess

import pytest

import bigmod_ref as ref

HERE = os.path.dirname(os.path.abspath(__file__))
HARNESS = os.path.join(HERE, "csrc", "bigmod_conformance.cu")
MODEL_WIDTHS = (8, 32, 64)  # 1, 4 and 8 lanes
EVENT_WIDTHS = (32, 64)     # 4 and 8 lanes; 32 lanes on ref.probe_tuples below
N_RANDOM = 300


def _run(N, items, ev):
    """the limb model over (op, operands) items: the items whose result differs from the integer model"""
    bad = []
    for op, xs in items:
        assert ref.in_domain(N, op, xs), (N, op, [hex(x) for x in xs])
        if op == "mont_mul":
            got = ref.model_mont_mul(N, *xs, ev=ev)
        elif op == "cond_sub":
            t, m, hi = xs
            got = ref.model_cond_sub(N, t, hi, m, ev)
        elif op == "add":
            got = ref.model_add(N, *xs, ev)
        else:
            got = ref.model_sub(N, *xs, ev)
        want = ref.expect(N, op, xs)
        if got != (want if op in ("add", "sub") else want[0]):
            bad.append((op, xs))
    return bad


def edge_model_items(N):
    V = ref.values(N)
    return ([("mont_mul", it) for it in ref.mont_edges(N)] + [("cond_sub", it) for it in ref.cond_sub_edges(N)]
            + [(op, (a, b)) for op in ("add", "sub") for a in V for b in V])


def random_model_items(N, seed):
    rng = random.Random(f"{seed}/{N}")
    return [(op, it) for op in ("mont_mul", "cond_sub", "add", "sub") for it in ref.random_items(N, op, rng, N_RANDOM)]


@functools.lru_cache(maxsize=None)
def edge_run(N):
    ev = set()
    bad = _run(N, edge_model_items(N), ev)
    return frozenset(ev), bad


@pytest.mark.parametrize("N", MODEL_WIDTHS)
def test_limb_model_equals_integers_on_edges(N):
    ev, bad = edge_run(N)
    assert not bad, f"N = {N}: {len(bad)} edge items differ, first {bad[0][0]} {[hex(x) for x in bad[0][1]]}"
    assert not ev & set(ref.VIOLATIONS), f"N = {N}: the header's bounds broken: {sorted(ev & set(ref.VIOLATIONS))}"


@pytest.mark.parametrize("N", MODEL_WIDTHS)
def test_limb_model_equals_integers_on_random(N):
    ev = set()
    bad = _run(N, random_model_items(N, "model"), ev)
    assert not bad, f"N = {N}: {len(bad)} random items differ, first {bad[0][0]} {[hex(x) for x in bad[0][1]]}"
    assert not ev & set(ref.VIOLATIONS), f"N = {N}: the header's bounds broken: {sorted(ev & set(ref.VIOLATIONS))}"


@pytest.mark.parametrize("N,event", [(N, e) for N in EVENT_WIDTHS for e in ref.EVENTS],
                         ids=[f"{N // 8}lanes-{e}" for N in EVENT_WIDTHS for e in ref.EVENTS])
def test_edges_reach_event(N, event):
    ev, _ = edge_run(N)
    assert event in ev, f"{N // 8} lanes: no edge item reaches {event}"


@functools.lru_cache(maxsize=None)
def probe_run(N):
    ev = set()
    V = ref.chain_values(N) + [0, 1]
    items = [("mont_mul", it) for it in ref.probe_tuples(N)] + [(op, (a, b)) for op in ("add", "sub") for a in V for b in V]
    bad = _run(N, items, ev)
    return frozenset(ev), bad


@pytest.mark.parametrize("event", ref.EVENTS)
def test_probe_tuples_reach_event_at_32_lanes(event):
    ev, bad = probe_run(256)
    assert not bad and not ev & set(ref.VIOLATIONS)
    assert event in ev, f"32 lanes: no probe tuple reaches {event}"


def mutant_catches(N, mutant, items):
    """the first item on which the mutant's result differs from the integer model, or None"""
    for op, xs in items:
        if op == "mont_mul":
            got = ref.model_mont_mul(N, *xs, mutant=mutant)
        elif op == "cond_sub":
            t, m, hi = xs
            got = ref.model_cond_sub(N, t, hi, m, mutant=mutant)
        else:
            continue
        if got != ref.expect(N, op, xs)[0]:
            return op, xs
    return None


@pytest.mark.parametrize("N,mutant", [(N, mu) for N in EVENT_WIDTHS for mu in ref.MUTANTS],
                         ids=[f"{N // 8}lanes-{mu}" for N in EVENT_WIDTHS for mu in ref.MUTANTS])
def test_edges_catch_mutant(N, mutant):
    assert mutant_catches(N, mutant, edge_model_items(N)) is not None, f"{N // 8} lanes: the edge items miss mutant {mutant}"


@pytest.mark.parametrize("N", EVENT_WIDTHS)
def test_random_inputs_miss_the_resolve_mutant(N):
    """the final resolve without its propagate bits gives the right answer on every random product"""
    items = random_model_items(N, "model")
    assert mutant_catches(N, "resolve_no_propagate", items) is None
    assert mutant_catches(N, "resolve_no_propagate", [("mont_mul", it) for it in ref.probe_tuples(N)]) is not None


@pytest.mark.parametrize("N", ref.WIDTHS)
def test_edge_and_random_items_inside_domain(N):
    rng = random.Random(N)
    for op in ref.OPS:
        items = ref.edge_items(N, op) + ref.random_items(N, op, rng, 64)
        assert items and len(set(items)) > len(items) // 2, op
        for xs in items:
            assert len(xs) == ref.ARITY[op] and ref.in_domain(N, op, xs), (N, op, [hex(x) for x in xs])
    R = ref.R_of(N)
    ms = ref.moduli(N)
    assert {3, R - 1, R - 3, R // 2 + 1, (1 << (32 * N - 32)) + 1} <= set(ms)
    assert all(0 < m < R for m in ms) and len(set(ms)) == len(ms)
    assert ref.chain_values(N)[-1] == R - 1


def test_integer_model_against_formulas():
    rng = random.Random(7)
    for N in ref.WIDTHS:
        R = ref.R_of(N)
        m = ref.random_modulus(rng, N, odd=True)
        a, b = rng.randrange(m), rng.randrange(m)
        for x, y in ((a, b), (R - 1, b), (a, m - 1), (R - 1, m - 1), (0, b)):
            assert ref.expect(N, "mont_mul", (x, y, m)) == (x * y * pow(R, -1, m) % m, 0)
        for q in (1, R - 1, rng.getrandbits(32 * N) | 1):
            assert ref.expect(N, "inv_mod_r", (q,)) == (pow(q, -1, R), 0)
        assert ref.expect(N, "add", (R - 1, 1)) == (0, 1) and ref.expect(N, "sub", (0, 1)) == (R - 1, 1)
        assert ref.expect(N, "cond_sub", (0, R - 1, 1)) == (1, 0)  # t + hi R = R = m + 1
    x = 0x12345679
    assert (ref.expect(8, "neg_inv32", (x,))[1] * x + 1) % (1 << 32) == 0


def test_harness_ids_match_model():
    src = open(HARNESS).read()
    m = re.search(r"enum : int \{ B_ADD = 0,([^}]*)\}", src)
    ids = ["B_ADD"] + [t.strip() for t in m.group(1).split(",") if t.strip()]
    assert [i[2:].lower() for i in ids[:-1]] == ref.OPS and ids[-1] == "N_BIGMOD_OPS"
    modexp = open(os.path.join(HERE, "..", "ethrex_b200", "csrc", "modexp.cu")).read()
    # the widths and the block size modexp.cu launches
    assert re.search(r"kClassLimbs\[kClasses\] = \{([^}]*)\}", modexp).group(1).replace(" ", "") == ",".join(map(str, ref.WIDTHS))
    assert re.search(r"kModexpThreads = (\d+);", modexp).group(1) == re.search(r"constexpr int kThreads = (\d+);", src).group(1)


def test_harness_lists_every_width():
    """build() leaves tests/build/libb200zk_conformance.so and its ptxas report: one bigmod kernel per width, exported
    launcher"""
    log = os.path.join(HERE, "build", "conformance.ptxas.log")
    lib = os.path.join(HERE, "build", "libb200zk_conformance.so")
    if not os.path.exists(log) or not os.path.exists(lib):
        pytest.skip("the conformance harness is not built")
    text = open(log).read()
    for N in ref.WIDTHS:
        assert re.search(rf"Function properties for \w*bigmod_kernelILi{N}ELi{N // 8}EE\w*\n\s*\d+ bytes stack frame", text), N
    syms = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    assert re.search(r"\bT b200zk_bigmod_conformance_run\b", syms)
