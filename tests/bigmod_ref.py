"""bigmod.cuh in Python: the integer result and the documented domain of every primitive, the edge values of each width,
and a limb-exact model of the carry machinery (add, sub, cond_sub, mont_mul) that reports which carry events an input
reaches.

A number of N 32-bit limbs lives on TPI = N / 8 lanes, 256 bits per lane; R = 2^(32N).  The model keeps one Python
integer per lane and follows the header step by step: per-lane rows whose carries stay pending at the upper neighbour's
limb 0, the fold of the pending words after the last round, and the generate / propagate ballot of `resolve`.  Its
mutants are the header with one mechanism broken, so tests/test_bigmod_model.py can show that the edge values (and not
only random ones) tell the difference.

Shared by tests/test_bigmod_model.py (the model, on the CPU) and tests/test_gpu_bigmod_conformance.py (the device
harness tests/csrc/bigmod_conformance.cu against the integer model)."""
import functools
import random

WIDTHS = (8, 32, 64, 128, 256)  # N limbs, as modexp.cu instantiates them; TPI = N / 8
LANE_BITS = 256
M32 = (1 << 32) - 1
M256 = (1 << LANE_BITS) - 1

# ids of tests/csrc/bigmod_conformance.cu
OPS = ["add", "sub", "mod_add", "mod_dbl", "cond_sub", "mont_mul", "lo_mul", "inv_mod_r", "truncate_bits", "is_zero", "is_one",
       "neg_inv32"]
OP = {name: i for i, name in enumerate(OPS)}
# operands in harness slot order; m comes last where there is one, cond_sub's hi after m
ARITY = {"add": 2, "sub": 2, "mod_add": 3, "mod_dbl": 2, "cond_sub": 3, "mont_mul": 3, "lo_mul": 2, "inv_mod_r": 1,
         "truncate_bits": 2, "is_zero": 1, "is_one": 1, "neg_inv32": 1}

# mechanisms the header must have, each broken once (tests/test_bigmod_model.py)
MUTANTS = ["resolve_no_propagate",  # mont_mul's final resolve: carry-in bits C = G << 1
           "fold_dropped",          # mont_mul: the pending words never added to the upper neighbours
           "cond_sub_ignores_hi",   # cond_sub keeps t - m only when it does not borrow
           "from_below_two_lanes",  # from_below reads lane - 2
           "from_below_own_lane",   # from_below reads the lane itself
           "from_above_two_lanes",  # from_above reads lane + 2
           "from_above_own_lane"]   # from_above reads the lane itself

# carry events the edge values must reach at 4 and 8 lanes (tests/test_bigmod_model.py); "mont." are inside mont_mul
EVENTS = ["mont.pending=2",              # a pending word of 2 after some round
          "mont.fold_carry",             # a lane carries out when its lower neighbour's pending word is folded in
          "mont.fold_carry_through_ones",  # ... and that carry crosses an all-ones lane
          "mont.hi=1",                   # the product reaches R: cond_sub gets hi = 1
          "cond_sub.borrow=0",           # both outcomes of cond_sub's compare
          "cond_sub.borrow=1",
          "cond_sub.borrow_through_zero",  # cond_sub's borrow crosses an all-zero lane
          "add.chain_all_lanes",         # a carry from lane 0 through every lane and out of the top
          "sub.chain_all_lanes"]
# the header's bounds: never reached by any input in the domain
VIOLATIONS = ["mont.pending>=4", "mont.t>=2m"]


def lanes(N):
    return N // 8


def R_of(N):
    return 1 << (32 * N)


# ---- integer model ------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=1 << 12)
def inv_pow2(x, bits):
    """x^-1 mod 2^bits for odd x, by Newton from 2^-bits precision 1 (as fast at 8192 bits as pow(x, -1, R) is slow)"""
    y, k = 1, 1
    while k < bits:
        k *= 2
        y = y * (2 - x * y) % (1 << k)
    return y % (1 << bits)


def mont(N, a, b, m):
    """a b R^-1 mod m for odd m, a < R and b < m (or the other way round), by one big-integer Montgomery reduction"""
    R = R_of(N)
    t = a * b
    u = (t % R) * (R - inv_pow2(m, 32 * N)) % R  # t + u m = 0 mod R
    r = (t + u * m) >> (32 * N)
    return r - m if r >= m else r


def expect(N, op, xs):
    """(number, scalar) the harness writes for one item: the number result (0 for the flag ops) and the carry, borrow,
    flag or neg_inv32 word (0 for the ops without one)"""
    R = R_of(N)
    if op == "add":
        s = xs[0] + xs[1]
        return s % R, s >> (32 * N)
    if op == "sub":
        return (xs[0] - xs[1]) % R, int(xs[0] < xs[1])
    if op == "mod_add":
        a, b, m = xs
        return (a + b) % m, 0
    if op == "mod_dbl":
        a, m = xs
        return 2 * a % m, 0
    if op == "cond_sub":
        t, m, hi = xs
        return (t + hi * R) % m, 0
    if op == "mont_mul":
        return mont(N, *xs), 0
    if op == "lo_mul":
        return xs[0] * xs[1] % R, 0
    if op == "inv_mod_r":
        return inv_pow2(xs[0], 32 * N), 0
    if op == "truncate_bits":
        a, s = xs
        return a % (1 << s), 0
    if op == "is_zero":
        return 0, int(xs[0] == 0)
    if op == "is_one":
        return 0, int(xs[0] == 1)
    if op == "neg_inv32":
        return 0, -pow(xs[0], -1, 1 << 32) % (1 << 32)
    raise KeyError(op)


def in_domain(N, op, xs):
    """the header's documented domain of each op"""
    R = R_of(N)
    if op in ("add", "sub", "lo_mul"):
        return all(0 <= x < R for x in xs)
    if op == "mod_add":
        a, b, m = xs
        return 0 < m < R and 0 <= a < m and 0 <= b < m
    if op == "mod_dbl":
        a, m = xs
        return 0 < m < R and 0 <= a < m
    if op == "cond_sub":
        t, m, hi = xs
        return 0 < m < R and 0 <= t < R and hi >= 0 and t + hi * R < 2 * m
    if op == "mont_mul":
        a, b, m = xs
        return 3 <= m < R and m & 1 and 0 <= a < R and 0 <= b < R and (a < m or b < m)
    if op == "inv_mod_r":
        return 0 < xs[0] < R and xs[0] & 1
    if op == "truncate_bits":
        a, s = xs
        return 0 <= a < R and 0 <= s <= 32 * N
    if op in ("is_zero", "is_one"):
        return 0 <= xs[0] < R
    if op == "neg_inv32":
        return 0 < xs[0] <= M32 and xs[0] & 1
    raise KeyError(op)


# ---- edge values --------------------------------------------------------------------------------------------------------
def _dedupe(xs):
    return list(dict.fromkeys(xs))


def _join(ls):
    return sum(v << (LANE_BITS * l) for l, v in enumerate(ls))


def _alternating(N, phase):
    """lanes alternately all ones and all zero, lane 0 all ones for phase 0"""
    return _join([M256 if (l + phase) % 2 == 0 else 0 for l in range(lanes(N))])


def _random_top(N, below, tag=""):
    """a random nonzero top lane over lanes of `below` (all ones, all zero, alternating); within the one lane of N = 8, a
    random upper half over a lower half of that pattern.  Seeded by its arguments, so every edge set is fixed."""
    T = lanes(N)
    rng = random.Random(f"bigmod/{N}/{below}/{tag}")
    if T == 1:
        low = {"ones": (1 << 128) - 1, "zero": 0, "alt": (1 << 64) - 1}[below]
        return (rng.getrandbits(128) | 1 << 127) << 128 | low
    low = {"ones": M256, "zero": 0}
    ls = [low[below] if below in low else (M256 if l % 2 == 0 else 0) for l in range(T - 1)]
    return _join(ls + [rng.getrandbits(LANE_BITS) | 1 << (LANE_BITS - 1)])


def chain_values(N):
    """2^(256 j) and 2^(256 j) - 1: carry and borrow chains through j lanes (every j up to 8 lanes, then a spread)"""
    T = lanes(N)
    js = range(1, T + 1) if T <= 8 else sorted({1, 2, 3, T // 2, T - 2, T - 1, T})
    out = []
    for j in js:
        if j < T:
            out.append(1 << (LANE_BITS * j))
        out.append((1 << (LANE_BITS * j)) - 1)
    return out


def moduli(N):
    """edge moduli of width N (odd and even, all < R): the small and near-R ones, half of R, one or two top limbs, lanes
    alternating all ones and all zero, and a random odd modulus over all-ones lower lanes"""
    R = R_of(N)
    ms = [3, (1 << 32) - 1, (1 << 32) + 1, R - 1, R - 3, R // 2 - 1, R // 2 + 1, R - (1 << 32) + 1, (1 << (32 * N - 32)) + 1,
          _alternating(N, 0), _alternating(N, 1), _random_top(N, "ones", "modulus") | 1]
    return [m for m in _dedupe(ms) if 0 < m < R]


def values(N):
    """modulus-free edge values below R: 0, 1, 2, R - 1, R - 2, the lane chains, random tops over patterned lanes, and
    the edge moduli with their neighbours"""
    R = R_of(N)
    vs = [0, 1, 2, 3, R - 1, R - 2, R // 2, R // 2 - 1] + chain_values(N)
    vs += [_random_top(N, below) for below in ("ones", "zero", "alt")]
    for m in moduli(N):
        vs += [m, m - 1, m - 2]
    return [v for v in _dedupe(vs) if 0 <= v < R]


def operands(N, m):
    """edge operands for modulus m, all below R: 0, 1, 2, m - 1, m - 2, R - 1, random tops over patterned lanes and
    the lane chains; the caller reduces them below m where the op needs it"""
    R = R_of(N)
    vs = [0, 1, 2, m - 1, m - 2, R - 1, R - 2] + [_random_top(N, below) for below in ("ones", "zero", "alt")]
    vs += chain_values(N)[:4] + chain_values(N)[-2:]
    return [v for v in _dedupe(vs) if 0 <= v < R]


def below(vs, m):
    return _dedupe(v % m for v in vs)


def mont_edges(N):
    """(a, b, m) for every odd edge modulus: a over the edge operands, b over them reduced below m, and swapped"""
    items = []
    for m in moduli(N):
        if m < 3 or not m & 1:
            continue
        ops = operands(N, m)
        red = below(ops, m)
        items += [(a, b, m) for a in ops for b in red]
        items += [(b, a, m) for a in ops for b in red if a >= m]  # a < m, b < R: the other way round
    return items


def cond_sub_edges(N):
    """(t, m, hi) with t + hi R = x for x < 2m at the edges: 0, 1, m - 1, m, m + 1, 2m - 2, 2m - 1, R - 1 .. R + 1 where
    they fit, and the edge operands below m with and without m added"""
    R = R_of(N)
    items = []
    for m in moduli(N):
        xs = [0, 1, m - 1, m, m + 1, 2 * m - 2, 2 * m - 1, R - 1, R, R + 1]
        red = below(operands(N, m), m)
        xs += red + [v + m for v in red]
        items += [(x % R, m, x >> (32 * N)) for x in _dedupe(xs) if 0 <= x < 2 * m]
    return items


def edge_items(N, op):
    """operand tuples at the edges, each inside the op's domain"""
    R = R_of(N)
    V = values(N)
    if op in ("add", "sub", "lo_mul"):
        return [(a, b) for a in V for b in V]
    if op == "mod_add":
        items = []
        for m in moduli(N):
            red = below(operands(N, m), m)
            items += [(a, b, m) for a in red for b in red]
        return items
    if op == "mod_dbl":
        return [(a, m) for m in moduli(N) for a in below(operands(N, m) + [m // 2, m // 2 + 1, (m + 1) // 2], m)]
    if op == "cond_sub":
        return cond_sub_edges(N)
    if op == "mont_mul":
        return mont_edges(N)
    if op == "inv_mod_r":
        return [(q,) for q in _dedupe(v | 1 for v in V)]
    if op == "truncate_bits":
        ss = _dedupe(s for s in [0, 1, 31, 32, 33, 255, 256, 257, 32 * N // 2, 32 * N - 32, 32 * N - 1, 32 * N]
                     + [LANE_BITS * j + d for j in range(1, lanes(N)) for d in (-1, 0, 1)] if 0 <= s <= 32 * N)
        return [(a, s) for a in [R - 1, _alternating(N, 0), _random_top(N, "ones")] for s in ss]
    if op in ("is_zero", "is_one"):
        singles = [1 << (32 * k) for k in range(N)] + [1 | (1 << (32 * k)) for k in range(1, N)]  # a one in every limb
        return [(a,) for a in _dedupe(V + singles)]
    if op == "neg_inv32":
        return [(x,) for x in (1, 3, 5, 0x7fffffff, 0x80000001, 0xfffffffd, 0xffffffff, 0x12345679)]
    raise KeyError(op)


def random_modulus(rng, N, odd=False):
    """a modulus of at least 2 bits below R: full width half the time, else a random bit length; odd, or of either
    parity"""
    bits = 32 * N if rng.random() < 0.5 else rng.randrange(2, 32 * N + 1)
    return rng.getrandbits(bits) | 1 << (bits - 1) | int(odd)


def random_items(N, op, rng, count):
    """random operand tuples inside the op's domain"""
    R = R_of(N)
    rnd = lambda: rng.getrandbits(32 * N)
    items = []
    for _ in range(count):
        if op in ("add", "sub", "lo_mul"):
            items.append((rnd(), rnd()))
        elif op == "mod_add":
            m = random_modulus(rng, N)
            items.append((rng.randrange(m), rng.randrange(m), m))
        elif op == "mod_dbl":
            m = random_modulus(rng, N)
            items.append((rng.randrange(m), m))
        elif op == "cond_sub":
            m = random_modulus(rng, N)
            x = rng.randrange(2 * m)
            items.append((x % R, m, x >> (32 * N)))
        elif op == "mont_mul":
            m = random_modulus(rng, N, odd=True)
            a, b = rnd(), rng.randrange(m)
            items.append((a, b, m) if rng.random() < 0.5 else (b, a, m))
        elif op == "inv_mod_r":
            items.append((rnd() | 1,))
        elif op == "truncate_bits":
            items.append((rnd(), rng.randrange(32 * N + 1)))
        elif op in ("is_zero", "is_one"):
            items.append((rnd() >> rng.randrange(32 * N + 1),))  # zero and one now and then
        elif op == "neg_inv32":
            items.append((rng.getrandbits(32) | 1,))
        else:
            raise KeyError(op)
    return items


# ---- limb-exact model ---------------------------------------------------------------------------------------------------
def _lanes(x, N):
    return [(x >> (LANE_BITS * l)) & M256 for l in range(lanes(N))]


def _neighbour(xs, d):
    """xs of lane + d, 0 outside the group"""
    return [xs[l + d] if 0 <= l + d < len(xs) else 0 for l in range(len(xs))]


def _resolve(gen, prop, no_propagate=False):
    """resolve(): the carry-in bit of each lane and the carry out of the top, from the generate and propagate ballots"""
    T = len(gen)
    G = sum(1 << l for l in range(T) if gen[l])
    P = sum(1 << l for l in range(T) if prop[l])
    assert not G & P, "a lane both generates and propagates"
    C = G << 1 if no_propagate else ((G << 1) + P) ^ P
    return [(C >> l) & 1 for l in range(T)], (C >> T) & 1


def model_add(N, a, b, ev=None):
    """add(): per-lane sums, then one resolve; (a + b mod R, carry out)"""
    s = [x + y for x, y in zip(_lanes(a, N), _lanes(b, N))]
    gen, t = [v >> LANE_BITS for v in s], [v & M256 for v in s]
    prop = [v == M256 for v in t]
    cin, cout = _resolve(gen, prop)
    if ev is not None and gen[0] and all(prop[1:]) and cout:
        ev.add("add.chain_all_lanes")
    return _join([(v + c) & M256 for v, c in zip(t, cin)]), cout


def model_sub(N, a, b, ev=None, tag="sub"):
    """sub(): per-lane differences, then one resolve of the borrows; (a - b mod R, borrow out)"""
    d = [x - y for x, y in zip(_lanes(a, N), _lanes(b, N))]
    gen, t = [int(v < 0) for v in d], [v & M256 for v in d]
    prop = [v == 0 for v in t]
    bin_, bout = _resolve(gen, prop)
    if ev is not None:
        if any(p and c for p, c in zip(prop, bin_)):
            ev.add(tag + ".borrow_through_zero")
        if gen[0] and all(prop[1:]) and bout:
            ev.add(tag + ".chain_all_lanes")
    return _join([(v - c) & M256 for v, c in zip(t, bin_)]), bout


def model_cond_sub(N, t, hi, m, ev=None, mutant=None):
    """cond_sub(): t - m kept when hi is set or the subtraction does not borrow"""
    d, borrow = model_sub(N, t, m, ev, "cond_sub")
    if ev is not None:
        ev.add(f"cond_sub.borrow={borrow}")
    keep = not borrow if mutant == "cond_sub_ignores_hi" else hi or not borrow
    return d if keep else t


def model_mont_mul(N, a, b, m, ev=None, mutant=None):
    """mont_mul() lane by lane: a * b / R mod m for odd m, a < R and b < m (or the other way round)"""
    T = lanes(N)
    below = {"from_below_two_lanes": -2, "from_below_own_lane": 0}.get(mutant, -1)
    above = {"from_above_two_lanes": 2, "from_above_own_lane": 0}.get(mutant, 1)
    A, M = _lanes(a, N), _lanes(m, N)
    mp = -pow(m & M32, -1, 1 << 32) & M32
    t, p = [0] * T, [0] * T
    for i in range(N):
        bi = (b >> (32 * i)) & M32
        s = [x + y * bi for x, y in zip(t, A)]  # mad_row(t, a, b_i)
        c1, t = [v >> LANE_BITS for v in s], [v & M256 for v in s]
        q = (t[0] & M32) * mp & M32  # from lane 0
        s = [x + y * q for x, y in zip(t, M)]  # mad_row(t, m, q)
        c2, t = [v >> LANE_BITS for v in s], [v & M256 for v in s]
        # shift_down: the limb arriving from above, plus the pending word and both row carries, becomes the top limb
        top = [u + pw + x + y for u, pw, x, y in zip(_neighbour([v & M32 for v in t], above), p, c1, c2)]
        t = [(v >> 32) | (w & M32) << (LANE_BITS - 32) for v, w in zip(t, top)]
        p = [w >> 32 for w in top]
        if ev is not None:
            ev.update(f"mont.pending={w}" for w in p if w >= 2)
            if max(p) >= 4:
                ev.add("mont.pending>=4")
    # fold: each lane adds its lower neighbour's pending word, then one resolve settles the 0/1 carries
    fold = [0] * T if mutant == "fold_dropped" else _neighbour(p, below)
    s = [v + w for v, w in zip(t, fold)]
    co, t = [v >> LANE_BITS for v in s], [v & M256 for v in s]
    prop = [v == M256 for v in t]
    cin, cout = _resolve([c != 0 for c in co], prop, mutant == "resolve_no_propagate")
    t = _join([(v + c) & M256 for v, c in zip(t, cin)])
    hi = p[T - 1] + cout
    if ev is not None:
        if any(co):
            ev.add("mont.fold_carry")
        if any(pr and c for pr, c in zip(prop, cin)):
            ev.add("mont.fold_carry_through_ones")
        if hi:
            ev.add(f"mont.hi={hi}")
        if t + hi * R_of(N) >= 2 * m:
            ev.add("mont.t>=2m")
    return model_cond_sub(N, t, hi, m, ev, mutant)


def probe_tuples(N):
    """a few mont_mul tuples that reach every carry event at any width: m = R - 1 with a = b = m - 1 (the product is
    R, folded through every lane), m = 2^(32N - 32) + 1 with small and top products, and R - 2^32 + 1"""
    R = R_of(N)
    items = []
    for m in (R - 1, (1 << (32 * N - 32)) + 1, R - (1 << 32) + 1, _alternating(N, 0)):
        for a, b in ((m - 1, m - 1), (m - 2, m - 1), (R - 1, m - 1), (R - 1, 1), (2, m - 2)):
            items.append((a, b % m, m))
    return items
