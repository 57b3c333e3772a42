"""EIP-7594 cell recovery in Python integers -- TEST INFRASTRUCTURE ONLY (the library recovers cells on the device,
ethrex_b200/csrc/kzg_cells.cu).  Two independent routes from a partial set of cells to the blob's 4096 coefficients:

  recover_coefficients   the consensus-specs route (polynomial-commitments-sampling, recover_polynomialcoeff): the
                         vanishing polynomial Z of the missing cells' cosets, (E Z) from the zero-filled extension E by a
                         size-8192 NTT, division by Z on the shifted coset 7 <w_8192>, and the inverse transform
  recover_columns        the device's route, with the kernel's indexing: per given cell a size-64 inverse NTT unshifted by
                         h_c^-j gives P_j(s_c) (p = sum_j X^j P_j(X^64)); Lagrange interpolation of each P_j on the first
                         64 given cells' s_c is one 64 x 64 by 64 x 64 product
"""
import random

import bls_ref as bls
import kzg_cells_ref as cells_ref

R = bls.R
N, EXT, CELL, CELLS = cells_ref.N, cells_ref.EXT, cells_ref.CELL, cells_ref.CELLS
SHIFT = 7  # the coset the spec divides on: 7 <w_8192>, off the domain since 7 is not an 8192nd root


def _brp(i: int, bits: int) -> int:
    return bls.bit_reverse(i, bits)


def _mul_poly(a, b):
    out = [0] * (len(a) + len(b) - 1)
    for i, x in enumerate(a):
        if x:
            for j, y in enumerate(b):
                out[i + j] = (out[i + j] + x * y) % R
    return out


def _coset_ntt(coeffs, inverse=False):
    """values of coeffs on SHIFT w^j (natural order), or (inverse) the coefficients from such values"""
    w = cells_ref.ROOT_8192
    if not inverse:
        return cells_ref.ntt([c * pow(SHIFT, i, R) % R for i, c in enumerate(coeffs)], w)
    ninv, sinv = pow(EXT, -1, R), pow(SHIFT, -1, R)
    return [c * ninv % R * pow(sinv, i, R) % R for i, c in enumerate(cells_ref.ntt(coeffs, pow(w, -1, R)))]


def recover_coefficients(indices, cells):
    """the blob's 4096 coefficients from cells (2048-byte each) at distinct indices, by the consensus-specs route"""
    given = dict(zip(indices, cells))
    missing = [c for c in range(CELLS) if c not in given]
    # Z(X) = prod_(c missing) (X^64 - s_c): the short product over the 128th roots, spread to X^64
    short = [1]
    for c in missing:
        short = _mul_poly(short, [(-cells_ref.shift64(c)) % R, 1])
    zero_poly = [0] * EXT
    for i, v in enumerate(short):
        zero_poly[CELL * i] = v
    # E on the 8192 roots in natural order: cell c's point t sits at brp13(64 c + t)
    ext = [0] * EXT
    for c, cell in given.items():
        for t, v in enumerate(cells_ref.cell_values(cell)):
            ext[_brp(CELL * c + t, 13)] = v
    w = cells_ref.ROOT_8192
    z_eval = cells_ref.ntt(zero_poly, w)
    ez_eval = [a * b % R for a, b in zip(ext, z_eval)]
    ninv = pow(EXT, -1, R)
    ez_coeffs = [c * ninv % R for c in cells_ref.ntt(ez_eval, pow(w, -1, R))]
    # (E Z) / Z on the shifted coset, where Z has no zeros
    quotient = [a * pow(b, -1, R) % R for a, b in zip(_coset_ntt(ez_coeffs), _coset_ntt(zero_poly))]
    coeffs = _coset_ntt(quotient, inverse=True)
    assert not any(coeffs[N:]), "the recovered polynomial has degree >= 4096"
    return coeffs[:N]


def recover_columns(indices, cells):
    """the same coefficients by the device's route, from the first 64 given cells (kzg_recover_blob's indexing)"""
    w = cells_ref.ROOT_8192
    w64inv = pow(w, -(EXT // CELL), R)
    sel = list(zip(indices, cells))[:CELL]
    s = [pow(w, CELL * _brp(c, 7), R) for c, _ in sel]
    # Z = prod (X - s_k), lowest coefficient first, built one factor at a time as the kernel's 65 threads do
    z = [1] + [0] * CELL
    for sk in s:
        z = [((z[t - 1] if t else 0) - sk * z[t]) % R for t in range(CELL + 1)]
    coef = [0] * N
    e_rows, q_rows = [], []
    for k, (c, cell) in enumerate(sel):
        vals = cells_ref.cell_values(cell)
        nat = [0] * CELL
        for t, v in enumerate(vals):
            nat[_brp(t, 6)] = v
        a = cells_ref.ntt(nat, w64inv)  # 64 P_j(s_k) h_k^j, unscaled
        q = [0] * CELL
        q[CELL - 1] = 1
        for m in range(CELL - 1, 0, -1):
            q[m - 1] = (z[m] + s[k] * q[m]) % R
        d = 1
        for l, sl in enumerate(s):
            if l != k:
                d = d * (s[k] - sl) % R
        scale = pow(CELL * d % R, -1, R)
        h = _brp(c, 7)
        e_rows.append([a[j] * pow(w, (EXT - h * j) % EXT, R) % R * scale % R for j in range(CELL)])
        q_rows.append(q)
    for m in range(CELL):
        for j in range(CELL):
            coef[CELL * m + j] = sum(e_rows[k][j] * q_rows[k][m] for k in range(CELL)) % R
    return coef


def patterns(seed: int):
    """name -> the given cell indices, in the order they are passed"""
    rng = random.Random(seed)
    pick = lambda k: rng.sample(range(CELLS), k)  # noqa: E731
    shuffled = list(range(0, CELLS, 2))
    rng.shuffle(shuffled)
    return {
        "first64": list(range(CELL)),
        "last64": list(range(CELL, CELLS)),
        "even": list(range(0, CELLS, 2)),
        "odd": list(range(1, CELLS, 2)),
        "random64": pick(64),
        "random65": pick(65),
        "random96": pick(96),
        "random127": pick(127),
        "all128": list(range(CELLS)),
        "shuffled": shuffled,
    }
