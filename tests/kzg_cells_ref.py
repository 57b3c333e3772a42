"""EIP-7594 cells and cell proofs in Python integers -- TEST INFRASTRUCTURE ONLY (the library computes the cells and checks
the proofs on the device, ethrex_b200/csrc/kzg_cells.cu and bls_pairing.cu).  Names follow the consensus-specs
polynomial-commitments-sampling document.

  compute_cells      a plain recursive NTT: blob values (bit-reversed) -> coefficients -> the zero-padded size-8192 NTT ->
                     bit-reversed order -> 128 cells of 64 elements
  cell proofs        over a known-tau setup, in the exponent: pi_k = [q_k(tau)]G1, q_k(tau) = (p(tau) - I_k(tau)) /
                     (tau^64 - h_k^64), I_k the interpolation of cell k's values on its coset (Lagrange form, not the
                     coefficient folding the device uses)
  the batch check    the universal equation as a scalar identity in tau, and through tests/bls_pairing_ref.py's pairing
"""
import bls_pairing_ref as B
import bls_ref as bls
import kzg_ref

R = bls.R
N, EXT, CELL, CELLS = 4096, 8192, 64, 128
ROOT_8192 = pow(7, (R - 1) // EXT, R)
_NAT = None


def _roots_8192():
    global _NAT
    if _NAT is None:
        nat = [1] * EXT
        for i in range(1, EXT):
            nat[i] = nat[i - 1] * ROOT_8192 % R
        _NAT = nat
    return _NAT


def ntt(vals, root):
    """out[j] = sum_i vals[i] root^(i j), natural order in and out (recursive radix 2)"""
    n = len(vals)
    if n == 1:
        return list(vals)
    r2 = root * root % R
    even, odd = ntt(vals[0::2], r2), ntt(vals[1::2], r2)
    out, w = [0] * n, 1
    for j in range(n // 2):
        t = w * odd[j] % R
        out[j], out[j + n // 2] = (even[j] + t) % R, (even[j] - t) % R
        w = w * root % R
    return out


def coefficients(blob: bytes):
    nat = [0] * N
    for i, v in enumerate(kzg_ref.blob_values(blob)):
        nat[bls.bit_reverse(i, 12)] = v
    ninv = pow(N, -1, R)
    return [c * ninv % R for c in ntt(nat, pow(bls.ROOT_4096, -1, R))]


def extension(blob: bytes):
    """p on the 8192 roots of unity, bit-reversed order"""
    ext = ntt(coefficients(blob) + [0] * N, ROOT_8192)
    return [ext[bls.bit_reverse(i, 13)] for i in range(EXT)]


def cells_of(ext):
    return [b"".join(v.to_bytes(32, "big") for v in ext[CELL * k:CELL * (k + 1)]) for k in range(CELLS)]


def compute_cells(blob: bytes):
    return cells_of(extension(blob))


def cell_values(cell: bytes):
    return [int.from_bytes(cell[32 * t:32 * t + 32], "big") for t in range(CELL)]


def coset(k: int):
    nat = _roots_8192()
    return [nat[bls.bit_reverse(CELL * k + t, 13)] for t in range(CELL)]


def shift64(k: int) -> int:
    """h_k^64 for h_k = the first root of cell k's coset"""
    return pow(_roots_8192()[bls.bit_reverse(CELL * k, 13)], CELL, R)


def interpolate_at(k: int, ys, tau: int) -> int:
    """I_k(tau): the degree < 64 polynomial through cell k's values on its coset, the roots of X^64 - s, whose Lagrange
    basis is L_t(tau) = x_t (tau^64 - s) / (64 s (tau - x_t))"""
    s = shift64(k)
    acc = sum(y * x % R * pow((tau - x) % R, -1, R) for x, y in zip(coset(k), ys)) % R
    return (pow(tau, CELL, R) - s) % R * acc % R * pow(CELL * s % R, -1, R) % R


def horner(coeffs, x: int) -> int:
    acc = 0
    for c in reversed(coeffs):
        acc = (acc * x + c) % R
    return acc


def proof_scalars(blob: bytes, tau: int):
    """(p(tau), [q_k(tau) for the 128 cells])"""
    pt = horner(coefficients(blob), tau)
    ext = extension(blob)
    t64 = pow(tau, CELL, R)
    qs = [(pt - interpolate_at(k, ext[CELL * k:CELL * (k + 1)], tau)) * pow((t64 - shift64(k)) % R, -1, R) % R for k in range(CELLS)]
    return pt, qs


def bundle(blobs, tau: int):
    """(commitments, proofs): 48-byte compressed each, proofs blob-major with the cell index inner"""
    commitments, proofs = [], []
    for blob in blobs:
        pt, qs = proof_scalars(blob, tau)
        pts = bls.generator_multiples([pt] + qs)
        commitments.append(bls.compress(pts[0]))
        proofs += [bls.compress(p) for p in pts[1:]]
    return commitments, proofs


def g2_setup(tau: int) -> bytes:
    """[tau^i]2 for i = 0..64, 96-byte compressed: the g2_monomial points the check reads"""
    return b"".join(B.g2_compress(B.g2_mul(pow(tau, i, R), B.G2)) for i in range(CELL + 1))


def equation_in_exponent(tau: int, r: int, p_taus, cells, qs) -> bool:
    """tau^64 sum r^k q_k = sum_i (sum_(k in i) r^k) p_i(tau) - sum r^k I_k(tau) + sum r^k h_k^64 q_k, k over every cell
    (blob-major); p_taus[i] the commitments' logs, cells[k] the claimed cell bytes, qs[k] the proofs' logs"""
    lhs = rhs = 0
    for k, (cell, q) in enumerate(zip(cells, qs)):
        rk, c = pow(r, k, R), k % CELLS
        lhs += rk * q
        rhs += rk * (p_taus[k // CELLS] - interpolate_at(c, cell_values(cell), tau) + shift64(c) * q)
    return (pow(tau, CELL, R) * lhs - rhs) % R == 0


def equation_by_pairing(tau: int, r: int, commitments, cells, proofs) -> bool:
    """e(sum r^k pi_k, [tau^64]2) = e(sum_i (sum_(k in i) r^k) C_i - [sum r^k I_k(tau)]1 + sum r^k h_k^64 pi_k, [1]2) on the
    points themselves; [sum r^k I_k(tau)]1 is what the Lagrange setup's MSM gives, here [A(tau)]G1"""
    left = right = None
    a_tau = 0
    weights = [0] * len(commitments)
    for k, (cell, proof) in enumerate(zip(cells, proofs)):
        rk, c = pow(r, k, R), k % CELLS
        pi = bls.decompress(proof)
        left = bls.add(left, bls.mul(rk, pi))
        right = bls.add(right, bls.mul(rk * shift64(c), pi))
        weights[k // CELLS] += rk
        a_tau += rk * interpolate_at(c, cell_values(cell), tau)
    for w, cm in zip(weights, commitments):
        right = bls.add(right, bls.mul(w, bls.decompress(cm)))
    right = bls.add(right, bls.mul(-a_tau % R, bls.G1))
    neg = None if right is None else (right[0], bls.P - right[1])
    return B.pairing_check([(left, B.g2_mul(pow(tau, CELL, R), B.G2)), (neg, B.G2)])
