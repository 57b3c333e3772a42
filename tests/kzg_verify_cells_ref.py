"""verify_cell_kzg_proof_batch over arbitrary cells, restated from the consensus-specs polynomial-commitments-sampling
document -- TEST INFRASTRUCTURE ONLY (the library runs it on the device: b200zk_kzg_verify_cells, bls_pairing.cu and
kzg_cells.cu).  Over the known-tau setup of tests/kzg_cells_ref.py.

  deduplicate        the deduplicated commitments in order of first occurrence and each cell's commitment index
  challenge          compute_verify_cell_kzg_proof_batch_challenge
  whole_blob_challenge  the construction of DESIGN section 4.12 (per-blob commitments, blob and cell index per cell),
                     restated separately: for whole blobs with distinct commitments the two agree
  equation_in_exponent / equation_by_pairing
                     verify_cell_kzg_proof_batch_impl as a scalar identity in tau, and on the points through
                     tests/bls_pairing_ref.py's pairing; I_k by Lagrange on the coset (kzg_cells_ref.interpolate_at)
  column_route       the device's route to A = sum r^k I_k: per cell index c, agg_c = sum r^k y_k, an inverse NTT of size
                     64 and the unshift by h_c^-i / 64; its coefficients, summed over the columns
"""
import hashlib

import bls_pairing_ref as B
import bls_ref as bls
import kzg_cells_ref as cref

R = bls.R
DOMAIN = b"RCKZGCBATCH__V1_"
ROOT_64 = pow(cref.ROOT_8192, 128, R)


def _u64(v: int) -> bytes:
    return v.to_bytes(8, "big")


def deduplicate(commitments):
    """(deduplicated commitments, commitment index of each cell)"""
    unique, pos, index = [], {}, []
    for c in commitments:
        if c not in pos:
            pos[c] = len(unique)
            unique.append(c)
        index.append(pos[c])
    return unique, index


def challenge(commitments, cell_indices, cells, proofs) -> int:
    unique, index = deduplicate(commitments)
    data = DOMAIN + _u64(cref.N) + _u64(cref.CELL) + _u64(len(unique)) + _u64(len(cell_indices)) + b"".join(unique)
    for i, c, cell, proof in zip(index, cell_indices, cells, proofs):
        data += _u64(i) + _u64(c) + cell + proof
    return int.from_bytes(hashlib.sha256(data).digest(), "big") % R


def whole_blob_challenge(blob_commitments, cells, proofs) -> int:
    """section 4.12: every cell of every blob, blob-major; the commitments listed per blob"""
    n = len(blob_commitments)
    data = DOMAIN + _u64(cref.N) + _u64(cref.CELL) + _u64(n) + _u64(cref.CELLS * n) + b"".join(blob_commitments)
    for k, (cell, proof) in enumerate(zip(cells, proofs)):
        data += _u64(k // cref.CELLS) + _u64(k % cref.CELLS) + cell + proof
    return int.from_bytes(hashlib.sha256(data).digest(), "big") % R


def equation_in_exponent(tau: int, r: int, commitment_logs, cell_indices, cells, proof_logs) -> bool:
    """tau^64 sum r^k q_k = sum_i w_i p_i - sum r^k I_k(tau) + sum r^k h_k^64 q_k; commitment_logs[k] is cell k's
    commitment's log (cells sharing a commitment share it), proof_logs[k] its proof's"""
    lhs = rhs = 0
    for k, (p, c, cell, q) in enumerate(zip(commitment_logs, cell_indices, cells, proof_logs)):
        rk = pow(r, k, R)
        lhs += rk * q
        rhs += rk * (p - cref.interpolate_at(c, cref.cell_values(cell), tau) + cref.shift64(c) * q)
    return (pow(tau, cref.CELL, R) * lhs - rhs) % R == 0


def equation_by_pairing(tau: int, r: int, commitments, cell_indices, cells, proofs) -> bool:
    """verify_cell_kzg_proof_batch_impl on the points: e(LL, -[tau^64]2) e(RLC - RLI + RLP, [1]2) = 1"""
    unique, index = deduplicate(commitments)
    weights = [0] * len(unique)
    ll = rlp = None
    a_tau = 0
    for k, (i, c, cell, proof) in enumerate(zip(index, cell_indices, cells, proofs)):
        rk = pow(r, k, R)
        pi = bls.decompress(proof)
        ll = bls.add(ll, bls.mul(rk, pi))
        rlp = bls.add(rlp, bls.mul(rk * cref.shift64(c) % R, pi))
        weights[i] = (weights[i] + rk) % R
        a_tau += rk * cref.interpolate_at(c, cref.cell_values(cell), tau)
    rl = rlp
    for w, cm in zip(weights, unique):
        rl = bls.add(rl, bls.mul(w, bls.decompress(cm)))
    rl = bls.add(rl, bls.mul(-a_tau % R, bls.G1))
    neg = None if ll is None else (ll[0], bls.P - ll[1])
    return B.pairing_check([(neg, B.g2_mul(pow(tau, cref.CELL, R), B.G2)), (rl, B.G2)])


def verify(tau: int, commitments, cell_indices, cells, proofs) -> bool:
    """the whole call: n = 0 is true; the challenge, then the pairing check"""
    if not cell_indices:
        return True
    return equation_by_pairing(tau, challenge(commitments, cell_indices, cells, proofs), commitments, cell_indices, cells, proofs)


def column_route(r: int, cell_indices, cells):
    """the 64 coefficients of A = sum r^k I_k as the device forms them, one column per cell index that occurs"""
    agg = {}
    for k, (c, cell) in enumerate(zip(cell_indices, cells)):
        rk = pow(r, k, R)
        acc = agg.setdefault(c, [0] * cref.CELL)
        for t, y in enumerate(cref.cell_values(cell)):
            acc[t] = (acc[t] + rk * y) % R
    a = [0] * cref.CELL
    inv64 = pow(cref.CELL, -1, R)
    for c, vals in agg.items():
        nat = [0] * cref.CELL
        for t, y in enumerate(vals):
            nat[bls.bit_reverse(t, 6)] = y
        g = cref.ntt(nat, pow(ROOT_64, -1, R))
        h_inv = pow(pow(cref.ROOT_8192, bls.bit_reverse(c, 7), R), -1, R)
        for i in range(cref.CELL):
            a[i] = (a[i] + g[i] * inv64 * pow(h_inv, i, R)) % R
    return a
