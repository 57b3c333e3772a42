"""EIP-7594 cell proofs by FK20, restated in scalars -- TEST INFRASTRUCTURE ONLY (the library computes them on the device,
ethrex_b200/csrc/kzg_cells.cu: kzg_fk20_table, kzg_fk20_columns, kzg_fk20_msm, kzg_fk20_proofs).  Over a known-tau setup
every point [tau^i]1 is replaced by the scalar tau^i, so each step below is the kernel's step with its group operation
done on discrete logarithms.  The indexing is exactly the kernels'.

With c_0 .. c_4095 the blob's coefficients, C_b[t] = c_(64 t + b) and S_b[a] = tau^(64 a + b) (b < 64, t, a < 64):
  T_m = sum_(i <= 4095 - 64 m) c_(i + 64 m) tau^i = sum_b sum_(a <= 63 - m) C_b[a + m] S_b[a]      (m = 1 .. 63)
is, per column b, a correlation, i.e. a circular convolution of length 128 of C_b (zero-padded) with
  S''_b[0] = S_b[0],  S''_b[128 - a] = S_b[a] (a = 1 .. 63),  S''_b[k] = 0 (k = 1 .. 64)
that does not wrap for m < 64.  So
  table[b] = DFT(S''_b)                       once per setup (64 G1 DFTs of size 128)
  u = sum_b DFT(C_b) * table[b]               per blob: 64 Fr DFTs, then 128 MSMs of 64 terms
  z = DFT^-1(u),  T_m = z[m]                  one inverse G1 DFT (its 1/128 folded into the Fr side)
  pi_k = sum_(m=1..63) s_k^(m-1) T_m = DFT(v)[brp7(k)],  v[t] = z[t + 1] (t < 63), 0 else
All DFTs have root w_128 = w_8192^64 (w_8192 = 7^((r-1)/8192)).  Forward DFTs are Gentleman-Sande (natural order in,
bit-reversed out); the inverse is Cooley-Tukey (bit-reversed in, natural out), as ntt_forward_brp / ntt_inverse_brp of
kzg_cells.cu.  The Fr DFTs and the table are therefore both in bit-reversed order, the pointwise sums need no
permutation, and the final DFT leaves pi_k at position k.
"""
import bls_ref as bls
import kzg_cells_ref as ref

R = bls.R
N, EXT, CELL, CELLS = 4096, 8192, 64, 128
M = 128  # the circulant's size


def _tw(i: int) -> int:
    return ref._roots_8192()[i % EXT]


def dif(vals, mul, add, sub):
    """Gentleman-Sande, size 128, root w_128: natural order in, position i out holds DFT(vals)[brp7(i)]"""
    s = list(vals)
    h = M // 2
    while h >= 1:
        step = EXT // (2 * h)
        for b in range(M // 2):
            j = b & (h - 1)
            i0 = 2 * b - j
            i1 = i0 + h
            u, v = s[i0], s[i1]
            s[i0], s[i1] = add(u, v), mul(sub(u, v), _tw(j * step))
        h //= 2
    return s


def dit_inverse(vals, mul, add, sub):
    """Cooley-Tukey, size 128, root w_128^-1, unscaled: bit-reversed order in, natural order out"""
    s = list(vals)
    h = 1
    while h < M:
        step = EXT // (2 * h)
        for b in range(M // 2):
            j = b & (h - 1)
            i0 = 2 * b - j
            i1 = i0 + h
            u, v = s[i0], mul(s[i1], _tw((EXT - j * step) % EXT))
            s[i0], s[i1] = add(u, v), sub(u, v)
        h *= 2
    return s


FR = (lambda x, w: x * w % R, lambda a, b: (a + b) % R, lambda a, b: (a - b) % R)


def table_scalars(tau: int):
    """table[b][i]: the FK20 table as discrete logarithms, bit-reversed position i (kzg_fk20_table)"""
    out = []
    for b in range(CELL):
        col = [0] * M
        col[0] = pow(tau, b, R)
        for a in range(1, CELL):
            col[M - a] = pow(tau, CELL * a + b, R)
        out.append(dif(col, *FR))
    return out


def column_dfts(blob: bytes):
    """hat[b][i] = DFT(C_b)[brp7(i)] / 128 (kzg_fk20_columns: the inverse DFT's 1/128 folded in)"""
    c = ref.coefficients(blob)
    inv128 = pow(M, -1, R)
    return [[x * inv128 % R for x in dif([c[CELL * t + b] for t in range(CELL)] + [0] * CELL, *FR)] for b in range(CELL)]


def toeplitz_sums(blob: bytes, tau: int):
    """z = DFT^-1(sum_b hat_b * table_b): z[m] = T_m for m = 1 .. 63 (kzg_fk20_msm, then kzg_fk20_proofs' first half)"""
    tab, hat = table_scalars(tau), column_dfts(blob)
    u = [sum(hat[b][i] * tab[b][i] for b in range(CELL)) % R for i in range(M)]
    return dit_inverse(u, *FR)


def proof_scalars(blob: bytes, tau: int):
    """the 128 cell proofs' discrete logarithms in cell order (kzg_fk20_proofs' second half)"""
    z = toeplitz_sums(blob, tau)
    v = [z[t + 1] for t in range(CELL - 1)] + [0] * (M - CELL + 1)
    return dif(v, *FR)


def toeplitz_direct(blob: bytes, tau: int):
    """T_m = sum_(i <= 4095 - 64 m) c_(i + 64 m) tau^i for m = 1 .. 63 (index 0 unused)"""
    c = ref.coefficients(blob)
    t = [0] * CELL
    for m in range(1, CELL):
        t[m] = ref.horner(c[CELL * m:], tau)
    return t


def proofs_from_toeplitz(t):
    """pi_k = sum_(m=1..63) s_k^(m-1) T_m, s_k = h_k^64 = w_128^brp7(k)"""
    out = []
    for k in range(CELLS):
        s = ref.shift64(k)
        acc, sp = 0, 1
        for m in range(1, CELL):
            acc = (acc + sp * t[m]) % R
            sp = sp * s % R
        out.append(acc)
    return out
