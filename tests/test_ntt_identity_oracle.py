"""The CPU oracle's O(n) whole-vector NTT check (cpu_oracle.NttIdentity) and its chunked output evaluation, on the CPU.

The check is what the GPU sweep relies on from 2^25 up, where the oracle's own transform is too slow to run, so it has to
be shown to accept exactly the transforms the oracle computes and nothing near them: every mode, both roots of unity, fed
whole and in uneven chunks; then one changed limb at the first, last and a middle output, and two swapped outputs, must
each be refused."""
import numpy as np
import pytest

import cpu_oracle as orc
import pyref

HALO2_ROOT = pow(7, (pyref.R - 1) >> 28, pyref.R)
# (oracle flags, coset generator): forward, inverse, coset and inverse coset with the default generator 5, then both
# coset directions with a caller's generator
MODES = [(0, None), (orc.NTT_INVERSE, None), (orc.NTT_COSET, None), (orc.NTT_INVERSE | orc.NTT_COSET, None),
         (orc.NTT_COSET, 7), (orc.NTT_INVERSE | orc.NTT_COSET, pyref.R - 3)]


def _check(a, y, log_n, flags, gen, root, chunk):
    chk = orc.NttIdentity(log_n, flags, gen, root)
    n = 1 << log_n
    for s in range(0, n, chunk):
        chk.update(a[s:s + chunk], y[s:s + chunk], s)
    return chk.ok()


@pytest.mark.parametrize("root", [None, HALO2_ROOT], ids=["ark", "halo2"])
@pytest.mark.parametrize("log_n", list(range(0, 17)))
def test_identity_accepts_the_oracle_transform_and_rejects_one_wrong_output(log_n, root):
    n = 1 << log_n
    a = orc.fr_to_mont(orc.rand_fr(pyref.SEED_NTT + log_n, 0, n))
    for flags, gen in MODES:
        y = orc.fr_ntt(a, log_n, flags, coset_gen=gen, root_2_28=root)
        what = f"log_n={log_n} flags={flags} gen={gen}"
        assert _check(a, y, log_n, flags, gen, root, n), what
        assert _check(a, y, log_n, flags, gen, root, max(1, n // 3 + 1)), what  # chunks that do not divide n
        assert orc.fr_ntt_identity(a, y, log_n, flags, gen, root), what
        if log_n < 4:
            continue
        for i, limb in ((0, 0), (n // 2 + 3, 1), (n - 1, 2)):
            bad = y.copy()
            bad[i, limb] ^= np.uint64(1)
            assert not _check(a, bad, log_n, flags, gen, root, n), (what, i, limb)
        bad = y.copy()
        bad[[1, n - 2]] = bad[[n - 2, 1]]
        assert not (bad == y).all()
        assert not _check(a, bad, log_n, flags, gen, root, n), (what, "swap")
        # the same output under the other direction, or the other root where the two differ, is refused too
        other = flags ^ orc.NTT_INVERSE
        assert not _check(a, y, log_n, other, gen, root, n), (what, "direction")


def test_identity_tells_the_two_roots_apart():
    log_n, n = 12, 1 << 12
    a = orc.fr_to_mont(orc.rand_fr(pyref.SEED_NTT, 0, n))
    for flags, gen in MODES:
        y = orc.fr_ntt(a, log_n, flags, coset_gen=gen, root_2_28=HALO2_ROOT)
        assert _check(a, y, log_n, flags, gen, HALO2_ROOT, n)
        assert not _check(a, y, log_n, flags, gen, None, n)


def test_identity_refuses_a_partial_feed():
    log_n, n = 6, 64
    a = orc.fr_to_mont(orc.rand_fr(pyref.SEED_NTT, 0, n))
    chk = orc.NttIdentity(log_n)
    chk.update(a[:32], orc.fr_ntt(a, log_n)[:32], 0)
    with pytest.raises(AssertionError):
        chk.ok()
    with pytest.raises(ValueError):
        chk.update(a[:32], a[:32], 48)  # runs past n


@pytest.mark.parametrize("log_n", [1, 7, 13])
def test_chunked_output_evaluation_is_the_definition(log_n):
    """fr_ntt_eval_output_chunk summed over uneven chunks equals the oracle's forward output k."""
    n = 1 << log_n
    a = orc.fr_to_mont(orc.rand_fr(pyref.SEED_NTT, 5, n))
    y = orc.array_to_ints(orc.fr_from_mont(orc.fr_ntt(a, log_n)))
    chunk = n // 3 + 1
    for k in {0, 1, n // 2, n - 1}:
        got = sum(orc.fr_ntt_eval_output_chunk(a[s:s + chunk], s, log_n, k) for s in range(0, n, chunk)) % pyref.R
        assert got == y[k], k
