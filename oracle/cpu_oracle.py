"""oracle/cpu_oracle.py -- TEST INFRASTRUCTURE ONLY: ctypes view of oracle/libb200zk_oracle.so.

Importable only from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs.  numpy arrays are the interchange type:
  * field element  : uint64[4] little-endian limbs (canonical or Montgomery as documented)
  * G1 native point: uint64[8]  = x|y Montgomery, (0,0) identity
  * G2 native point: uint64[16] = x.c0|x.c1|y.c0|y.c1 Montgomery
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libb200zk_oracle.so")


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "bn254_oracle.cpp")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        _lib.orc_chain_dot.restype = None
        _lib.orc_g1_msm.restype = C.c_int
        _lib.orc_g2_msm.restype = C.c_int
        _lib.orc_fr_ntt.restype = C.c_int
        _lib.orc_fr_ntt_identity_update.restype = C.c_int
        _lib.orc_fr_ntt_identity_check.restype = C.c_int
        _lib.orc_fr_ntt_eval_output_chunk.restype = C.c_int
    return _lib


def _p(a: np.ndarray):
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


def int_to_limbs(v: int) -> np.ndarray:
    return np.array([(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


def limbs_to_int(a) -> int:
    return sum(int(x) << (64 * i) for i, x in enumerate(a))


def ints_to_array(vals) -> np.ndarray:
    out = np.empty((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        out[i] = int_to_limbs(v)
    return out


def array_to_ints(a: np.ndarray):
    return [limbs_to_int(row) for row in a.reshape(-1, 4)]


def effective_cpus() -> int:
    """CPUs this process can really use: min(affinity mask, cgroup cpu.max quota).  Spawning one OpenMP
    thread per *visible* core under a smaller cgroup quota oversubscribes and runs slower."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if quota != "max":
            n = min(n, max(1, -(-int(quota) // int(period))))
    except Exception:  # noqa: BLE001
        pass
    return max(1, n)


def num_threads() -> int:
    """Threads the timed oracle calls use: every CPU the process may really use.  Deliberately NOT
    omp_get_max_threads(): torchrun exports OMP_NUM_THREADS=1 to its workers, which would silently turn the CPU
    baseline of a multi-rank bench into a single-thread run.  B200ZK_ORACLE_THREADS overrides."""
    env = os.environ.get("B200ZK_ORACLE_THREADS", "")
    if env.isdigit() and int(env) > 0:
        return int(env)
    return effective_cpus()


def _thr(threads: int) -> int:
    return threads if threads > 0 else num_threads()


def rand_fr(seed: int, start: int, n: int) -> np.ndarray:
    """canonical scalars, identical to pyref.rand_fr(seed, start+i)."""
    out = np.empty((n, 4), dtype=np.uint64)
    lib().orc_rand_fr(_p(out), C.c_uint64(seed), C.c_uint64(start), C.c_size_t(n))
    return out


def fr_to_mont(a: np.ndarray) -> np.ndarray:
    a = np.ascontiguousarray(a.copy())
    lib().orc_fr_to_mont(_p(a), C.c_size_t(a.size // 4))
    return a


def fr_from_mont(a: np.ndarray) -> np.ndarray:
    a = np.ascontiguousarray(a.copy())
    lib().orc_fr_from_mont(_p(a), C.c_size_t(a.size // 4))
    return a


def fq_to_mont(a: np.ndarray) -> np.ndarray:
    a = np.ascontiguousarray(a.copy())
    lib().orc_fq_to_mont(_p(a), C.c_size_t(a.size // 4))
    return a


def fq_from_mont(a: np.ndarray) -> np.ndarray:
    a = np.ascontiguousarray(a.copy())
    lib().orc_fq_from_mont(_p(a), C.c_size_t(a.size // 4))
    return a


def field_mul(field: str, a: np.ndarray, b: np.ndarray) -> np.ndarray:
    out = np.empty_like(a)
    getattr(lib(), f"orc_{field}_mul")(_p(a), _p(b), _p(out), C.c_size_t(a.size // 4))
    return out


def fr_quotient(a: np.ndarray, b: np.ndarray, c: np.ndarray, zinv: int, threads: int = 0) -> np.ndarray:
    """(a*b - c) * zinv element-wise; a, b, c Montgomery limbs, zinv an integer mod r"""
    out = np.empty_like(a)
    z = fr_to_mont(int_to_limbs(zinv).reshape(1, 4))
    lib().orc_fr_quotient(_p(a), _p(b), _p(c), _p(z), _p(out), C.c_size_t(a.size // 4), C.c_int(_thr(threads)))
    return out


def g1_chain(n: int, k: int, d: int, threads: int = 0) -> np.ndarray:
    out = np.empty((n, 8), dtype=np.uint64)
    lib().orc_g1_chain(_p(out), C.c_size_t(n), _p(int_to_limbs(k)), _p(int_to_limbs(d)), C.c_int(_thr(threads)))
    return out


def g2_chain(n: int, k: int, d: int, threads: int = 0) -> np.ndarray:
    out = np.empty((n, 16), dtype=np.uint64)
    lib().orc_g2_chain(_p(out), C.c_size_t(n), _p(int_to_limbs(k)), _p(int_to_limbs(d)), C.c_int(_thr(threads)))
    return out


def chain_dot(scalars: np.ndarray, k: int, d: int) -> int:
    out = np.empty(4, dtype=np.uint64)
    lib().orc_chain_dot(_p(scalars), C.c_size_t(scalars.size // 4), _p(int_to_limbs(k)), _p(int_to_limbs(d)), _p(out))
    return limbs_to_int(out)


def g1_be_to_native(be: bytes) -> np.ndarray:
    n = len(be) // 64
    out = np.empty((n, 8), dtype=np.uint64)
    rc = lib().orc_g1_be_to_native(C.c_char_p(be), _p(out), C.c_size_t(n))
    if rc:
        raise ValueError(f"g1 decode status {rc}")
    return out


def g1_native_to_be(a: np.ndarray) -> bytes:
    n = a.size // 8
    buf = C.create_string_buffer(64 * n)
    lib().orc_g1_native_to_be(_p(a), buf, C.c_size_t(n))
    return buf.raw


def g2_be_to_native(be: bytes) -> np.ndarray:
    n = len(be) // 128
    out = np.empty((n, 16), dtype=np.uint64)
    rc = lib().orc_g2_be_to_native(C.c_char_p(be), _p(out), C.c_size_t(n))
    if rc:
        raise ValueError(f"g2 decode status {rc}")
    return out


def g2_native_to_be(a: np.ndarray) -> bytes:
    n = a.size // 16
    buf = C.create_string_buffer(128 * n)
    lib().orc_g2_native_to_be(_p(a), buf, C.c_size_t(n))
    return buf.raw


def g1_add_be(p1: bytes, p2: bytes):
    buf = C.create_string_buffer(64)
    rc = lib().orc_g1_add_be(C.c_char_p(p1), C.c_char_p(p2), buf)
    return rc, buf.raw


def g1_mul_be(pt: bytes, scalar_be: bytes):
    buf = C.create_string_buffer(64)
    rc = lib().orc_g1_mul_be(C.c_char_p(pt), C.c_char_p(scalar_be), buf)
    return rc, buf.raw


def g2_mul_be(pt: bytes, scalar_be: bytes):
    buf = C.create_string_buffer(128)
    rc = lib().orc_g2_mul_be(C.c_char_p(pt), C.c_char_p(scalar_be), buf)
    return rc, buf.raw


def g1_msm(points: np.ndarray, scalars: np.ndarray, method: int = 0, threads: int = 0) -> bytes:
    n = scalars.size // 4
    assert points.size // 8 >= n
    buf = C.create_string_buffer(64)
    lib().orc_g1_msm(_p(points), _p(scalars), C.c_size_t(n), C.c_int(method), C.c_int(_thr(threads)), buf)
    return buf.raw


def g2_msm(points: np.ndarray, scalars: np.ndarray, method: int = 0, threads: int = 0) -> bytes:
    n = scalars.size // 4
    assert points.size // 16 >= n
    buf = C.create_string_buffer(128)
    lib().orc_g2_msm(_p(points), _p(scalars), C.c_size_t(n), C.c_int(method), C.c_int(_thr(threads)), buf)
    return buf.raw


NTT_INVERSE = 1
NTT_COSET = 2


def fr_ntt(data_mont: np.ndarray, log_n: int, flags: int = 0, coset_gen: int | None = None,
           root_2_28: int | None = None, threads: int = 0) -> np.ndarray:
    a = np.ascontiguousarray(data_mont.copy())
    assert a.size // 4 == 1 << log_n
    cg = _p(int_to_limbs(coset_gen)) if coset_gen is not None else None
    rt = _p(int_to_limbs(root_2_28)) if root_2_28 is not None else None
    rc = lib().orc_fr_ntt(_p(a), C.c_uint(log_n), C.c_uint(flags), cg, rt, C.c_int(_thr(threads)))
    if rc:
        raise ValueError(f"ntt status {rc}")
    return a


def fr_ntt_eval_output(data_mont: np.ndarray, log_n: int, k: int) -> np.ndarray:
    """output k of the forward NTT by direct evaluation (O(n)); Montgomery limbs in and out."""
    a = np.ascontiguousarray(data_mont)
    out = np.empty(4, dtype=np.uint64)
    rc = lib().orc_fr_ntt_eval_output(_p(a), C.c_uint(log_n), C.c_uint64(k), _p(out))
    if rc:
        raise ValueError(f"ntt eval status {rc}")
    return out


def fr_ntt_eval_output_chunk(chunk_mont: np.ndarray, start: int, log_n: int, k: int) -> int:
    """the share of coefficients [start, start + len(chunk)) in output k of the forward NTT, as an integer mod r: summed
    over the chunks of a vector it is output k by its definition, without holding the vector on the host."""
    a = np.ascontiguousarray(chunk_mont)
    out = np.empty((1, 4), dtype=np.uint64)
    rc = lib().orc_fr_ntt_eval_output_chunk(_p(a), C.c_size_t(a.size // 4), C.c_uint64(start), C.c_uint(log_n), C.c_uint64(k), _p(out))
    if rc:
        raise ValueError(f"ntt eval status {rc}")
    return limbs_to_int(fr_from_mont(out)[0])


class NttIdentity:
    """O(n) whole-vector check that y is the transform of a in one mode of fr_ntt, fed chunk by chunk.

    Every mode is y_k = s d^k sum_j a_j c^j w^(e j k), so at a point z
        sum_k y_k z^k = s ((dz)^n - 1) sum_j a_j c^j / (dz w^(e j) - 1);
    update() accumulates both sums over [start, start + len(chunk)) of a and y (Montgomery limbs, any chunking, each
    index once), ok() compares them.  Exact in Fr: a wrong output passes with probability <= n / r over z."""

    def __init__(self, log_n: int, flags: int = 0, coset_gen: int | None = None, root_2_28: int | None = None,
                 z: int = 0x1d3a7f5c9e2b48d06a1c3e5f7092b4d6e8fa1c3e5f70921b3d5f7a9cbedf0123, threads: int = 0):
        self.log_n, self.flags, self.threads = log_n, flags, threads
        self._keep = [int_to_limbs(z)]
        self._cg = self._keep_ptr(coset_gen)
        self._rt = self._keep_ptr(root_2_28)
        self._z = _p(self._keep[0])
        self.acc = np.zeros(8, dtype=np.uint64)
        self.seen = 0

    def _keep_ptr(self, v):
        if v is None:
            return None
        self._keep.append(int_to_limbs(v))
        return _p(self._keep[-1])

    def update(self, inp_mont: np.ndarray, out_mont: np.ndarray, start: int) -> None:
        a, y = np.ascontiguousarray(inp_mont), np.ascontiguousarray(out_mont)
        assert a.size == y.size and a.size % 4 == 0
        rc = lib().orc_fr_ntt_identity_update(_p(a), _p(y), C.c_size_t(start), C.c_size_t(a.size // 4), C.c_uint(self.log_n),
                                              C.c_uint(self.flags), self._cg, self._rt, self._z, _p(self.acc), C.c_int(_thr(self.threads)))
        if rc:
            raise ValueError(f"ntt identity status {rc}")
        self.seen += a.size // 4

    def ok(self) -> bool:
        assert self.seen == 1 << self.log_n, f"fed {self.seen} of {1 << self.log_n} indices"
        rc = lib().orc_fr_ntt_identity_check(_p(self.acc), C.c_uint(self.log_n), C.c_uint(self.flags), self._cg, self._rt, self._z)
        if rc not in (0, 1):
            raise ValueError(f"ntt identity status {rc}")
        return rc == 1


def fr_ntt_identity(inp_mont: np.ndarray, out_mont: np.ndarray, log_n: int, flags: int = 0, coset_gen: int | None = None,
                    root_2_28: int | None = None, chunk: int = 1 << 20) -> bool:
    """NttIdentity over two whole vectors held on the host"""
    chk = NttIdentity(log_n, flags, coset_gen, root_2_28)
    a, y = inp_mont.reshape(-1, 4), out_mont.reshape(-1, 4)
    for s in range(0, 1 << log_n, chunk):
        chk.update(a[s:s + chunk], y[s:s + chunk], s)
    return chk.ok()
