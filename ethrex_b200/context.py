"""Host-side handle on one H100: the Python mirror of the `B200zk` wrapper in rust/ethrex-backend.

One `Context` per process per GPU (SURVEY.md section 8b: the reference's prover actor runs on one
blocking thread, `/root/reference/crates/prover/src/prover.rs:240-251`, and scales out as one process
per GPU, `/root/reference/docs/l2/fundamentals/distributed_proving.md:36-50`).

Host entry points take numpy arrays / bytes (the buffers the Rust backend would pass); device entry
points take torch CUDA tensors, which are used only as owners of device memory and as the source of the
current stream -- all arithmetic happens in libb200zk.so.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _ffi as F
from .errors import B200Error, NoDeviceError, status_to_error


def _host_ptr(buf):
    """(pointer, keepalive) for bytes / bytearray / numpy input."""
    if isinstance(buf, np.ndarray):
        if not buf.flags["C_CONTIGUOUS"]:
            raise B200Error.serialization("host buffer must be C-contiguous")
        return buf.ctypes.data_as(C.c_void_p), buf
    if isinstance(buf, (bytes, bytearray, memoryview)):
        arr = np.frombuffer(buf, dtype=np.uint8)
        return arr.ctypes.data_as(C.c_void_p), arr
    if hasattr(buf, "data_ptr"):  # a (pinned) CPU torch tensor
        if buf.is_cuda:
            raise B200Error.serialization("expected a host buffer, got a CUDA tensor")
        return C.c_void_p(buf.data_ptr()), buf
    raise B200Error.serialization(f"unsupported host buffer type {type(buf)!r}")


def _dev_ptr(t):
    if not (hasattr(t, "is_cuda") and t.is_cuda):
        raise B200Error.serialization("expected a CUDA tensor")
    if not t.is_contiguous():
        raise B200Error.serialization("device tensor must be contiguous")
    return C.c_void_p(t.data_ptr())


_CUDA_STREAM_LEGACY = 0x1  # cudaStreamLegacy: the C ABI reserves NULL for "the context's own stream"


def _current_stream_ptr(device=None):
    """torch's current stream ON THE CONTEXT'S DEVICE, so library work is ordered with the caller's tensors and events
    (torch's current device may be another GPU)."""
    import torch
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream or _CUDA_STREAM_LEGACY)


def _host_len(buf) -> int:
    """bytes a host buffer holds (numpy / bytes-like / CPU torch tensor)"""
    if isinstance(buf, np.ndarray):
        return buf.nbytes
    if isinstance(buf, (bytes, bytearray)):
        return len(buf)
    if isinstance(buf, memoryview):
        return buf.nbytes
    if hasattr(buf, "element_size"):
        return buf.numel() * buf.element_size()
    raise B200Error.serialization(f"unsupported host buffer type {type(buf)!r}")


def _need(buf, nbytes: int, what: str):
    """the library copies `nbytes` out of (or into) the caller's buffer: refuse short buffers here instead of reading
    past their end (the Rust wrapper checks the same way, rust/ethrex-backend/src/ffi.rs)"""
    have = _host_len(buf)
    if have < nbytes:
        raise B200Error.serialization(f"{what}: buffer holds {have} bytes, the call needs {nbytes}")


class Context:
    def __init__(self, device: int = 0):
        h = C.c_void_p()
        rc = F.lib.b200zk_init(device, C.byref(h))
        if rc == F.ERR_NO_DEVICE:
            raise NoDeviceError("b200zk_init: no CUDA device -- libb200zk has no CPU fallback")
        if rc != F.OK:
            raise B200Error.proving(f"b200zk_init(device={device}): {F.lib.b200zk_strerror(rc).decode()}")
        self._h = h
        self.device = device

    # ------------------------------------------------------------------ lifecycle
    def close(self):
        if getattr(self, "_h", None):
            F.lib.b200zk_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _check(self, rc: int, what: str) -> int:
        if rc > F.OK_INFINITY:
            detail = F.lib.b200zk_last_error(self._h).decode(errors="replace")
            raise status_to_error(rc, f"{what}: {F.lib.b200zk_strerror(rc).decode()} ({detail})")
        return rc

    @property
    def launch_count(self) -> int:
        return int(F.lib.b200zk_launch_count(self._h))

    def synchronize(self):
        self._check(F.lib.b200zk_synchronize(self._h), "synchronize")

    def set_msm_window(self, c: int):
        self._check(F.lib.b200zk_set_msm_window(self._h, c), "set_msm_window")

    def set_msm_chunks(self, chunks: int):
        self._check(F.lib.b200zk_set_msm_chunks(self._h, chunks), "set_msm_chunks")

    def set_msm_pair_rounds(self, rounds: int):
        self._check(F.lib.b200zk_set_msm_pair_rounds(self._h, rounds), "set_msm_pair_rounds")

    def set_profiling(self, on: bool):
        self._check(F.lib.b200zk_set_profiling(self._h, 1 if on else 0), "set_profiling")

    def last_msm_phase_ms(self):
        out = (C.c_float * 6)()
        self._check(F.lib.b200zk_last_msm_phase_ms(self._h, out), "last_msm_phase_ms")
        return dict(zip(("hist", "scan", "scatter", "accumulate", "bucket_reduce", "horner"), (float(x) for x in out)))

    # ------------------------------------------------------------------ batched precompile arithmetic
    # Twins of Crypto::{bn254_g1_add, bn254_g1_mul, bn254_pairing_check}
    # (/root/reference/crates/common/crypto/provider.rs:201-330); per-item status as in include/b200zk.h.
    def bn254_g1_add_batch(self, a: bytes, b: bytes):
        """a, b: count*64 bytes each -> (count*64 result bytes, [status])"""
        if len(a) != len(b) or len(a) % 64:
            raise B200Error.serialization("G1 point must be 64 bytes")
        count = len(a) // 64
        out, st = C.create_string_buffer(max(1, 64 * count)), C.create_string_buffer(max(1, count))
        pa, k1 = _host_ptr(a)
        pb, k2 = _host_ptr(b)
        self._check(F.lib.b200zk_bn254_g1_add_batch(self._h, pa, pb, count, out, st), "bn254_g1_add_batch")
        return out.raw[:64 * count], list(st.raw[:count])

    def bn254_g1_mul_batch(self, points: bytes, scalars: bytes):
        if len(points) % 64 or len(scalars) != len(points) // 2:
            raise B200Error.serialization("invalid input length")
        count = len(points) // 64
        out, st = C.create_string_buffer(max(1, 64 * count)), C.create_string_buffer(max(1, count))
        pp, k1 = _host_ptr(points)
        ps, k2 = _host_ptr(scalars)
        self._check(F.lib.b200zk_bn254_g1_mul_batch(self._h, pp, ps, count, out, st), "bn254_g1_mul_batch")
        return out.raw[:64 * count], list(st.raw[:count])

    def bn254_pairing_check_batch(self, checks):
        """checks: list of calldata byte strings (k*192 bytes each, the ecpairing precompile's input) ->
        ([result 0/1], [status])"""
        offs, blob = [0], bytearray()
        for cd in checks:
            if len(cd) % 192:
                raise B200Error.serialization("ecpairing input must be a multiple of 192 bytes")
            blob += cd
            offs.append(len(blob) // 192)
        count = len(checks)
        offsets = np.asarray(offs, dtype=np.uint32)
        res, st = C.create_string_buffer(max(1, count)), C.create_string_buffer(max(1, count))
        pairs = np.frombuffer(bytes(blob) or b"\0", dtype=np.uint8)
        self._check(F.lib.b200zk_bn254_pairing_check_batch(self._h, pairs.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p),
                                                          count, res, st), "bn254_pairing_check_batch")
        return list(res.raw[:count]), list(st.raw[:count])

    # ------------------------------------------------------------------ host-buffer entry points
    def g1_msm(self, points, scalars, n: int, flags: int = 0) -> bytes:
        return self._msm_host(F.lib.b200zk_g1_msm, 64, points, scalars, n, flags)

    def g2_msm(self, points, scalars, n: int, flags: int = 0) -> bytes:
        return self._msm_host(F.lib.b200zk_g2_msm, 128, points, scalars, n, flags)

    def _msm_host(self, fn, out_bytes, points, scalars, n, flags):
        _need(points, n * out_bytes, fn.__name__ + " points")
        _need(scalars, n * 32, fn.__name__ + " scalars")
        pp, k1 = _host_ptr(points)
        sp, k2 = _host_ptr(scalars)
        out = C.create_string_buffer(out_bytes)
        self._check(fn(self._h, pp, sp, n, flags, out), fn.__name__)
        return out.raw

    def fr_ntt(self, data, log_n: int, flags: int = 0, coset_gen: bytes | None = None):
        """In place on a host buffer of 2^log_n 32-byte elements."""
        if not 0 <= log_n <= 28:
            raise B200Error.serialization("fr_ntt: log_n must be 0..28")
        _need(data, 32 << log_n, "b200zk_fr_ntt data")
        dp, keep = _host_ptr(data)
        cg = C.c_char_p(coset_gen) if coset_gen is not None else None
        self._check(F.lib.b200zk_fr_ntt(self._h, dp, log_n, flags, C.cast(cg, C.c_void_p) if cg else None), "b200zk_fr_ntt")
        return data

    def g1_bases_upload(self, points, n: int, flags: int = 0) -> int:
        _need(points, 64 * n, "b200zk_g1_bases_upload points")
        pp, keep = _host_ptr(points)
        h = C.c_uint64()
        self._check(F.lib.b200zk_g1_bases_upload(self._h, pp, n, flags, C.byref(h)), "b200zk_g1_bases_upload")
        return h.value

    def g2_bases_upload(self, points, n: int, flags: int = 0) -> int:
        _need(points, 128 * n, "b200zk_g2_bases_upload points")
        pp, keep = _host_ptr(points)
        h = C.c_uint64()
        self._check(F.lib.b200zk_g2_bases_upload(self._h, pp, n, flags, C.byref(h)), "b200zk_g2_bases_upload")
        return h.value

    def g1_bases_from_device(self, d_points, n: int) -> int:
        h = C.c_uint64()
        self._check(F.lib.b200zk_g1_bases_from_device(self._h, _dev_ptr(d_points), n, _current_stream_ptr(self.device), C.byref(h)), "b200zk_g1_bases_from_device")
        return h.value

    def g2_bases_from_device(self, d_points, n: int) -> int:
        h = C.c_uint64()
        self._check(F.lib.b200zk_g2_bases_from_device(self._h, _dev_ptr(d_points), n, _current_stream_ptr(self.device), C.byref(h)), "b200zk_g2_bases_from_device")
        return h.value

    def bases_precompute(self, handle: int, window_bits: int = 0):
        """One-off: expand resident bases into their window multiples 2^(c*w)*P_i (fewer additions per MSM)."""
        self._check(F.lib.b200zk_bases_precompute(self._h, handle, window_bits), "b200zk_bases_precompute")

    def g1_msm_resident_device(self, handle: int, d_scalars, n: int, flags: int = 0) -> bytes:
        out = C.create_string_buffer(64)
        self._check(F.lib.b200zk_g1_msm_resident_device(self._h, handle, _dev_ptr(d_scalars), n, flags, _current_stream_ptr(self.device), out), "b200zk_g1_msm_resident_device")
        return out.raw

    def g2_msm_resident_device(self, handle: int, d_scalars, n: int, flags: int = 0) -> bytes:
        out = C.create_string_buffer(128)
        self._check(F.lib.b200zk_g2_msm_resident_device(self._h, handle, _dev_ptr(d_scalars), n, flags, _current_stream_ptr(self.device), out), "b200zk_g2_msm_resident_device")
        return out.raw

    def bases_free(self, handle: int):
        self._check(F.lib.b200zk_bases_free(self._h, handle), "b200zk_bases_free")

    def msm_multi_resident_device(self, handles, is_g2, d_scalars, n: int, flags: int = 0):
        """MSMs of several resident columns against ONE device scalar vector, sharing the scalar sort.
        handles: list of base handles; is_g2: matching list of booleans -> list of result byte strings (64 / 128 B)."""
        count = len(handles)
        hs = (C.c_uint64 * max(1, count))(*handles)
        out = C.create_string_buffer(max(1, 128 * count))
        st = (C.c_int * max(1, count))()
        self._check(F.lib.b200zk_msm_multi_resident_device(self._h, hs, count, _dev_ptr(d_scalars), n, flags, _current_stream_ptr(self.device), out, st),
                    "b200zk_msm_multi_resident_device")
        return [out.raw[128 * i:128 * i + (128 if g2 else 64)] for i, g2 in enumerate(is_g2)]

    def g1_msm_resident(self, handle: int, scalars, n: int, flags: int = 0) -> bytes:
        _need(scalars, 32 * n, "b200zk_g1_msm_resident scalars")
        sp, keep = _host_ptr(scalars)
        out = C.create_string_buffer(64)
        self._check(F.lib.b200zk_g1_msm_resident(self._h, handle, sp, n, flags, out), "b200zk_g1_msm_resident")
        return out.raw

    def g2_msm_resident(self, handle: int, scalars, n: int, flags: int = 0) -> bytes:
        _need(scalars, 32 * n, "b200zk_g2_msm_resident scalars")
        sp, keep = _host_ptr(scalars)
        out = C.create_string_buffer(128)
        self._check(F.lib.b200zk_g2_msm_resident(self._h, handle, sp, n, flags, out), "b200zk_g2_msm_resident")
        return out.raw

    # ------------------------------------------------------------------ device-pointer entry points
    def g1_msm_device(self, d_points, d_scalars, n: int, flags: int = 0) -> bytes:
        out = C.create_string_buffer(64)
        self._check(F.lib.b200zk_g1_msm_device(self._h, _dev_ptr(d_points), _dev_ptr(d_scalars), n, flags, _current_stream_ptr(self.device), out), "b200zk_g1_msm_device")
        return out.raw

    def g2_msm_device(self, d_points, d_scalars, n: int, flags: int = 0) -> bytes:
        out = C.create_string_buffer(128)
        self._check(F.lib.b200zk_g2_msm_device(self._h, _dev_ptr(d_points), _dev_ptr(d_scalars), n, flags, _current_stream_ptr(self.device), out), "b200zk_g2_msm_device")
        return out.raw

    def g1_msm_device_async(self, d_points, d_scalars, n: int, d_out, flags: int = 0):
        """d_out: device buffer of at least 68 bytes = point (64) | u32 is_infinity (ABI v2)"""
        if d_out.numel() * d_out.element_size() < 68:
            raise B200Error.serialization("g1_msm_device_async: d_out must hold 64 + 4 bytes")
        self._check(F.lib.b200zk_g1_msm_device_async(self._h, _dev_ptr(d_points), _dev_ptr(d_scalars), n, flags, _current_stream_ptr(self.device), _dev_ptr(d_out)), "b200zk_g1_msm_device_async")

    def g2_msm_device_async(self, d_points, d_scalars, n: int, d_out, flags: int = 0):
        """d_out: device buffer of at least 132 bytes = point (128) | u32 is_infinity (ABI v2)"""
        if d_out.numel() * d_out.element_size() < 132:
            raise B200Error.serialization("g2_msm_device_async: d_out must hold 128 + 4 bytes")
        self._check(F.lib.b200zk_g2_msm_device_async(self._h, _dev_ptr(d_points), _dev_ptr(d_scalars), n, flags, _current_stream_ptr(self.device), _dev_ptr(d_out)), "b200zk_g2_msm_device_async")

    def fr_ntt_device(self, d_data, log_n: int, flags: int = 0, coset_gen: bytes | None = None):
        cg = C.cast(C.c_char_p(coset_gen), C.c_void_p) if coset_gen is not None else None
        self._check(F.lib.b200zk_fr_ntt_device(self._h, _dev_ptr(d_data), log_n, flags, cg, _current_stream_ptr(self.device)), "b200zk_fr_ntt_device")

    # ------------------------------------------------------------------ BLS12-381 G1 / EIP-4844 blob commitments (SURVEY.md 8f row 3)
    def bls12_381_g1_bases_upload(self, points, n: int, flags: int = F.POINTS_COMPRESSED) -> int:
        """points: n x 48 bytes compressed (default, the trusted setup's form) or n x 96 bytes uncompressed (flags=0)"""
        _need(points, n * (48 if flags & F.POINTS_COMPRESSED else 96), "b200zk_bls12_381_g1_bases_upload points")
        pp, keep = _host_ptr(points)
        h = C.c_uint64()
        self._check(F.lib.b200zk_bls12_381_g1_bases_upload(self._h, pp, n, flags, C.byref(h)), "b200zk_bls12_381_g1_bases_upload")
        return h.value

    def bls12_381_g1_msm_resident(self, handle: int, scalars, n: int, flags: int = F.SCALARS_BE) -> bytes:
        """-> 48 bytes compressed; scalars 32-byte big-endian (default) or little-endian limbs, each < the group order"""
        _need(scalars, 32 * n, "b200zk_bls12_381_g1_msm_resident scalars")
        sp, keep = _host_ptr(scalars)
        out = C.create_string_buffer(48)
        self._check(F.lib.b200zk_bls12_381_g1_msm_resident(self._h, handle, sp, n, flags, out), "b200zk_bls12_381_g1_msm_resident")
        return out.raw

    def kzg_blob_to_commitment(self, setup_handle: int, blobs) -> list:
        """blobs: bytes-like of k x 131072 bytes (4096 x 32-byte big-endian field elements each) -> [48-byte commitments]"""
        total = _host_len(blobs)
        if total % (4096 * 32):
            raise B200Error.serialization("a blob is 4096 x 32 bytes")
        k = total // (4096 * 32)
        bp, keep = _host_ptr(blobs)
        out = C.create_string_buffer(max(1, 48 * k))
        self._check(F.lib.b200zk_kzg_blob_to_commitment(self._h, setup_handle, bp, k, out), "b200zk_kzg_blob_to_commitment")
        return [out.raw[48 * i:48 * i + 48] for i in range(k)]

    @staticmethod
    def _blob_count(blobs) -> int:
        total = _host_len(blobs)
        if total % (4096 * 32):
            raise B200Error.serialization("a blob is 4096 x 32 bytes")
        return total // (4096 * 32)

    def kzg_blob_to_commitment_and_proof(self, setup_handle: int, blobs) -> tuple:
        """blobs: k x 131072 bytes -> ([48-byte commitments], [48-byte proofs at the EIP-4844 Fiat-Shamir challenge])"""
        k = self._blob_count(blobs)
        bp, keep = _host_ptr(blobs)
        cm, pr = C.create_string_buffer(max(1, 48 * k)), C.create_string_buffer(max(1, 48 * k))
        self._check(F.lib.b200zk_kzg_blob_to_commitment_and_proof(self._h, setup_handle, bp, k, cm, pr), "b200zk_kzg_blob_to_commitment_and_proof")
        return [cm.raw[48 * i:48 * i + 48] for i in range(k)], [pr.raw[48 * i:48 * i + 48] for i in range(k)]

    def kzg_compute_proof(self, setup_handle: int, blobs, z) -> tuple:
        """blobs: k x 131072 bytes, z: k x 32-byte big-endian -> ([48-byte proofs], [y = p(z), 32-byte big-endian])"""
        k = self._blob_count(blobs)
        _need(z, 32 * k, "b200zk_kzg_compute_proof z")
        bp, keep = _host_ptr(blobs)
        zp, keep_z = _host_ptr(z)
        pr, y = C.create_string_buffer(max(1, 48 * k)), C.create_string_buffer(max(1, 32 * k))
        self._check(F.lib.b200zk_kzg_compute_proof(self._h, setup_handle, bp, k, zp, pr, y), "b200zk_kzg_compute_proof")
        return [pr.raw[48 * i:48 * i + 48] for i in range(k)], [y.raw[32 * i:32 * i + 32] for i in range(k)]

    # ------------------------------------------------------------------ BLS12-381 pairing / EIP-4844 KZG verification
    def bls12_381_g2_bases_upload(self, points, n: int, flags: int = F.POINTS_COMPRESSED) -> int:
        """points: n x 96 bytes compressed G2 (the trusted setup's g2_monomial form); subgroup-checked"""
        _need(points, 96 * n, "b200zk_bls12_381_g2_bases_upload points")
        pp, keep = _host_ptr(points)
        h = C.c_uint64()
        self._check(F.lib.b200zk_bls12_381_g2_bases_upload(self._h, pp, n, flags, C.byref(h)), "b200zk_bls12_381_g2_bases_upload")
        return h.value

    def bls12_381_pairing_check_batch(self, checks):
        """checks: list of EIP-2537 pairing calldata byte strings (k*384 bytes each) -> ([result 0/1], [status])"""
        offs, blob = [0], bytearray()
        for cd in checks:
            if len(cd) % 384:
                raise B200Error.serialization("bls12 pairing input must be a multiple of 384 bytes")
            blob += cd
            offs.append(len(blob) // 384)
        count = len(checks)
        offsets = np.asarray(offs, dtype=np.uint32)
        res, st = C.create_string_buffer(max(1, count)), C.create_string_buffer(max(1, count))
        pairs = np.frombuffer(bytes(blob) or b"\0", dtype=np.uint8)
        self._check(F.lib.b200zk_bls12_381_pairing_check_batch(self._h, pairs.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p),
                                                              count, res, st), "b200zk_bls12_381_pairing_check_batch")
        return list(res.raw[:count]), list(st.raw[:count])

    # ------------------------------------------------------------------ EIP-2537 addition and MSM (precompiles 0x0b-0x0e)
    # Twins of Crypto::bls12_381_{g1,g2}_{add,msm} (/root/reference/crates/common/crypto/provider.rs:549-640); EIP-2537
    # encodings and per-item status as in include/b200zk.h.
    def _bls12_add(self, fn, what: str, a, b, size: int):
        if len(a) != len(b) or len(a) % size:
            raise B200Error.serialization(f"{what}: inputs must be equal multiples of {size} bytes")
        count = len(a) // size
        out, st = C.create_string_buffer(max(1, size * count)), C.create_string_buffer(max(1, count))
        pa, k1 = _host_ptr(a)
        pb, k2 = _host_ptr(b)
        self._check(fn(self._h, pa, pb, count, out, st), what)
        return out.raw[:size * count], list(st.raw[:count])

    def _bls12_msm(self, fn, what: str, calls, pair: int, size: int):
        offs, blob = [0], bytearray()
        for cd in calls:
            if len(cd) % pair:
                raise B200Error.serialization(f"{what}: calldata must be a multiple of {pair} bytes")
            blob += cd
            offs.append(len(blob) // pair)
        count = len(calls)
        offsets = np.asarray(offs, dtype=np.uint32)
        out, st = C.create_string_buffer(max(1, size * count)), C.create_string_buffer(max(1, count))
        pairs = np.frombuffer(bytes(blob) or b"\0", dtype=np.uint8)
        self._check(fn(self._h, pairs.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p), count, out, st), what)
        return [out.raw[size * i:size * (i + 1)] for i in range(count)], list(st.raw[:count])

    def bls12_381_g1_add_batch(self, a: bytes, b: bytes):
        """a, b: count x 128 bytes (EIP-2537 G1) each -> (count x 128 result bytes, [status])"""
        return self._bls12_add(F.lib.b200zk_bls12_381_g1_add_batch, "b200zk_bls12_381_g1_add_batch", a, b, 128)

    def bls12_381_g2_add_batch(self, a: bytes, b: bytes):
        """a, b: count x 256 bytes (EIP-2537 G2) each -> (count x 256 result bytes, [status])"""
        return self._bls12_add(F.lib.b200zk_bls12_381_g2_add_batch, "b200zk_bls12_381_g2_add_batch", a, b, 256)

    def bls12_381_g1_msm_batch(self, calls):
        """calls: list of G1MSM calldata byte strings (k x 160 bytes each) -> ([128-byte output per call], [status])"""
        return self._bls12_msm(F.lib.b200zk_bls12_381_g1_msm_batch, "b200zk_bls12_381_g1_msm_batch", calls, 160, 128)

    def bls12_381_g2_msm_batch(self, calls):
        """calls: list of G2MSM calldata byte strings (k x 288 bytes each) -> ([256-byte output per call], [status])"""
        return self._bls12_msm(F.lib.b200zk_bls12_381_g2_msm_batch, "b200zk_bls12_381_g2_msm_batch", calls, 288, 256)

    # ------------------------------------------------------------------ secp256k1 signer recovery (ECRECOVER)
    def secp256k1_ecrecover_batch(self, sigs, msgs, low_s: bool = False):
        """sigs: count x 65 bytes (r | s | recid), msgs: count x 32-byte hashes -> (count x 32 bytes, [status]).
        Item i's 32 bytes are keccak256 of the recovered public key (the address is bytes 12..32), zero when status[i]
        != 0 (2 InvalidSignature, 3 RecoveryFailed, 4 InvalidRecoveryId).  low_s: EIP-2's s <= n/2, as recover_signer."""
        ns, nm = _host_len(sigs), _host_len(msgs)
        if ns % 65 or nm % 32 or ns // 65 != nm // 32:
            raise B200Error.serialization("b200zk_secp256k1_ecrecover_batch: sigs must be count x 65 bytes and msgs count x 32 bytes")
        count = ns // 65
        sp, k1 = _host_ptr(sigs) if count else (None, None)
        mp, k2 = _host_ptr(msgs) if count else (None, None)
        out, st = C.create_string_buffer(max(1, 32 * count)), C.create_string_buffer(max(1, count))
        self._check(F.lib.b200zk_secp256k1_ecrecover_batch(self._h, sp, mp, count, F.ECRECOVER_LOW_S if low_s else 0, out, st),
                    "b200zk_secp256k1_ecrecover_batch")
        return out.raw[:32 * count], list(st.raw[:count])

    # ------------------------------------------------------------------ P-256 signature verification (P256VERIFY)
    def secp256r1_verify_batch(self, inputs) -> list:
        """inputs: count x 160 bytes, the P256VERIFY calldata h | r | s | qx | qy each -> [bool] per item (EIP-7951:
        True when the signature verifies; malformed or off-curve items are False)."""
        n = _host_len(inputs)
        if n % 160:
            raise B200Error.serialization("b200zk_secp256r1_verify_batch: inputs must be count x 160 bytes")
        count = n // 160
        ip, keep = _host_ptr(inputs) if count else (None, None)
        res = C.create_string_buffer(max(1, count))
        self._check(F.lib.b200zk_secp256r1_verify_batch(self._h, ip, count, res), "b200zk_secp256r1_verify_batch")
        return [b == 1 for b in res.raw[:count]]

    def kzg_verify_proof_batch(self, g2_setup: int, commitments, z, y, proofs) -> tuple:
        """n items: commitments and proofs n x 48 bytes, z and y n x 32-byte big-endian -> ([result 0/1], [status])"""
        n = _host_len(commitments) // 48
        _need(z, 32 * n, "b200zk_kzg_verify_proof_batch z")
        _need(y, 32 * n, "b200zk_kzg_verify_proof_batch y")
        _need(proofs, 48 * n, "b200zk_kzg_verify_proof_batch proofs")
        bufs = [_host_ptr(b) for b in (commitments, z, y, proofs)]
        res, st = C.create_string_buffer(max(1, n)), C.create_string_buffer(max(1, n))
        self._check(F.lib.b200zk_kzg_verify_proof_batch(self._h, g2_setup, *[p for p, _ in bufs], n, res, st), "b200zk_kzg_verify_proof_batch")
        return list(res.raw[:n]), list(st.raw[:n])

    def kzg_verify_blob_proof_batch(self, g2_setup: int, blobs, commitments, proofs) -> bool:
        """blobs: k x 131072 bytes, commitments and proofs k x 48 bytes -> one bool for the batch"""
        k = self._blob_count(blobs)
        _need(commitments, 48 * k, "b200zk_kzg_verify_blob_proof_batch commitments")
        _need(proofs, 48 * k, "b200zk_kzg_verify_blob_proof_batch proofs")
        bufs = [_host_ptr(b) if _host_len(b) else (None, None) for b in (blobs, commitments, proofs)]
        valid = C.c_int(-1)
        self._check(F.lib.b200zk_kzg_verify_blob_proof_batch(self._h, g2_setup, *[p for p, _ in bufs], k, C.byref(valid)),
                    "b200zk_kzg_verify_blob_proof_batch")
        return valid.value == 1

    # ------------------------------------------------------------------ EIP-7594 cells (PeerDAS, wrapper version 1)
    def kzg_compute_cells(self, blobs) -> list:
        """blobs: k x 131072 bytes -> k lists of 128 cells, 2048 bytes each (64 x 32-byte big-endian elements)"""
        k = self._blob_count(blobs)
        bp, keep = _host_ptr(blobs) if k else (None, None)
        out = C.create_string_buffer(max(1, 262144 * k))
        self._check(F.lib.b200zk_kzg_compute_cells(self._h, bp, k, out), "b200zk_kzg_compute_cells")
        raw = out.raw
        return [[raw[262144 * b + 2048 * c:262144 * b + 2048 * (c + 1)] for c in range(128)] for b in range(k)]

    def kzg_blob_to_commitment_and_cell_proofs(self, g1_lagrange: int, g1_monomial: int, blobs) -> tuple:
        """blobs: k x 131072 bytes -> ([48-byte commitments], [48-byte cell proofs]), the proofs blob-major (128 per blob, cell
        index inner).  g1_monomial: a 4096-point G1 handle of the setup's [tau^i]1 points."""
        k = self._blob_count(blobs)
        bp, keep = _host_ptr(blobs) if k else (None, None)
        cm, pr = C.create_string_buffer(max(1, 48 * k)), C.create_string_buffer(max(1, 128 * 48 * k))
        self._check(F.lib.b200zk_kzg_blob_to_commitment_and_cell_proofs(self._h, g1_lagrange, g1_monomial, bp, k, cm, pr),
                    "b200zk_kzg_blob_to_commitment_and_cell_proofs")
        return [cm.raw[48 * i:48 * i + 48] for i in range(k)], [pr.raw[48 * i:48 * i + 48] for i in range(128 * k)]

    def kzg_verify_cell_proof_batch(self, g1_setup: int, g2_setup: int, blobs, commitments, proofs) -> bool:
        """blobs: k x 131072 bytes, commitments k x 48 bytes, proofs k x 128 x 48 bytes (blob-major, cell index inner) ->
        one bool for every cell of every blob"""
        k = self._blob_count(blobs)
        _need(commitments, 48 * k, "b200zk_kzg_verify_cell_proof_batch commitments")
        _need(proofs, 128 * 48 * k, "b200zk_kzg_verify_cell_proof_batch proofs")
        bufs = [_host_ptr(b) if _host_len(b) else (None, None) for b in (blobs, commitments, proofs)]
        valid = C.c_int(-1)
        self._check(F.lib.b200zk_kzg_verify_cell_proof_batch(self._h, g1_setup, g2_setup, *[p for p, _ in bufs], k, C.byref(valid)),
                    "b200zk_kzg_verify_cell_proof_batch")
        return valid.value == 1

    # ------------------------------------------------------------------ NTT root of unity (SURVEY.md section 8c)
    NTT_ROOT_ARK, NTT_ROOT_HALO2 = 0, 1

    @staticmethod
    def ntt_root_preset(preset: int) -> bytes:
        out = C.create_string_buffer(32)
        if F.lib.b200zk_ntt_root_preset(preset, out) != F.OK:
            raise B200Error.serialization(f"unknown NTT root preset {preset}")
        return out.raw

    def set_ntt_root(self, root_le: bytes | None):
        """root_le: canonical little-endian 32 bytes of a primitive 2^28-th root of unity of Fr; None = the ark/gnark default"""
        if root_le is not None and len(root_le) != 32:
            raise B200Error.serialization("NTT root must be 32 bytes")
        self._check(F.lib.b200zk_set_ntt_root(self._h, C.cast(C.c_char_p(root_le), C.c_void_p) if root_le is not None else None), "b200zk_set_ntt_root")

    # ------------------------------------------------------------------ Groth16 prove arithmetic in one call
    @staticmethod
    def groth16_pk(log_n: int, handles, counts, offsets) -> "F.Groth16Pk":
        """columns 0..4 = A_g1, B_g1 (handle 0 = absent), B_g2, L_g1, H_g1"""
        pk = F.Groth16Pk()
        pk.log_n, pk.reserved = log_n, 0
        for k in range(5):
            pk.handle[k], pk.count[k], pk.offset[k] = handles[k], counts[k], offsets[k]
        return pk

    def _g16_ptrs(self, pk, witness, a, b, c, flags):
        if flags & F.G16_INPUTS_DEVICE:
            ptr = lambda t: _dev_ptr(t) if t is not None else None  # noqa: E731
            return ptr(witness), ptr(a), ptr(b), ptr(c), None
        n = 1 << pk.log_n
        wit_end = max(pk.offset[k] + pk.count[k] for k in range(4) if pk.handle[k])
        _need(witness, 32 * wit_end, "b200zk_groth16_commit witness")
        keep, out = [], []
        for nm, buf in (("a_evals", a), ("b_evals", b), ("c_evals", c)):
            if buf is None:
                out.append(None)
                continue
            _need(buf, 32 * n, "b200zk_groth16_commit " + nm)
            pp, k = _host_ptr(buf)
            out.append(pp); keep.append(k)
        wp, kw = _host_ptr(witness)
        keep.append(kw)
        return wp, out[0], out[1], out[2], keep

    def groth16_commit(self, pk, witness, a_evals, b_evals, c_evals, flags: int = 0):
        """-> (proof 256 bytes = A | B2 | C, [B]1 64 bytes).  Host buffers, or device tensors with G16_INPUTS_DEVICE."""
        wp, ap, bp, cp, keep = self._g16_ptrs(pk, witness, a_evals, b_evals, c_evals, flags)
        proof, b1 = C.create_string_buffer(256), C.create_string_buffer(64)
        self._check(F.lib.b200zk_groth16_commit(self._h, C.byref(pk), wp, ap, bp, cp, flags, _current_stream_ptr(self.device), proof, b1), "b200zk_groth16_commit")
        return proof.raw, b1.raw

    def groth16_commit_partial(self, pk, witness, a_evals, b_evals, c_evals, d_partials, flags: int = 0):
        """asynchronous: leaves this rank's 768-byte block of XYZZ partial sums in d_partials (device tensor)"""
        if d_partials.numel() * d_partials.element_size() < 768:
            raise B200Error.serialization("groth16_commit_partial: d_partials must hold 768 bytes")
        wp, ap, bp, cp, keep = self._g16_ptrs(pk, witness, a_evals, b_evals, c_evals, flags)
        self._check(F.lib.b200zk_groth16_commit_partial(self._h, C.byref(pk), wp, ap, bp, cp, flags, _current_stream_ptr(self.device), _dev_ptr(d_partials)), "b200zk_groth16_commit_partial")

    def groth16_fold(self, d_partials, count: int):
        if d_partials.numel() * d_partials.element_size() < 768 * count:
            raise B200Error.serialization("groth16_fold: d_partials must hold 768 bytes per block")
        proof, b1 = C.create_string_buffer(256), C.create_string_buffer(64)
        self._check(F.lib.b200zk_groth16_fold(self._h, _dev_ptr(d_partials), count, _current_stream_ptr(self.device), proof, b1), "b200zk_groth16_fold")
        return proof.raw, b1.raw

    @staticmethod
    def groth16_zk(g1_terms: int, g2_terms: int, r: int, s: int) -> "F.Groth16Zk":
        """g1_terms: handle of alpha1, beta1, delta1; g2_terms: handle of beta2, delta2 (plain resident bases);
        r, s: blinding scalars, integers in [0, group order) -- the library refuses larger values, it does not reduce them"""
        if not (0 <= r < 1 << 256 and 0 <= s < 1 << 256):
            raise B200Error.serialization("groth16_zk: r and s must be 256-bit non-negative integers")
        zk = F.Groth16Zk()
        zk.g1_terms, zk.g2_terms = g1_terms, g2_terms
        zk.r[:] = list(int(r).to_bytes(32, "little"))
        zk.s[:] = list(int(s).to_bytes(32, "little"))
        return zk

    def groth16_prove(self, pk, zk, witness, a_evals, b_evals, c_evals, flags: int = 0) -> bytes:
        """-> the blinded proof A | B2 | C (256 bytes) over a key with separate alpha / beta / delta terms (`zk`, from
        groth16_zk).  Host buffers, or device tensors with G16_INPUTS_DEVICE, as groth16_commit."""
        wp, ap, bp, cp, keep = self._g16_ptrs(pk, witness, a_evals, b_evals, c_evals, flags)
        proof = C.create_string_buffer(256)
        self._check(F.lib.b200zk_groth16_prove(self._h, C.byref(pk), C.byref(zk) if zk is not None else None, wp, ap, bp, cp, flags,
                                               _current_stream_ptr(self.device), proof), "b200zk_groth16_prove")
        return proof.raw

    def groth16_fold_zk(self, zk, d_partials, count: int) -> bytes:
        """folds `count` 768-byte blocks of groth16_commit_partial, then adds the key terms and the blinding once"""
        if d_partials.numel() * d_partials.element_size() < 768 * count:
            raise B200Error.serialization("groth16_fold_zk: d_partials must hold 768 bytes per block")
        proof = C.create_string_buffer(256)
        self._check(F.lib.b200zk_groth16_fold_zk(self._h, C.byref(zk) if zk is not None else None, _dev_ptr(d_partials), count,
                                                 _current_stream_ptr(self.device), proof), "b200zk_groth16_fold_zk")
        return proof.raw

    def g1_msm_partial_device(self, d_points, d_scalars, n: int, d_partial, flags: int = 0):
        self._check(F.lib.b200zk_g1_msm_partial_device(self._h, _dev_ptr(d_points), _dev_ptr(d_scalars), n, flags, _current_stream_ptr(self.device), _dev_ptr(d_partial)), "b200zk_g1_msm_partial_device")

    def g2_msm_partial_device(self, d_points, d_scalars, n: int, d_partial, flags: int = 0):
        self._check(F.lib.b200zk_g2_msm_partial_device(self._h, _dev_ptr(d_points), _dev_ptr(d_scalars), n, flags, _current_stream_ptr(self.device), _dev_ptr(d_partial)), "b200zk_g2_msm_partial_device")

    def g1_msm_partial_resident_device(self, handle: int, d_scalars, n: int, d_partial, flags: int = 0):
        self._check(F.lib.b200zk_g1_msm_partial_resident_device(self._h, handle, _dev_ptr(d_scalars), n, flags, _current_stream_ptr(self.device), _dev_ptr(d_partial)), "b200zk_g1_msm_partial_resident_device")

    def g2_msm_partial_resident_device(self, handle: int, d_scalars, n: int, d_partial, flags: int = 0):
        self._check(F.lib.b200zk_g2_msm_partial_resident_device(self._h, handle, _dev_ptr(d_scalars), n, flags, _current_stream_ptr(self.device), _dev_ptr(d_partial)), "b200zk_g2_msm_partial_resident_device")

    def g1_msm_partial_resident(self, handle: int, scalars, n: int, d_partial, flags: int = 0):
        _need(scalars, 32 * n, "b200zk_g1_msm_partial_resident scalars")
        sp, keep = _host_ptr(scalars)
        self._check(F.lib.b200zk_g1_msm_partial_resident(self._h, handle, sp, n, flags, _current_stream_ptr(self.device), _dev_ptr(d_partial)), "b200zk_g1_msm_partial_resident")

    def g2_msm_partial_resident(self, handle: int, scalars, n: int, d_partial, flags: int = 0):
        _need(scalars, 32 * n, "b200zk_g2_msm_partial_resident scalars")
        sp, keep = _host_ptr(scalars)
        self._check(F.lib.b200zk_g2_msm_partial_resident(self._h, handle, sp, n, flags, _current_stream_ptr(self.device), _dev_ptr(d_partial)), "b200zk_g2_msm_partial_resident")

    def g1_fold_partials_device(self, d_partials, count: int, flags: int = 0) -> bytes:
        out = C.create_string_buffer(64)
        self._check(F.lib.b200zk_g1_fold_partials_device(self._h, _dev_ptr(d_partials), count, flags, _current_stream_ptr(self.device), out), "b200zk_g1_fold_partials_device")
        return out.raw

    def g2_fold_partials_device(self, d_partials, count: int, flags: int = 0) -> bytes:
        out = C.create_string_buffer(128)
        self._check(F.lib.b200zk_g2_fold_partials_device(self._h, _dev_ptr(d_partials), count, flags, _current_stream_ptr(self.device), out), "b200zk_g2_fold_partials_device")
        return out.raw

    # ------------------------------------------------------------------ device utilities
    def field_to_mont_device(self, d, n: int, which: int):
        self._check(F.lib.b200zk_field_to_mont_device(self._h, _dev_ptr(d), n, which, _current_stream_ptr(self.device)), "field_to_mont")

    def field_from_mont_device(self, d, n: int, which: int):
        self._check(F.lib.b200zk_field_from_mont_device(self._h, _dev_ptr(d), n, which, _current_stream_ptr(self.device)), "field_from_mont")

    def field_mul_device(self, d_a, d_b, d_out, n: int, which: int, repeat: int = 1):
        self._check(F.lib.b200zk_field_mul_device(self._h, _dev_ptr(d_a), _dev_ptr(d_b), _dev_ptr(d_out), n, which, repeat, _current_stream_ptr(self.device)), "field_mul")

    def fr_quotient_device(self, d_a, d_b, d_c, d_out, n: int, zinv: int):
        """d_out[i] = (a[i]*b[i] - c[i]) * zinv (Montgomery data, zinv an integer mod r)."""
        z = C.cast(C.c_char_p(int(zinv).to_bytes(32, "little")), C.c_void_p)
        self._check(F.lib.b200zk_fr_quotient_device(self._h, _dev_ptr(d_a), _dev_ptr(d_b), _dev_ptr(d_c), _dev_ptr(d_out), n, z, _current_stream_ptr(self.device)), "fr_quotient")

    def fr_random_device(self, d_out, n: int, seed: int, start: int = 0, flags: int = 0):
        self._check(F.lib.b200zk_fr_random_device(self._h, _dev_ptr(d_out), n, seed, start, flags, _current_stream_ptr(self.device)), "fr_random")

    def g1_chain_device(self, d_out, start: int, n: int, k: int, d: int):
        self._check(F.lib.b200zk_g1_chain_device(self._h, _dev_ptr(d_out), start, n, C.cast(C.c_char_p(k.to_bytes(32, "little")), C.c_void_p),
                                                 C.cast(C.c_char_p(d.to_bytes(32, "little")), C.c_void_p), _current_stream_ptr(self.device)), "g1_chain")

    def g2_chain_device(self, d_out, start: int, n: int, k: int, d: int):
        self._check(F.lib.b200zk_g2_chain_device(self._h, _dev_ptr(d_out), start, n, C.cast(C.c_char_p(k.to_bytes(32, "little")), C.c_void_p),
                                                 C.cast(C.c_char_p(d.to_bytes(32, "little")), C.c_void_p), _current_stream_ptr(self.device)), "g2_chain")

    def g1_check_device(self, d_points, n: int) -> int:
        bad = C.c_size_t()
        rc = F.lib.b200zk_g1_check_device(self._h, _dev_ptr(d_points), n, _current_stream_ptr(self.device), C.byref(bad))
        if rc == F.ERR_NOT_ON_CURVE:
            return bad.value
        self._check(rc, "g1_check")
        return n

    def g2_check_device(self, d_points, n: int) -> int:
        bad = C.c_size_t()
        rc = F.lib.b200zk_g2_check_device(self._h, _dev_ptr(d_points), n, _current_stream_ptr(self.device), C.byref(bad))
        if rc == F.ERR_NOT_ON_CURVE:
            return bad.value
        self._check(rc, "g2_check")
        return n
