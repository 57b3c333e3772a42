"""Groth16 from circom artifacts: a snarkjs `.zkey` loaded once into HBM, each `.wtns` witness proved in one call.

The two files risc0-groth16's shrink-wrap hands its prover (the proving key, the witness circom-witnesscalc computed),
taken byte for byte; formats and the proof they give are stated in include/b200zk.h (b200zk_groth16_zkey_*).  The
sparse evaluation of the constraint rows, the NTTs onto the odd coset, the MSMs and the blinding all run in
libb200zk.so; Python passes bytes.
"""
from __future__ import annotations

import ctypes as C
import os

from . import _ffi as F
from .context import _current_stream_ptr, _host_ptr
from .groth16 import Groth16Verifier, random_scalar


def _bytes(src) -> bytes:
    """file contents from bytes-like data or a path"""
    if isinstance(src, (str, os.PathLike)):
        with open(src, "rb") as f:
            return f.read()
    return bytes(src)


class ZkeyProver:
    """`ZkeyProver(ctx, zkey, precompute=True)`: zkey is the .zkey file's bytes or its path.  `precompute` builds the
    window tables of the five columns (faster MSMs, about 13x the columns' memory)."""

    def __init__(self, ctx, zkey, precompute: bool = True):
        data = _bytes(zkey)
        ptr, keep = _host_ptr(data)
        h = C.c_uint64()
        ctx._check(F.lib.b200zk_groth16_zkey_load(ctx._h, ptr, len(data), 1 if precompute else 0, C.byref(h)), "b200zk_groth16_zkey_load")
        del keep
        self.ctx, self.key = ctx, h.value
        try:
            nv, npub, log_n = C.c_uint32(), C.c_uint32(), C.c_uint32()
            ctx._check(F.lib.b200zk_groth16_zkey_info(ctx._h, self.key, C.byref(nv), C.byref(npub), C.byref(log_n), None, 0), "b200zk_groth16_zkey_info")
            self.n_vars, self.n_public, self.log_n = nv.value, npub.value, log_n.value
            vk = C.create_string_buffer(448 + 64 * (self.n_public + 1))
            ctx._check(F.lib.b200zk_groth16_zkey_info(ctx._h, self.key, None, None, None, vk, len(vk.raw)), "b200zk_groth16_zkey_info")
            self.vk = vk.raw  # alpha1 | beta2 | gamma2 | delta2 | IC, EIP-196/197 bytes
        except BaseException:
            self.close()  # a prover that failed to construct leaves no key behind
            raise

    def verifier(self) -> Groth16Verifier:
        """the Groth16 verifier of this key (public inputs: signals 1..nPublic of the witness)"""
        v = self.vk
        ic = [v[448 + 64 * i: 512 + 64 * i] for i in range(self.n_public + 1)]
        return Groth16Verifier(self.ctx, v[:64], v[64:192], v[192:320], v[320:448], ic)

    def prove(self, wtns, r: int | None = None, s: int | None = None) -> bytes:
        """-> proof A (64) | B (128) | C (64) of the .wtns witness (bytes or a path), blinded with r and s (each in
        [0, group order); None = a fresh draw of `random_scalar`).  ONE call of the C ABI (b200zk_groth16_zkey_prove)."""
        if self.key is None:
            raise ValueError("ZkeyProver is closed")
        data = _bytes(wtns)
        r = random_scalar() if r is None else r
        s = random_scalar() if s is None else s
        if not (0 <= r < 1 << 256 and 0 <= s < 1 << 256):
            raise ValueError("r and s must be 256-bit non-negative integers")
        ptr, keep = _host_ptr(data)
        rb = C.create_string_buffer(int(r).to_bytes(32, "little"), 32)
        sb = C.create_string_buffer(int(s).to_bytes(32, "little"), 32)
        proof = C.create_string_buffer(256)
        self.ctx._check(F.lib.b200zk_groth16_zkey_prove(self.ctx._h, self.key, ptr, len(data), rb, sb, _current_stream_ptr(self.ctx.device), proof),
                        "b200zk_groth16_zkey_prove")
        del keep
        return proof.raw

    def close(self):
        if self.key is not None:
            self.ctx._check(F.lib.b200zk_groth16_zkey_free(self.ctx._h, self.key), "b200zk_groth16_zkey_free")
            self.key = None
