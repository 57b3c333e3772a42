"""Groth16-shaped commitment pipeline on the library's CUDA kernels (SURVEY.md section 8f row 1, BASELINE config #5).

This is the arithmetic the SNARK wrap behind `ProofFormat::Groth16` performs
(/root/reference/crates/prover/src/backend/sp1.rs:97-134 -> gnark; risc0.rs:24-29,71-82 -> risc0-groth16):

    quotient   3 iNTT (A,B,C evaluations -> coefficients), 3 coset NTT, pointwise (a*b - c)/Z_H, 1 coset iNTT
    commit     [A]1 = MSM(pk.A_g1, w)   [B]1 = MSM(pk.B_g1, w)   [B]2 = MSM(pk.B_g2, w)
               [L]1 = MSM(pk.L_g1, w_private)   [H]1 = MSM(pk.H_g1, h)
    assemble   proof = A | B | C with C = [L]1 + [H]1      (EIP-197 byte order, 256 bytes)
    blinded    A += alpha1 + r delta1, B += beta2 + s delta2, C += s A + r B1 - rs delta1   (b200zk_groth16_prove)

The reference's real wrap circuit and proving key live inside the zkVM SDKs and are not in the tree, so the
circuit here is SYNTHETIC (SURVEY.md section 8d, config 5): witness and constraint evaluations are derived
deterministically from the serialized program input, with C = A o B on the domain so that the quotient is an
exact polynomial, and the proving key is a set of chain bases.  The STARK stage is excluded.  `prove` applies no
blinding; `prove_zk_device` (a circuit built with zk=True) adds synthetic alpha / beta / delta key terms and the r, s
blinding on the device.  What is measured and parity-checked is exactly the MSM + NTT work of a Groth16 prove.
`Groth16Prover` proves a caller-supplied key whose alpha / beta ride on variable 0 (no blinding); `Groth16ZkProver`
proves a key in the ark-groth16 / gnark layout, blinded, as those provers do.
All arithmetic runs in libb200zk.so; Python only sequences the calls.
"""
from __future__ import annotations

import hashlib
import secrets
from dataclasses import dataclass, field

from . import _ffi as F

R_MOD = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001
COSET_GEN = 5  # ark/gnark multiplicative generator of Fr


def _seed64(data: bytes, tag: bytes) -> int:
    return int.from_bytes(hashlib.sha256(tag + data).digest()[:8], "little")


def _chain_kd(tag: bytes) -> tuple[int, int]:
    h = hashlib.sha256(b"b200zk-pk-" + tag).digest()
    return (int.from_bytes(h[:16], "little") | 1), (int.from_bytes(h[16:], "little") | 1)


def random_scalar(randbits=secrets.randbits) -> int:
    """A uniform blinding scalar in [0, r): 254 random bits, drawn again while the value is >= r.  Rejection instead of
    a reduction mod r, which would make the values below 2^254 - r twice as likely; r > 2^253, so fewer than two draws
    are needed on average.  `randbits(k)` -> k random bits (a CSPRNG by default)."""
    while True:
        x = randbits(254)
        if x < R_MOD:
            return x


def quotient_on_device(ctx, log_n: int, a, b, c, zinv: int):
    """H coefficients (Montgomery) from the A, B, C evaluations on the domain (Montgomery device tensors);
    `a` is overwritten with H.  3 iNTT, 3 coset NTT, (a*b - c)/Z_H on the coset, 1 coset iNTT."""
    for poly in (a, b, c):
        ctx.fr_ntt_device(poly, log_n, F.NTT_INVERSE)   # evaluations -> coefficients
        ctx.fr_ntt_device(poly, log_n, F.NTT_COSET)     # coefficients -> evaluations on the coset
    ctx.fr_quotient_device(a, b, c, a, 1 << log_n, zinv)
    ctx.fr_ntt_device(a, log_n, F.NTT_INVERSE | F.NTT_COSET)
    return a


def coset_vanishing_inverse(log_n: int) -> int:
    """1 / Z_H on the coset g*<w>: Z_H = x^n - 1 is the constant g^n - 1 there."""
    return pow((pow(COSET_GEN, 1 << log_n, R_MOD) - 1) % R_MOD, -1, R_MOD)


class Groth16Prover:
    """The same pipeline over a CALLER-SUPPLIED proving key (what a zkVM SDK would hand to `B200Backend`): query
    columns as EIP-196/197 byte strings, one point per R1CS variable (`a_g1`, `b_g1`, `b_g2`), per private variable
    (`l_g1`) and per quotient coefficient (`h_g1`, n-1 points).  No blinding (r = s = 0): the proof verifies, it is
    not zero-knowledge (Groth16ZkProver is).  tests/test_gpu_parity.py proves a small real R1CS with it and checks the Groth16
    verification equation with the GPU pairing check."""

    def __init__(self, ctx, log_n: int, a_g1: bytes, b_g1: bytes, b_g2: bytes, l_g1: bytes, h_g1: bytes, n_public: int):
        self.ctx, self.log_n, self.n, self.n_public = ctx, log_n, 1 << log_n, n_public
        self.m = len(a_g1) // 64
        if len(b_g1) != 64 * self.m or len(b_g2) != 128 * self.m or len(l_g1) != 64 * (self.m - n_public) or len(h_g1) != 64 * (self.n - 1):
            raise ValueError("proving-key column sizes do not match")
        up1, up2 = ctx.g1_bases_upload, ctx.g2_bases_upload
        self.h = {"a_g1": up1(a_g1, self.m, F.POINTS_BE), "b_g1": up1(b_g1, self.m, F.POINTS_BE), "b_g2": up2(b_g2, self.m, F.POINTS_BE),
                  "l_g1": up1(l_g1, self.m - n_public, F.POINTS_BE), "h_g1": up1(h_g1, self.n - 1, F.POINTS_BE)}
        self.zinv = coset_vanishing_inverse(log_n)
        # struct b200zk_groth16_pk: whole columns on one GPU; L starts behind the public variables, H has n-1 points
        self.pk = ctx.groth16_pk(log_n, [self.h[q] for q in ("a_g1", "b_g1", "b_g2", "l_g1", "h_g1")],
                                 [self.m, self.m, self.m, self.m - n_public, self.n - 1], [0, 0, 0, n_public, 0])
        self.b_g1 = None  # [B]1 of the last proof (what blinding would consume)

    def close(self):
        for h in self.h.values():
            self.ctx.bases_free(h)
        self.h.clear()

    def _host_inputs(self, z, a_evals, b_evals, c_evals):
        """(witness, a, b, c) host buffers of the C ABI: canonical LE witness, Montgomery LE evaluations"""
        if len(z) != self.m or any(len(e) != self.n for e in (a_evals, b_evals, c_evals)):
            raise ValueError("assignment / evaluation vector sizes do not match the proving key")
        r_mont = (1 << 256) % R_MOD

        def mont(vals):  # host-side Montgomery form (the SDK's field code holds its vectors this way)
            return b"".join(int(v % R_MOD * r_mont % R_MOD).to_bytes(32, "little") for v in vals)

        zb = b"".join(int(v % R_MOD).to_bytes(32, "little") for v in z)
        return zb, bytearray(mont(a_evals)), bytearray(mont(b_evals)), bytearray(mont(c_evals))

    def prove(self, z, a_evals, b_evals, c_evals) -> bytes:
        """z: the full assignment (integers mod r, z[0] = 1, then the public inputs, then the private variables);
        a/b/c_evals: (A z), (B z), (C z) on the domain.  Returns A (64) | B (128) | C (64).
        ONE call of the C ABI (b200zk_groth16_commit) with host buffers -- what rust/ethrex-backend/src/b200.rs does."""
        proof, self.b_g1 = self.ctx.groth16_commit(self.pk, *self._host_inputs(z, a_evals, b_evals, c_evals))
        return proof


class Groth16ZkProver(Groth16Prover):
    """The zero-knowledge prove over a key in the ark-groth16 / gnark layout: the query columns WITHOUT alpha and beta
    folded into variable 0, and beside them the key terms alpha1, beta1, delta1 (G1, 64 bytes each) and beta2, delta2
    (G2, 128 bytes each), all EIP-196/197 bytes.  `prove` returns the proof ark-groth16 0.5 (create_proof_with_reduction)
    and gnark (groth16.Prove) return for the same blinding scalars r, s:
        A = alpha1 + sum z_i A_i + r delta1      B = beta2 + sum z_i B2_i + s delta2
        C = [L] + [H] + s A + r (beta1 + sum z_i B1_i + s delta1) - r s delta1
    r and s default to fresh draws of `random_scalar`; pass them to get a reproducible proof."""

    def __init__(self, ctx, log_n: int, a_g1: bytes, b_g1: bytes, b_g2: bytes, l_g1: bytes, h_g1: bytes, n_public: int,
                 alpha_g1: bytes, beta_g1: bytes, beta_g2: bytes, delta_g1: bytes, delta_g2: bytes):
        if any(len(x) != 64 for x in (alpha_g1, beta_g1, delta_g1)) or any(len(x) != 128 for x in (beta_g2, delta_g2)):
            raise ValueError("key terms: alpha1, beta1, delta1 are 64-byte G1 points, beta2 and delta2 128-byte G2 points")
        super().__init__(ctx, log_n, a_g1, b_g1, b_g2, l_g1, h_g1, n_public)
        self.h["terms_g1"] = ctx.g1_bases_upload(alpha_g1 + beta_g1 + delta_g1, 3, F.POINTS_BE)
        self.h["terms_g2"] = ctx.g2_bases_upload(beta_g2 + delta_g2, 2, F.POINTS_BE)

    def prove(self, z, a_evals, b_evals, c_evals, r: int | None = None, s: int | None = None) -> bytes:
        """As Groth16Prover.prove, blinded with r and s (each in [0, group order); None = a fresh random draw).
        ONE call of the C ABI (b200zk_groth16_prove)."""
        r = random_scalar() if r is None else r
        s = random_scalar() if s is None else s
        zk = self.ctx.groth16_zk(self.h["terms_g1"], self.h["terms_g2"], r, s)
        return self.ctx.groth16_prove(self.pk, zk, *self._host_inputs(z, a_evals, b_evals, c_evals))


class Groth16Verifier:
    """Groth16 verification on the device, many proofs per launch: what `ProverBackend::verify` does off-chain
    (/root/reference/crates/prover/src/backend/mod.rs:116-117) and what the on-chain verifier contracts compute
    (/root/reference/crates/l2/contracts/src/l1/OnChainProposer.sol:365-388) --
        e(-A, B) * e(alpha, beta) * e(IC_0 + sum x_i IC_i, gamma) * e(C, delta) == 1
    through b200zk_bn254_pairing_check_batch; the public-input combination is a small G1 MSM through the host entry
    point.  All points are EIP-196/197 byte strings."""
    P_MOD = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47

    def __init__(self, ctx, alpha_g1: bytes, beta_g2: bytes, gamma_g2: bytes, delta_g2: bytes, ic):
        if len(alpha_g1) != 64 or any(len(x) != 128 for x in (beta_g2, gamma_g2, delta_g2)) or not ic or any(len(x) != 64 for x in ic):
            raise ValueError("verifying-key element sizes do not match")
        self.ctx, self.alpha_g1, self.beta_g2, self.gamma_g2, self.delta_g2, self.ic = ctx, alpha_g1, beta_g2, gamma_g2, delta_g2, list(ic)

    def _neg(self, g1: bytes):
        """-A for a CANONICAL encoding; None when a coordinate is >= p.  The levm ecpairing wrapper and the on-chain
        verifier reject such an A (CoordinateExceedsFieldModulus, crates/vm/levm/src/precompiles.rs:801-820); reducing y
        here first would turn (x, y + p) into a point that verifies -- proof malleability."""
        x, y = int.from_bytes(g1[:32], "big"), int.from_bytes(g1[32:], "big")
        if x >= self.P_MOD or y >= self.P_MOD:
            return None
        return g1 if (x == 0 and y == 0) else g1[:32] + (self.P_MOD - y).to_bytes(32, "big")

    def calldata(self, proof: bytes, public_inputs):
        """ecpairing calldata of the verification equation, or None when the proof / inputs are not canonically encoded
        (a public input outside [0, r) is rejected, not reduced: x and x + r must not verify alike)."""
        if len(proof) != 256 or len(public_inputs) != len(self.ic) - 1:
            raise ValueError("proof must be 256 bytes and carry one public input per IC point after the first")
        if any((not isinstance(x, int)) or x < 0 or x >= R_MOD for x in public_inputs):
            return None
        a, b, c = proof[:64], proof[64:192], proof[192:]
        neg_a = self._neg(a)
        if neg_a is None:
            return None
        scalars = (1).to_bytes(32, "big") + b"".join(int(x).to_bytes(32, "big") for x in public_inputs)
        vk_x = self.ctx.g1_msm(b"".join(self.ic), scalars, len(self.ic), F.POINTS_BE | F.SCALARS_BE)
        return neg_a + b + self.alpha_g1 + self.beta_g2 + vk_x + self.gamma_g2 + c + self.delta_g2

    def verify_batch(self, proofs, public_inputs):
        """-> list of booleans; a proof with a malformed point (status != 0) or a non-canonical encoding is False."""
        cds = [self.calldata(p, x) for p, x in zip(proofs, public_inputs)]
        live = [cd for cd in cds if cd is not None]
        res, st = self.ctx.bn254_pairing_check_batch(live) if live else ([], [])
        it = iter(zip(res, st))
        out = []
        for cd in cds:
            if cd is None:
                out.append(False)
            else:
                r, s = next(it)
                out.append(bool(r) and s == 0)
        return out

    def verify(self, proof: bytes, public_inputs) -> bool:
        return self.verify_batch([proof], [public_inputs])[0]


@dataclass
class ProvingKey:
    """Resident (precomputed) proving-key columns: handles into the context + the chain scalars that define them."""
    log_n: int
    handles: dict = field(default_factory=dict)   # name -> b200zk bases handle
    chains: dict = field(default_factory=dict)    # name -> (k, d, is_g2)


class SyntheticWrapCircuit:
    """Domain size 2^log_n; `n` witness entries; H has n-1 coefficients."""
    QUERIES = (("a_g1", False), ("b_g1", False), ("b_g2", True), ("l_g1", False), ("h_g1", False))
    # device bytes per domain point a context may hold beside the proving key: the witness and the three evaluation
    # vectors (128 B), the NTT scratch (32 B), the one-shot digit sort of a plain-bases MSM (16 B per entry x 15 windows
    # = 240 B), the two sort slots of a host-scalar MSM (2 x 16 B x 12 entries = 384 B), G2 bucket runs (~200 B) and
    # the workspaces' 1/8 growth slack
    PROVE_WORKSPACE_PER_POINT = 1152

    # synthetic ark-layout key terms (zk=True): alpha1, beta1, delta1 and beta2, delta2 as short chains
    ZK_TERMS = (("terms_g1", False, 3), ("terms_g2", True, 2))

    def __init__(self, ctx, log_n: int, precompute: bool = True, g2: bool = True, rank: int = 0, world: int = 1, zk: bool = False):
        """rank/world: every rank keeps only its contiguous shard [lo, hi) of each proving-key column (point-split
        MSMs, ethrex_b200.dist.msm_sharded); the NTTs of the quotient are cheap and computed on every rank.
        zk: also hold the alpha / beta / delta key terms (whole, on every rank) that prove_zk_device blinds with."""
        import torch
        from .dist import shard_range
        self.ctx, self.log_n, self.n = ctx, log_n, 1 << log_n
        self.rank, self.world = rank, world
        self.lo, self.hi = shard_range(self.n, rank, world)
        self.pk = ProvingKey(log_n)
        m = self.hi - self.lo
        # A window table holds ceil(255/c) multiples of every base (13x the bases at 2^24), and at domain 2^24 the five
        # tables alone take 78 GiB: more than an 80 GB GPU holds beside the prove's workspaces.  Columns get their tables
        # in QUERIES order while the key fits in the device's TOTAL memory less PROVE_WORKSPACE_PER_POINT * n bytes (a
        # rule that depends on the device model only, not on what else runs on it); the others keep plain bases (same
        # proof, slower MSMs).  H comes last in QUERIES and has scalars of its own, so it is the first to go and no
        # shared digit sort is lost.  The table's size per plain byte is read off the first table built (an integer).
        self.plain_columns = []
        widths = [16 if is_g2 else 8 for _, is_g2 in self.QUERIES if g2 or not is_g2]
        key_bytes = sum(8 * w for w in widths) * max(m, 1)  # every column as plain bases
        budget = torch.cuda.mem_get_info()[1] - self.PROVE_WORKSPACE_PER_POINT * self.n
        expand = None
        for name, is_g2 in self.QUERIES:
            if is_g2 and not g2:
                continue
            k, d = _chain_kd(name.encode())
            pts = torch.empty((16 if is_g2 else 8) * m, dtype=torch.int64, device="cuda")
            (ctx.g2_chain_device if is_g2 else ctx.g1_chain_device)(pts, self.lo, m, k, d)
            h = (ctx.g2_bases_from_device if is_g2 else ctx.g1_bases_from_device)(pts, m)
            del pts
            if precompute:
                plain = (128 if is_g2 else 64) * max(m, 1)
                if expand is None:
                    torch.cuda.empty_cache()
                    free = torch.cuda.mem_get_info()[0]
                    ctx.bases_precompute(h, 0)
                    expand = round((free - torch.cuda.mem_get_info()[0]) / plain) + 1
                    key_bytes += (expand - 1) * plain
                elif key_bytes + (expand - 1) * plain <= budget:
                    ctx.bases_precompute(h, 0)
                    key_bytes += (expand - 1) * plain
                else:
                    self.plain_columns.append(name)
            self.pk.handles[name] = h
            self.pk.chains[name] = (k, d, is_g2)
        if zk:
            for name, is_g2, cnt in self.ZK_TERMS:
                k, d = _chain_kd(name.encode())
                pts = torch.empty((16 if is_g2 else 8) * cnt, dtype=torch.int64, device="cuda")
                (ctx.g2_chain_device if is_g2 else ctx.g1_chain_device)(pts, 0, cnt, k, d)
                self.pk.handles[name] = (ctx.g2_bases_from_device if is_g2 else ctx.g1_bases_from_device)(pts, cnt)
                self.pk.chains[name] = (k, d, is_g2)
        self.zinv = coset_vanishing_inverse(log_n)

    def close(self):
        for h in self.pk.handles.values():
            self.ctx.bases_free(h)
        self.pk.handles.clear()

    # ---- witness / constraint evaluations from the serialized input (deterministic) ----
    def assign(self, serialized_input: bytes):
        """Returns device tensors (witness canonical, a/b/c evaluations Montgomery)."""
        import torch
        n, ctx = self.n, self.ctx
        w = torch.empty(4 * n, dtype=torch.int64, device="cuda")
        a = torch.empty(4 * n, dtype=torch.int64, device="cuda")
        b = torch.empty(4 * n, dtype=torch.int64, device="cuda")
        c = torch.empty(4 * n, dtype=torch.int64, device="cuda")
        ctx.fr_random_device(w, n, _seed64(serialized_input, b"witness"), 0)
        ctx.fr_random_device(a, n, _seed64(serialized_input, b"A"), 0, F.SCALARS_MONT)
        ctx.fr_random_device(b, n, _seed64(serialized_input, b"B"), 0, F.SCALARS_MONT)
        ctx.field_mul_device(a, b, c, n, 1)  # C = A o B on the domain: the R1CS is satisfied
        return w, a, b, c

    # ---- the hot path ----
    def quotient(self, a, b, c):
        """H coefficients (Montgomery) from the A,B,C evaluations; a is overwritten with H."""
        return quotient_on_device(self.ctx, self.log_n, a, b, c, self.zinv)

    def pk_struct(self):
        """struct b200zk_groth16_pk of THIS rank's shard: every column holds points [lo, hi) of its whole column, so the
        first scalar a column multiplies is entry `lo` of the witness (A, B1, B2, L) or of the quotient (H).  The
        synthetic circuit has no public inputs: L spans the whole witness like A."""
        lo, m = self.lo, self.hi - self.lo
        mh = max(0, min(self.hi, self.n - 1) - lo)  # H has n-1 points: the last rank's shard is one short
        hd = self.pk.handles
        return self.ctx.groth16_pk(self.log_n, [hd["a_g1"], hd["b_g1"], hd.get("b_g2", 0), hd["l_g1"], hd["h_g1"]], [m, m, m, m, mh], [lo] * 5)

    def prove_device(self, serialized_input: bytes, group=None):
        """-> (proof bytes A | B2 | C, [B]1 bytes).  One GPU: ONE C-ABI call (b200zk_groth16_commit) on device inputs.
        Several GPUs: the quotient's NTTs are dealt across ranks (dist.quotient_dealt), every rank commits its shard of
        the proving key (b200zk_groth16_commit_partial), ONE all_gather moves the 768-byte blocks and every rank folds."""
        ctx = self.ctx
        w, a, b, c = self.assign(serialized_input)
        pk = self.pk_struct()
        if "b_g2" not in self.pk.handles:
            raise ValueError("the one-call path needs the G2 column")
        if self.world == 1:
            return ctx.groth16_commit(pk, w, a, b, c, F.G16_INPUTS_DEVICE)
        return ctx.groth16_fold(self._gathered_blocks(pk, w, a, b, c, group), self.world)

    def _gathered_blocks(self, pk, w, a, b, c, group):
        """several GPUs: the dealt quotient, this rank's commit_partial and ONE all_gather of the 768-byte blocks"""
        import torch
        import torch.distributed as dist
        from .dist import quotient_dealt
        h = quotient_dealt(self.ctx, self.log_n, a, b, c, self.zinv, self.rank, self.world, group)
        block = torch.zeros(96, dtype=torch.int64, device=w.device)  # 768 bytes: A | B1 | B2 | L | H partial sums
        self.ctx.groth16_commit_partial(pk, w, h, None, None, block, F.G16_INPUTS_DEVICE | F.G16_H_COEFFS)
        gathered = torch.empty(96 * self.world, dtype=torch.int64, device=w.device)
        dist.all_gather_into_tensor(gathered, block, group=group)
        return gathered

    def prove_zk_device(self, serialized_input: bytes, r: int | None = None, s: int | None = None, group=None) -> bytes:
        """-> the blinded proof A | B2 | C over the synthetic key with its alpha / beta / delta terms (built with zk=True).
        r, s: blinding scalars in [0, group order); None = a fresh random draw.  One GPU: ONE C-ABI call
        (b200zk_groth16_prove).  Several GPUs: rank 0's r and s are broadcast, every rank commits its shard, the blocks
        are all-gathered once and every rank folds them with the same r and s (b200zk_groth16_fold_zk)."""
        import torch
        ctx, hd = self.ctx, self.pk.handles
        if "terms_g1" not in hd:
            raise ValueError("prove_zk_device needs the key terms: build the circuit with zk=True")
        if "b_g2" not in hd:
            raise ValueError("the one-call path needs the G2 column")
        r = random_scalar() if r is None else r
        s = random_scalar() if s is None else s
        w, a, b, c = self.assign(serialized_input)
        pk = self.pk_struct()
        if self.world > 1:
            import torch.distributed as dist
            rs = torch.tensor(list(int(r).to_bytes(32, "little") + int(s).to_bytes(32, "little")), dtype=torch.uint8, device=w.device)
            dist.broadcast(rs, src=0 if group is None else dist.get_global_rank(group, 0), group=group)
            rsb = bytes(rs.cpu().tolist())
            r, s = int.from_bytes(rsb[:32], "little"), int.from_bytes(rsb[32:], "little")
        zk = ctx.groth16_zk(hd["terms_g1"], hd["terms_g2"], r, s)
        if self.world == 1:
            return ctx.groth16_prove(pk, zk, w, a, b, c, F.G16_INPUTS_DEVICE)
        return ctx.groth16_fold_zk(zk, self._gathered_blocks(pk, w, a, b, c, group), self.world)

    def commit(self, w, h_coeffs, msm=None):
        """The five MSMs as separate calls (the pre-ABI-v2 path, kept as a cross-check of the one-call path and for the
        `msm` hook).  `msm(name, scalars, n, flags)` lets a driver substitute its own MSM."""
        ctx, n = self.ctx, self.n

        def local(name, scalars, count, flags):
            hnd = self.pk.handles[name]
            is_g2 = self.pk.chains[name][2]
            if self.world > 1:  # this rank's slice of the scalars against its shard of the column, then all-gather + fold
                from .dist import msm_sharded
                hi = min(self.hi, count)
                m = max(0, hi - self.lo)
                return msm_sharded(ctx, None, scalars[4 * self.lo: 4 * (self.lo + max(m, 1))], m, flags, g2=is_g2, handle=hnd)
            if is_g2:
                return ctx.g2_msm_resident_device(hnd, scalars, count, flags)
            return ctx.g1_msm_resident_device(hnd, scalars, count, flags)

        run = msm or local
        names = [q for q in ("a_g1", "b_g1", "b_g2", "l_g1") if q in self.pk.handles]
        if msm is None and self.world == 1:
            # the witness MSMs over window tables share one scalar sort (b200zk_msm_multi_resident_device)
            shared = [q for q in names if q not in self.plain_columns]
            res = ctx.msm_multi_resident_device([self.pk.handles[q] for q in shared], [self.pk.chains[q][2] for q in shared], w, n, 0)
            out = dict(zip(shared, res))
            out.update({q: run(q, w, n, 0) for q in names if q in self.plain_columns})
        else:
            out = {q: run(q, w, n, 0) for q in names}
        out["h_g1"] = run("h_g1", h_coeffs, n - 1, F.SCALARS_MONT)
        return out

    def assemble(self, commitments) -> bytes:
        """proof = A (64) | B (128, x_im|x_re|y_im|y_re) | C (64), C = L + H folded on the device."""
        one = (1).to_bytes(32, "little")
        # C = 1*L + 1*H: a 2-point MSM through the host entry point (validates the two encodings on the way in)
        c_pt = self.ctx.g1_msm(commitments["l_g1"] + commitments["h_g1"], one + one, 2, F.POINTS_BE)
        b2 = commitments.get("b_g2", bytes(128))
        return commitments["a_g1"] + b2 + c_pt

    def prove_separate(self, serialized_input: bytes, msm=None):
        """the pre-ABI-v2 sequence: quotient, five separately read-back MSMs, host-side assembly -> (proof, commitments)"""
        w, a, b, c = self.assign(serialized_input)
        h = self.quotient(a, b, c)
        cm = self.commit(w, h, msm)
        return self.assemble(cm), cm

    def prove(self, serialized_input: bytes, msm=None) -> bytes:
        if msm is not None or "b_g2" not in self.pk.handles:
            return self.prove_separate(serialized_input, msm)[0]
        return self.prove_device(serialized_input)[0]
