//! Safe wrapper over the raw C ABI (`b200zk-sys`).  One process-global context, like the reference's
//! `static PROVER_SETUP: OnceLock<ProverSetup>` (`crates/prover/src/backend/sp1.rs:30,93-95`).
//! Obeys the prover crate's lint policy (`crates/prover/Cargo.toml:72-80`): no unwrap / expect / panic /
//! indexing / `as`.
use std::ffi::CStr;
use std::ptr::NonNull;
use std::sync::{Mutex, OnceLock};

use b200zk_sys as sys;
use ethrex_prover::backend::BackendError;

/// Owned `b200zk_ctx*`.  The library serialises work on its own stream; the `Mutex` in [`global`] makes the
/// handle usable from the prover actor's blocking thread (`crates/prover/src/prover.rs:240-251`) or any other.
pub struct B200zk {
    ctx: NonNull<sys::b200zk_ctx>,
}

// SAFETY: the context owns only device resources and is never aliased outside the Mutex in `global()`.
unsafe impl Send for B200zk {}

static GLOBAL: OnceLock<Result<Mutex<B200zk>, String>> = OnceLock::new();

/// EIP-7823's bound on each MODEXP operand (`B200ZK_MODEXP_MAX_BYTES`); longer operands are not taken by the device.
pub const MODEXP_MAX_BYTES: usize = 1024;

/// Lazily initialised process-global context on the device selected by `CUDA_VISIBLE_DEVICES`.
pub fn global() -> Result<&'static Mutex<B200zk>, BackendError> {
    GLOBAL
        .get_or_init(|| B200zk::new(0).map(Mutex::new).map_err(|e| e.to_string()))
        .as_ref()
        .map_err(BackendError::proving)
}

/// The host buffers of a Groth16 call must hold what the library copies out of them: 2^log_n evaluations each, and a
/// witness that reaches the end of every column multiplying it (columns 0..3).
fn check_groth16_inputs(what: &str, pk: &sys::b200zk_groth16_pk, witness: &[u8], a: &[u8], b: &[u8], c: &[u8]) -> Result<(), BackendError> {
    let n_bytes = 32usize.checked_shl(pk.log_n).ok_or_else(|| BackendError::serialization(format!("{what}: log_n too large")))?;
    if a.len() != n_bytes || b.len() != n_bytes || c.len() != n_bytes {
        return Err(BackendError::serialization(format!("{what}: evaluation vectors must hold 2^log_n elements")));
    }
    let mut wit_end = 0u64;
    for ((h, cnt), off) in pk.handle.iter().zip(pk.count.iter()).zip(pk.offset.iter()).take(4) {
        if *h != 0 {
            wit_end = wit_end.max(off.checked_add(*cnt).ok_or_else(|| BackendError::serialization(format!("{what}: column range overflows")))?);
        }
    }
    let have = u64::try_from(witness.len() / 32).map_err(BackendError::serialization)?;
    if have < wit_end {
        return Err(BackendError::serialization(format!("{what}: witness holds {have} scalars, the proving key multiplies {wit_end}")));
    }
    Ok(())
}

fn status_message(ctx: Option<&B200zk>, status: i32) -> String {
    // SAFETY: both functions return NUL-terminated strings owned by the library / the context.
    let base = unsafe { CStr::from_ptr(sys::b200zk_strerror(status)) }.to_string_lossy().into_owned();
    match ctx {
        Some(c) => {
            let detail = unsafe { CStr::from_ptr(sys::b200zk_last_error(c.ctx.as_ptr())) }.to_string_lossy().into_owned();
            format!("b200zk status {status}: {base} ({detail})")
        }
        None => format!("b200zk status {status}: {base}"),
    }
}

/// C status -> `BackendError` (the table INTEGRATION.md documents): malformed input is a serialization
/// error, everything the device reports is a proving error.
fn check(ctx: &B200zk, status: i32) -> Result<bool, BackendError> {
    match status {
        sys::B200ZK_OK => Ok(false),
        sys::B200ZK_OK_INFINITY => Ok(true),
        sys::B200ZK_ERR_NOT_IN_FIELD | sys::B200ZK_ERR_NOT_ON_CURVE | sys::B200ZK_ERR_INVALID_ARG => {
            Err(BackendError::serialization(status_message(Some(ctx), status)))
        }
        sys::B200ZK_ERR_UNSUPPORTED => Err(BackendError::not_implemented(status_message(Some(ctx), status))),
        other => Err(BackendError::proving(status_message(Some(ctx), other))),
    }
}

impl B200zk {
    pub fn new(device: i32) -> Result<Self, BackendError> {
        let mut raw: *mut sys::b200zk_ctx = std::ptr::null_mut();
        // SAFETY: `raw` is a valid out-pointer.
        let status = unsafe { sys::b200zk_init(device, &mut raw) };
        match NonNull::new(raw) {
            Some(ctx) if status == sys::B200ZK_OK => Ok(Self { ctx }),
            _ => Err(BackendError::proving(status_message(None, status))),
        }
    }

    /// sum_i scalars[i] * bases[i] over BN254 G1.  `points`: n x 64 bytes, `scalars`: n x 32 bytes, formats per
    /// `flags` (see include/b200zk.h).  Returns the 64-byte EIP-196 encoding.
    pub fn g1_msm(&mut self, points: &[u8], scalars: &[u8], flags: u32) -> Result<[u8; 64], BackendError> {
        let n = scalars.len() / 32;
        if points.len() / 64 < n {
            return Err(BackendError::serialization("g1_msm: fewer points than scalars"));
        }
        let mut out = [0u8; 64];
        // SAFETY: lengths checked above; buffers outlive the (synchronous) call.
        let status = unsafe {
            sys::b200zk_g1_msm(self.ctx.as_ptr(), points.as_ptr().cast(), scalars.as_ptr().cast(), n, flags, out.as_mut_ptr())
        };
        check(self, status)?;
        Ok(out)
    }

    pub fn g2_msm(&mut self, points: &[u8], scalars: &[u8], flags: u32) -> Result<[u8; 128], BackendError> {
        let n = scalars.len() / 32;
        if points.len() / 128 < n {
            return Err(BackendError::serialization("g2_msm: fewer points than scalars"));
        }
        let mut out = [0u8; 128];
        // SAFETY: as above.
        let status = unsafe {
            sys::b200zk_g2_msm(self.ctx.as_ptr(), points.as_ptr().cast(), scalars.as_ptr().cast(), n, flags, out.as_mut_ptr())
        };
        check(self, status)?;
        Ok(out)
    }

    /// In-place NTT of `data` (2^log_n x 32 bytes).
    pub fn fr_ntt(&mut self, data: &mut [u8], log_n: u32, flags: u32, coset_gen: Option<&[u8; 32]>) -> Result<(), BackendError> {
        let want = 32usize.checked_shl(log_n).ok_or_else(|| BackendError::serialization("fr_ntt: log_n too large"))?;
        if data.len() != want {
            return Err(BackendError::serialization("fr_ntt: buffer length is not 32 * 2^log_n"));
        }
        let cg = coset_gen.map_or(std::ptr::null(), |g| g.as_ptr());
        // SAFETY: length checked above.
        let status = unsafe { sys::b200zk_fr_ntt(self.ctx.as_ptr(), data.as_mut_ptr().cast(), log_n, flags, cg) };
        check(self, status).map(|_| ())
    }

    /// Uploads a proving-key column once; later proofs only ship scalars.
    pub fn g1_bases_upload(&mut self, points: &[u8], flags: u32) -> Result<u64, BackendError> {
        let mut handle = 0u64;
        // SAFETY: slice is valid for points.len() bytes.
        let status = unsafe { sys::b200zk_g1_bases_upload(self.ctx.as_ptr(), points.as_ptr().cast(), points.len() / 64, flags, &mut handle) };
        check(self, status)?;
        Ok(handle)
    }

    pub fn g2_bases_upload(&mut self, points: &[u8], flags: u32) -> Result<u64, BackendError> {
        let mut handle = 0u64;
        // SAFETY: slice is valid for points.len() bytes.
        let status = unsafe { sys::b200zk_g2_bases_upload(self.ctx.as_ptr(), points.as_ptr().cast(), points.len() / 128, flags, &mut handle) };
        check(self, status)?;
        Ok(handle)
    }

    /// One-off per proving-key column: expand the resident bases into their window multiples (`window_bits` 0 = automatic).
    pub fn bases_precompute(&mut self, handle: u64, window_bits: u32) -> Result<(), BackendError> {
        // SAFETY: plain value arguments.
        let status = unsafe { sys::b200zk_bases_precompute(self.ctx.as_ptr(), handle, window_bits) };
        check(self, status).map(|_| ())
    }

    pub fn bases_free(&mut self, handle: u64) -> Result<(), BackendError> {
        // SAFETY: plain value arguments.
        let status = unsafe { sys::b200zk_bases_free(self.ctx.as_ptr(), handle) };
        check(self, status).map(|_| ())
    }

    /// Selects the 2^28-th root of unity the NTT domains derive from (`None` = ark/gnark default; halo2curves'
    /// value comes from `b200zk_ntt_root_preset(1, ..)`), for wraps built on another FFT convention (`openvm.rs:52-56`).
    pub fn set_ntt_root(&mut self, root_le: Option<&[u8; 32]>) -> Result<(), BackendError> {
        let p = root_le.map_or(std::ptr::null(), |g| g.as_ptr());
        // SAFETY: NULL or 32 valid bytes.
        let status = unsafe { sys::b200zk_set_ntt_root(self.ctx.as_ptr(), p) };
        check(self, status).map(|_| ())
    }

    /// The whole Groth16 prove arithmetic (quotient NTTs, five MSMs over the RESIDENT proving key, C = L + H) in one
    /// call with one synchronisation.  `witness`: canonical LE scalars; `a`, `b`, `c`: (A z), (B z), (C z) on the
    /// domain, Montgomery LE, 2^log_n elements each.  Returns (A | B2 | C, [B]1).
    pub fn groth16_commit(&mut self, pk: &sys::b200zk_groth16_pk, witness: &[u8], a: &mut [u8], b: &mut [u8], c: &mut [u8]) -> Result<([u8; 256], [u8; 64]), BackendError> {
        check_groth16_inputs("groth16_commit", pk, witness, a, b, c)?;
        let mut proof = [0u8; 256];
        let mut b1 = [0u8; 64];
        // SAFETY: lengths checked above; host buffers outlive the synchronous call; NULL stream = the context's own.
        let status = unsafe {
            sys::b200zk_groth16_commit(self.ctx.as_ptr(), pk, witness.as_ptr().cast(), a.as_mut_ptr().cast(), b.as_mut_ptr().cast(), c.as_mut_ptr().cast(), 0,
                                       std::ptr::null_mut(), proof.as_mut_ptr(), b1.as_mut_ptr())
        };
        check(self, status)?;
        Ok((proof, b1))
    }

    /// The blinded Groth16 proof (ark-groth16 / gnark) in one call: `groth16_commit`'s pipeline, then the key's alpha /
    /// beta / delta terms (`zk.g1_terms`, `zk.g2_terms`) and the blinding scalars `zk.r`, `zk.s` added on the device.
    /// Returns A | B2 | C.
    pub fn groth16_prove(&mut self, pk: &sys::b200zk_groth16_pk, zk: &sys::b200zk_groth16_zk, witness: &[u8], a: &mut [u8], b: &mut [u8], c: &mut [u8]) -> Result<[u8; 256], BackendError> {
        check_groth16_inputs("groth16_prove", pk, witness, a, b, c)?;
        let mut proof = [0u8; 256];
        // SAFETY: lengths checked above; host buffers outlive the synchronous call; NULL stream = the context's own.
        let status = unsafe {
            sys::b200zk_groth16_prove(self.ctx.as_ptr(), pk, zk, witness.as_ptr().cast(), a.as_mut_ptr().cast(), b.as_mut_ptr().cast(), c.as_mut_ptr().cast(), 0,
                                      std::ptr::null_mut(), proof.as_mut_ptr())
        };
        check(self, status)?;
        Ok(proof)
    }

    /// Loads a snarkjs Groth16 proving key (the bytes of a `.zkey` file, as rzup fetches it for risc0-groth16) into HBM:
    /// validated, columns resident, constraint rows sorted on the device.  `precompute` also builds the columns' window
    /// tables.  Returns the key handle for `groth16_zkey_prove`.
    pub fn groth16_zkey_load(&mut self, zkey: &[u8], precompute: bool) -> Result<u64, BackendError> {
        let mut key = 0u64;
        // SAFETY: the slice outlives the synchronous call; `key` is a valid out-pointer.
        let status = unsafe { sys::b200zk_groth16_zkey_load(self.ctx.as_ptr(), zkey.as_ptr().cast(), zkey.len(), precompute as i32, &mut key) };
        check(self, status)?;
        Ok(key)
    }

    pub fn groth16_zkey_free(&mut self, key: u64) -> Result<(), BackendError> {
        // SAFETY: plain handle; the library refuses unknown ones.
        let status = unsafe { sys::b200zk_groth16_zkey_free(self.ctx.as_ptr(), key) };
        check(self, status).map(|_| ())
    }

    /// (nVars, nPublic, log2 domainSize, verifying key alpha1 | beta2 | gamma2 | delta2 | IC as EIP-196/197 bytes)
    pub fn groth16_zkey_info(&mut self, key: u64) -> Result<(u32, u32, u32, Vec<u8>), BackendError> {
        let (mut nv, mut np, mut log_n) = (0u32, 0u32, 0u32);
        // SAFETY: valid out-pointers; vk NULL asks for the sizes only.
        let status = unsafe { sys::b200zk_groth16_zkey_info(self.ctx.as_ptr(), key, &mut nv, &mut np, &mut log_n, std::ptr::null_mut(), 0) };
        check(self, status)?;
        let mut vk = vec![0u8; 448 + 64 * (np as usize + 1)];
        // SAFETY: vk holds the whole verifying key of this key (its length is passed).
        let status = unsafe {
            sys::b200zk_groth16_zkey_info(self.ctx.as_ptr(), key, std::ptr::null_mut(), std::ptr::null_mut(), std::ptr::null_mut(), vk.as_mut_ptr(), vk.len())
        };
        check(self, status)?;
        Ok((nv, np, log_n, vk))
    }

    /// The Groth16 proof A | B2 | C (what snarkjs / rapidsnark return for the same r, s) of the witness in `wtns` (the bytes
    /// of a `.wtns` file) under a key of `groth16_zkey_load`.  r, s: canonical little-endian, below the group order.
    pub fn groth16_zkey_prove(&mut self, key: u64, wtns: &[u8], r: &[u8; 32], s: &[u8; 32]) -> Result<[u8; 256], BackendError> {
        let mut proof = [0u8; 256];
        // SAFETY: the buffers outlive the synchronous call; the library parses `wtns` within its length; NULL stream = the
        // context's own.
        let status = unsafe {
            sys::b200zk_groth16_zkey_prove(self.ctx.as_ptr(), key, wtns.as_ptr().cast(), wtns.len(), r.as_ptr(), s.as_ptr(), std::ptr::null_mut(), proof.as_mut_ptr())
        };
        check(self, status)?;
        Ok(proof)
    }

    /// Verifies `proofs` (256 bytes A | B | C each) against one verifying key `vk` (the layout `groth16_zkey_info` returns,
    /// 448 + 64 (n_pub + 1) bytes) with one pairing product for the batch; `public_inputs` holds n_pub 32-byte big-endian
    /// values per proof.  One verdict per proof: a malformed proof is false, and never changes another proof's verdict.
    pub fn groth16_verify_batch(&mut self, vk: &[u8], proofs: &[u8], public_inputs: &[u8]) -> Result<Vec<bool>, BackendError> {
        if vk.len() < 512 || (vk.len() - 448) % 64 != 0 || proofs.len() % 256 != 0 {
            return Err(BackendError::serialization("groth16_verify_batch: vk must be 448 + 64 (n_pub + 1) bytes and each proof 256 bytes"));
        }
        let (n_pub, count) = ((vk.len() - 448) / 64 - 1, proofs.len() / 256);
        if public_inputs.len() != 32 * n_pub * count {
            return Err(BackendError::serialization("groth16_verify_batch: need n_pub 32-byte public inputs per proof"));
        }
        let (mut valid, mut status) = (vec![0u8; count], vec![0u8; count]);
        // SAFETY: every input holds `count` proofs' worth of its items, the outputs hold `count` bytes; NULL batch_ok is allowed.
        let status_rc = unsafe {
            sys::b200zk_groth16_verify_batch(self.ctx.as_ptr(), vk.as_ptr(), vk.len(), proofs.as_ptr(), public_inputs.as_ptr(), count, valid.as_mut_ptr(),
                                             status.as_mut_ptr(), std::ptr::null_mut())
        };
        check(self, status_rc)?;
        Ok(valid.iter().map(|&v| v == 1).collect())
    }

    /// Loads a snarkjs 0.7 PLONK proving key (the bytes of a PLONK `.zkey`) into HBM: PTau as resident bases (window tables
    /// with `precompute`), the selector and permutation polynomials on the domain and on the quotient's coset.  Returns
    /// the key handle for `plonk_zkey_prove`; Groth16 handles are not accepted there, nor PLONK handles by the Groth16 calls.
    pub fn plonk_zkey_load(&mut self, zkey: &[u8], precompute: bool) -> Result<u64, BackendError> {
        let mut key = 0u64;
        // SAFETY: the library parses `zkey` within its length and copies what it keeps.
        let status = unsafe { sys::b200zk_plonk_zkey_load(self.ctx.as_ptr(), zkey.as_ptr().cast(), zkey.len(), precompute as i32, &mut key) };
        check(self, status)?;
        Ok(key)
    }

    pub fn plonk_zkey_free(&mut self, key: u64) -> Result<(), BackendError> {
        // SAFETY: plain handle.
        let status = unsafe { sys::b200zk_plonk_zkey_free(self.ctx.as_ptr(), key) };
        check(self, status)
    }

    /// (nVars, nPublic, log2 domainSize, vk): vk = Qm Ql Qr Qo Qc S1 S2 S3 | X_2 | k1 | k2 | w, 736 bytes.
    pub fn plonk_zkey_info(&mut self, key: u64) -> Result<(u32, u32, u32, Vec<u8>), BackendError> {
        let (mut nv, mut np, mut log_n) = (0u32, 0u32, 0u32);
        let mut vk = vec![0u8; 736];
        // SAFETY: out-pointers and a 736-byte buffer, all live for the call.
        let status = unsafe { sys::b200zk_plonk_zkey_info(self.ctx.as_ptr(), key, &mut nv, &mut np, &mut log_n, vk.as_mut_ptr(), vk.len()) };
        check(self, status)?;
        Ok((nv, np, log_n, vk))
    }

    /// The 768-byte snarkjs 0.7 PLONK proof (A B C Z T1 T2 T3 Wxi Wxiw, then the six evaluations) of a `.wtns` witness.
    /// blinding = b1..b11, 32 bytes each, canonical little-endian below the group order; the caller draws them.
    pub fn plonk_zkey_prove(&mut self, key: u64, wtns: &[u8], blinding: &[[u8; 32]; 11]) -> Result<[u8; 768], BackendError> {
        let mut proof = [0u8; 768];
        // SAFETY: the buffers outlive the synchronous call ([[u8; 32]; 11] is 352 contiguous bytes); NULL stream = the
        // context's own.
        let status = unsafe {
            sys::b200zk_plonk_zkey_prove(self.ctx.as_ptr(), key, wtns.as_ptr().cast(), wtns.len(), blinding.as_ptr().cast(), std::ptr::null_mut(), proof.as_mut_ptr())
        };
        check(self, status)?;
        Ok(proof)
    }

    pub fn g1_msm_resident(&mut self, handle: u64, scalars: &[u8], flags: u32) -> Result<[u8; 64], BackendError> {
        let mut out = [0u8; 64];
        // SAFETY: slice valid; n derived from its length.
        let status = unsafe {
            sys::b200zk_g1_msm_resident(self.ctx.as_ptr(), handle, scalars.as_ptr().cast(), scalars.len() / 32, flags, out.as_mut_ptr())
        };
        check(self, status)?;
        Ok(out)
    }

    /// `blob_to_kzg_commitment_and_proof` (kzg.rs:259-272) for a batch of blobs in one call: each blob is 4096 x 32-byte
    /// big-endian field elements; `setup_handle` holds the 4096-point Lagrange-form setup.  Returns (commitments, proofs),
    /// 48 bytes compressed each.
    pub fn kzg_blob_to_commitment_and_proof(&mut self, setup_handle: u64, blobs: &[u8]) -> Result<(Vec<[u8; 48]>, Vec<[u8; 48]>), BackendError> {
        const BLOB: usize = 4096 * 32;
        if blobs.len() % BLOB != 0 {
            return Err(BackendError::serialization("kzg_blob_to_commitment_and_proof: a blob is 4096 x 32 bytes"));
        }
        let n = blobs.len() / BLOB;
        let mut commitments = vec![[0u8; 48]; n];
        let mut proofs = vec![[0u8; 48]; n];
        // SAFETY: `blobs` holds n blobs; both outputs hold n x 48 contiguous bytes; the call is synchronous.
        let status = unsafe {
            sys::b200zk_kzg_blob_to_commitment_and_proof(self.ctx.as_ptr(), setup_handle, blobs.as_ptr(), n, commitments.as_mut_ptr().cast(),
                                                         proofs.as_mut_ptr().cast())
        };
        check(self, status)?;
        Ok((commitments, proofs))
    }
}

/// Per-item outcome of the batched precompile calls (include/b200zk.h: 0 ok, 1 ok-identity, 2 coordinate >= p,
/// 3 not on the curve / not in the subgroup).
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum ItemStatus {
    Ok,
    OkIdentity,
    NotInField,
    NotOnCurve,
}

impl ItemStatus {
    fn from_code(code: u8) -> Self {
        match code {
            0 => Self::Ok,
            1 => Self::OkIdentity,
            2 => Self::NotInField,
            _ => Self::NotOnCurve,
        }
    }
}

/// Per-item outcome of `b200zk_secp256k1_ecrecover_batch` (include/b200zk.h): the reference's `CryptoError` cases of
/// `Crypto::secp256k1_ecrecover` / `recover_signer`.  Its codes mean something else than [`ItemStatus`]'s.
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum RecoverStatus {
    Ok,
    InvalidSignature,
    RecoveryFailed,
    InvalidRecoveryId,
    Unknown(u8),
}

impl RecoverStatus {
    fn from_code(code: u8) -> Self {
        match code {
            0 => Self::Ok,
            2 => Self::InvalidSignature,
            3 => Self::RecoveryFailed,
            4 => Self::InvalidRecoveryId,
            other => Self::Unknown(other),
        }
    }
}

impl B200zk {
    /// `count` independent ecAdd items: `a`, `b` = count x 64 bytes.  Returns (count x 64 result bytes, per-item status).
    pub fn bn254_g1_add_batch(&mut self, a: &[u8], b: &[u8]) -> Result<(Vec<u8>, Vec<ItemStatus>), BackendError> {
        if a.len() != b.len() || a.len() % 64 != 0 {
            return Err(BackendError::serialization("bn254_g1_add_batch: inputs must be equal multiples of 64 bytes"));
        }
        let count = a.len() / 64;
        let mut out = vec![0u8; a.len()];
        let mut st = vec![0u8; count];
        // SAFETY: all four buffers hold `count` items of the documented sizes and outlive the synchronous call.
        let status = unsafe { sys::b200zk_bn254_g1_add_batch(self.ctx.as_ptr(), a.as_ptr(), b.as_ptr(), count, out.as_mut_ptr(), st.as_mut_ptr()) };
        check(self, status)?;
        Ok((out, st.into_iter().map(ItemStatus::from_code).collect()))
    }

    /// `count` independent ecMul items: `points` = count x 64 bytes, `scalars` = count x 32 bytes (big-endian).
    pub fn bn254_g1_mul_batch(&mut self, points: &[u8], scalars: &[u8]) -> Result<(Vec<u8>, Vec<ItemStatus>), BackendError> {
        if points.len() % 64 != 0 || scalars.len() != points.len() / 2 {
            return Err(BackendError::serialization("bn254_g1_mul_batch: need 64 bytes of point and 32 of scalar per item"));
        }
        let count = points.len() / 64;
        let mut out = vec![0u8; points.len()];
        let mut st = vec![0u8; count];
        // SAFETY: as above.
        let status = unsafe { sys::b200zk_bn254_g1_mul_batch(self.ctx.as_ptr(), points.as_ptr(), scalars.as_ptr(), count, out.as_mut_ptr(), st.as_mut_ptr()) };
        check(self, status)?;
        Ok((out, st.into_iter().map(ItemStatus::from_code).collect()))
    }

    /// Several ecPairing checks in one launch.  `checks[i]` is the precompile's calldata (k x 192 bytes).
    /// Returns, per check, `Ok(true/false)` or the input error.
    pub fn bn254_pairing_check_batch(&mut self, checks: &[&[u8]]) -> Result<Vec<Result<bool, ItemStatus>>, BackendError> {
        let mut blob = Vec::new();
        let mut offsets = Vec::with_capacity(checks.len().saturating_add(1));
        offsets.push(0u32);
        for cd in checks {
            if cd.len() % 192 != 0 {
                return Err(BackendError::serialization("bn254_pairing_check_batch: calldata must be a multiple of 192 bytes"));
            }
            blob.extend_from_slice(cd);
            let pairs = u32::try_from(blob.len() / 192).map_err(|_| BackendError::serialization("bn254_pairing_check_batch: too many pairs"))?;
            offsets.push(pairs);
        }
        let count = checks.len();
        let mut res = vec![0u8; count];
        let mut st = vec![0u8; count];
        // SAFETY: `offsets` has count + 1 entries, `blob` holds offsets[count] pairs, outputs hold `count` bytes.
        let status = unsafe {
            sys::b200zk_bn254_pairing_check_batch(self.ctx.as_ptr(), blob.as_ptr(), offsets.as_ptr(), count, res.as_mut_ptr(), st.as_mut_ptr())
        };
        check(self, status)?;
        Ok(res
            .into_iter()
            .zip(st)
            .map(|(r, s)| match ItemStatus::from_code(s) {
                ItemStatus::Ok | ItemStatus::OkIdentity => Ok(r == 1),
                bad => Err(bad),
            })
            .collect())
    }

    /// Several EIP-2537 pairing checks in one launch.  `checks[i]` is the precompile's calldata (k x 384 bytes:
    /// G1 128 B | G2 256 B, every Fp as 16 zero bytes + 48 bytes big-endian).  Per check `Ok(true/false)` or the input error.
    pub fn bls12_381_pairing_check_batch(&mut self, checks: &[&[u8]]) -> Result<Vec<Result<bool, ItemStatus>>, BackendError> {
        let mut blob = Vec::new();
        let mut offsets = Vec::with_capacity(checks.len().saturating_add(1));
        offsets.push(0u32);
        for cd in checks {
            if cd.len() % 384 != 0 {
                return Err(BackendError::serialization("bls12_381_pairing_check_batch: calldata must be a multiple of 384 bytes"));
            }
            blob.extend_from_slice(cd);
            let pairs = u32::try_from(blob.len() / 384).map_err(|_| BackendError::serialization("bls12_381_pairing_check_batch: too many pairs"))?;
            offsets.push(pairs);
        }
        let count = checks.len();
        let mut res = vec![0u8; count];
        let mut st = vec![0u8; count];
        // SAFETY: `offsets` has count + 1 entries, `blob` holds offsets[count] pairs, outputs hold `count` bytes.
        let status = unsafe {
            sys::b200zk_bls12_381_pairing_check_batch(self.ctx.as_ptr(), blob.as_ptr(), offsets.as_ptr(), count, res.as_mut_ptr(), st.as_mut_ptr())
        };
        check(self, status)?;
        Ok(res
            .into_iter()
            .zip(st)
            .map(|(r, s)| match ItemStatus::from_code(s) {
                ItemStatus::Ok | ItemStatus::OkIdentity => Ok(r == 1),
                bad => Err(bad),
            })
            .collect())
    }

    /// `count` independent EIP-2537 G1ADD items: `a`, `b` = count x 128 bytes.  Returns (count x 128 result bytes, per-item status).
    pub fn bls12_381_g1_add_batch(&mut self, a: &[u8], b: &[u8]) -> Result<(Vec<u8>, Vec<ItemStatus>), BackendError> {
        self.bls12_381_add_batch(a, b, 128, "bls12_381_g1_add_batch: inputs must be equal multiples of 128 bytes", sys::b200zk_bls12_381_g1_add_batch)
    }

    /// `count` independent EIP-2537 G2ADD items: `a`, `b` = count x 256 bytes.  Returns (count x 256 result bytes, per-item status).
    pub fn bls12_381_g2_add_batch(&mut self, a: &[u8], b: &[u8]) -> Result<(Vec<u8>, Vec<ItemStatus>), BackendError> {
        self.bls12_381_add_batch(a, b, 256, "bls12_381_g2_add_batch: inputs must be equal multiples of 256 bytes", sys::b200zk_bls12_381_g2_add_batch)
    }

    /// Several EIP-2537 G1MSM calls in one launch.  `calls[i]` is the precompile's calldata (k x 160 bytes: G1 128 B |
    /// 32-byte big-endian scalar).  Per call `Ok(128 output bytes)` or the input error; an empty call is the identity.
    pub fn bls12_381_g1_msm_batch(&mut self, calls: &[&[u8]]) -> Result<Vec<Result<Vec<u8>, ItemStatus>>, BackendError> {
        self.bls12_381_msm_batch(calls, 160, 128, "bls12_381_g1_msm_batch", sys::b200zk_bls12_381_g1_msm_batch)
    }

    /// Several EIP-2537 G2MSM calls in one launch.  `calls[i]` is the precompile's calldata (k x 288 bytes: G2 256 B |
    /// 32-byte big-endian scalar).  Per call `Ok(256 output bytes)` or the input error; an empty call is the identity.
    pub fn bls12_381_g2_msm_batch(&mut self, calls: &[&[u8]]) -> Result<Vec<Result<Vec<u8>, ItemStatus>>, BackendError> {
        self.bls12_381_msm_batch(calls, 288, 256, "bls12_381_g2_msm_batch", sys::b200zk_bls12_381_g2_msm_batch)
    }

    /// `count` independent EIP-2537 MAP_FP_TO_G1 items: `fps` = count x 64 bytes.  Returns (count x 128 result bytes,
    /// per-item status); a failed item's bytes are zero.
    pub fn bls12_381_map_fp_to_g1_batch(&mut self, fps: &[u8]) -> Result<(Vec<u8>, Vec<ItemStatus>), BackendError> {
        self.bls12_381_map_batch(fps, 64, 128, "bls12_381_map_fp_to_g1_batch: input must be a multiple of 64 bytes", sys::b200zk_bls12_381_map_fp_to_g1_batch)
    }

    /// `count` independent EIP-2537 MAP_FP2_TO_G2 items: `fp2s` = count x 128 bytes (c0 | c1).  Returns (count x 256
    /// result bytes, per-item status); a failed item's bytes are zero.
    pub fn bls12_381_map_fp2_to_g2_batch(&mut self, fp2s: &[u8]) -> Result<(Vec<u8>, Vec<ItemStatus>), BackendError> {
        self.bls12_381_map_batch(fp2s, 128, 256, "bls12_381_map_fp2_to_g2_batch: input must be a multiple of 128 bytes", sys::b200zk_bls12_381_map_fp2_to_g2_batch)
    }

    /// `count` independent ECRECOVER items: `sigs` = count x 65 bytes (r | s | recid, r and s big-endian), `msgs` =
    /// count x 32-byte hashes.  `low_s` rejects s > n/2 (EIP-2, as `Crypto::recover_signer`).  Per item
    /// `Ok(keccak256 of the recovered public key)` (the address is bytes 12..32) or its status.
    pub fn secp256k1_ecrecover_batch(&mut self, sigs: &[u8], msgs: &[u8], low_s: bool) -> Result<Vec<Result<[u8; 32], RecoverStatus>>, BackendError> {
        if sigs.len() % 65 != 0 || msgs.len() % 32 != 0 || sigs.len() / 65 != msgs.len() / 32 {
            return Err(BackendError::serialization("secp256k1_ecrecover_batch: sigs must be count x 65 bytes and msgs count x 32 bytes"));
        }
        let count = sigs.len() / 65;
        let mut out = vec![0u8; msgs.len()];
        let mut st = vec![0u8; count];
        let flags = if low_s { sys::B200ZK_ECRECOVER_LOW_S } else { 0 };
        // SAFETY: `sigs` holds count x 65 bytes, `msgs` and `out` count x 32, `st` count.
        let status = unsafe {
            sys::b200zk_secp256k1_ecrecover_batch(self.ctx.as_ptr(), sigs.as_ptr(), msgs.as_ptr(), count, flags, out.as_mut_ptr(), st.as_mut_ptr())
        };
        check(self, status)?;
        Ok(out
            .chunks_exact(32)
            .zip(st)
            .map(|(h, s)| match RecoverStatus::from_code(s) {
                RecoverStatus::Ok => <[u8; 32]>::try_from(h).map_err(|_| RecoverStatus::Unknown(s)),
                bad => Err(bad),
            })
            .collect())
    }

    /// `count` independent P256VERIFY items (EIP-7951): `inputs` = count x 160 bytes, the precompile's calldata
    /// h | r | s | qx | qy (32-byte big-endian words).  Per item `true` when the signature verifies.
    pub fn secp256r1_verify_batch(&mut self, inputs: &[u8]) -> Result<Vec<bool>, BackendError> {
        if inputs.len() % 160 != 0 {
            return Err(BackendError::serialization("secp256r1_verify_batch: inputs must be count x 160 bytes"));
        }
        let count = inputs.len() / 160;
        let mut res = vec![0u8; count];
        // SAFETY: `inputs` holds count x 160 bytes and `res` count, both outliving the synchronous call.
        let status = unsafe { sys::b200zk_secp256r1_verify_batch(self.ctx.as_ptr(), inputs.as_ptr(), count, res.as_mut_ptr()) };
        check(self, status)?;
        Ok(res.into_iter().map(|r| r == 1).collect())
    }

    /// `count` independent MODEXP items (precompile 0x05): `items[i]` = (base, exponent, modulus), big-endian byte
    /// strings of any length.  Per item `Some(output)` of exactly `modulus.len()` bytes (`Crypto::modexp`'s value), or
    /// `None` when an operand is longer than [`MODEXP_MAX_BYTES`] (EIP-7823), which the device does not take.
    pub fn modexp_batch(&mut self, items: &[(&[u8], &[u8], &[u8])]) -> Result<Vec<Option<Vec<u8>>>, BackendError> {
        let mut data = Vec::new();
        let mut lens = Vec::with_capacity(items.len().saturating_mul(3));
        let mut out_len = 0usize;
        for (b, e, m) in items {
            for op in [b, e, m] {
                data.extend_from_slice(op);
                lens.push(u32::try_from(op.len()).map_err(|_| BackendError::serialization("modexp_batch: an operand is longer than 2^32 - 1 bytes"))?);
            }
            out_len = out_len.checked_add(m.len()).ok_or_else(|| BackendError::serialization("modexp_batch: output length overflows"))?;
        }
        let count = items.len();
        let mut out = vec![0u8; out_len];
        let mut st = vec![0u8; count];
        // SAFETY: `lens` holds 3 x count lengths whose operands are back to back in `data`, `out` the sum of the modulus
        // lengths and `st` count bytes, all outliving the synchronous call.
        let status = unsafe { sys::b200zk_modexp_batch(self.ctx.as_ptr(), data.as_ptr(), lens.as_ptr(), count, out.as_mut_ptr(), st.as_mut_ptr()) };
        check(self, status)?;
        let mut rest = out.as_slice();
        let mut res = Vec::with_capacity(count);
        for ((_, _, m), s) in items.iter().zip(st) {
            let (head, tail) = rest.split_at(m.len().min(rest.len()));
            rest = tail;
            res.push(if s == 0 { Some(head.to_vec()) } else { None });
        }
        Ok(res)
    }

    fn bls12_381_add_batch(
        &mut self,
        a: &[u8],
        b: &[u8],
        size: usize,
        what: &'static str,
        f: unsafe extern "C" fn(*mut sys::b200zk_ctx, *const u8, *const u8, usize, *mut u8, *mut u8) -> std::os::raw::c_int,
    ) -> Result<(Vec<u8>, Vec<ItemStatus>), BackendError> {
        if a.len() != b.len() || a.len() % size != 0 {
            return Err(BackendError::serialization(what));
        }
        let count = a.len() / size;
        let mut out = vec![0u8; a.len()];
        let mut st = vec![0u8; count];
        // SAFETY: all four buffers hold `count` items of the documented sizes and outlive the synchronous call.
        let status = unsafe { f(self.ctx.as_ptr(), a.as_ptr(), b.as_ptr(), count, out.as_mut_ptr(), st.as_mut_ptr()) };
        check(self, status)?;
        Ok((out, st.into_iter().map(ItemStatus::from_code).collect()))
    }

    fn bls12_381_map_batch(
        &mut self,
        input: &[u8],
        size: usize,
        out_size: usize,
        what: &'static str,
        f: unsafe extern "C" fn(*mut sys::b200zk_ctx, *const u8, usize, *mut u8, *mut u8) -> std::os::raw::c_int,
    ) -> Result<(Vec<u8>, Vec<ItemStatus>), BackendError> {
        if input.len() % size != 0 {
            return Err(BackendError::serialization(what));
        }
        let count = input.len() / size;
        let mut out = vec![0u8; count.saturating_mul(out_size)];
        let mut st = vec![0u8; count];
        // SAFETY: all three buffers hold `count` items of the documented sizes and outlive the synchronous call.
        let status = unsafe { f(self.ctx.as_ptr(), input.as_ptr(), count, out.as_mut_ptr(), st.as_mut_ptr()) };
        check(self, status)?;
        Ok((out, st.into_iter().map(ItemStatus::from_code).collect()))
    }

    fn bls12_381_msm_batch(
        &mut self,
        calls: &[&[u8]],
        pair: usize,
        size: usize,
        what: &'static str,
        f: unsafe extern "C" fn(*mut sys::b200zk_ctx, *const u8, *const u32, usize, *mut u8, *mut u8) -> std::os::raw::c_int,
    ) -> Result<Vec<Result<Vec<u8>, ItemStatus>>, BackendError> {
        let mut blob = Vec::new();
        let mut offsets = Vec::with_capacity(calls.len().saturating_add(1));
        offsets.push(0u32);
        for cd in calls {
            if cd.len() % pair != 0 {
                return Err(BackendError::serialization(format!("{what}: calldata must be a multiple of {pair} bytes")));
            }
            blob.extend_from_slice(cd);
            let pairs = u32::try_from(blob.len() / pair).map_err(|_| BackendError::serialization(format!("{what}: too many pairs")))?;
            offsets.push(pairs);
        }
        let count = calls.len();
        let mut out = vec![0u8; count.saturating_mul(size)];
        let mut st = vec![0u8; count];
        // SAFETY: `offsets` has count + 1 entries, `blob` holds offsets[count] pairs, `out` holds count x size bytes and
        // `st` count bytes.
        let status = unsafe { f(self.ctx.as_ptr(), blob.as_ptr(), offsets.as_ptr(), count, out.as_mut_ptr(), st.as_mut_ptr()) };
        check(self, status)?;
        Ok(out
            .chunks(size)
            .zip(st)
            .map(|(o, s)| match ItemStatus::from_code(s) {
                ItemStatus::Ok | ItemStatus::OkIdentity => Ok(o.to_vec()),
                bad => Err(bad),
            })
            .collect())
    }

    /// Upload a KZG setup's G2 points (96-byte compressed, `g2_monomial` order: [1]2, [tau]2, ...), subgroup-checked.
    /// The handle is what the two KZG verify calls take; free it with `bases_free`.
    pub fn bls12_381_g2_bases_upload(&mut self, points: &[u8]) -> Result<u64, BackendError> {
        if points.len() % 96 != 0 {
            return Err(BackendError::serialization("bls12_381_g2_bases_upload: points are 96 bytes each"));
        }
        let mut handle = 0u64;
        // SAFETY: `points` holds len/96 compressed points; `handle` is a valid out pointer.
        let status = unsafe { sys::b200zk_bls12_381_g2_bases_upload(self.ctx.as_ptr(), points.as_ptr().cast(), points.len() / 96, sys::B200ZK_POINTS_COMPRESSED, &mut handle) };
        check(self, status)?;
        Ok(handle)
    }

    /// c-kzg `verify_kzg_proof` for n items (commitments and proofs n x 48 bytes, z and y n x 32 bytes big-endian):
    /// per item `Ok(valid)` or the input error (c-kzg's BADARGS).
    pub fn kzg_verify_proof_batch(&mut self, g2_setup: u64, commitments: &[u8], z: &[u8], y: &[u8], proofs: &[u8]) -> Result<Vec<Result<bool, ItemStatus>>, BackendError> {
        let n = commitments.len() / 48;
        if commitments.len() % 48 != 0 || proofs.len() != 48 * n || z.len() != 32 * n || y.len() != 32 * n {
            return Err(BackendError::serialization("kzg_verify_proof_batch: need 48 + 32 + 32 + 48 bytes per item"));
        }
        let mut res = vec![0u8; n];
        let mut st = vec![0u8; n];
        // SAFETY: every input holds n items of its size, outputs hold n bytes.
        let status = unsafe {
            sys::b200zk_kzg_verify_proof_batch(self.ctx.as_ptr(), g2_setup, commitments.as_ptr(), z.as_ptr(), y.as_ptr(), proofs.as_ptr(), n, res.as_mut_ptr(), st.as_mut_ptr())
        };
        check(self, status)?;
        Ok(res
            .into_iter()
            .zip(st)
            .map(|(r, s)| match ItemStatus::from_code(s) {
                ItemStatus::Ok | ItemStatus::OkIdentity => Ok(r == 1),
                bad => Err(bad),
            })
            .collect())
    }

    /// c-kzg `verify_blob_kzg_proof_batch`: one answer for n (blob, commitment, proof) triples; malformed input is an error.
    pub fn kzg_verify_blob_proof_batch(&mut self, g2_setup: u64, blobs: &[u8], commitments: &[u8], proofs: &[u8]) -> Result<bool, BackendError> {
        const BLOB: usize = 4096 * 32;
        let n = blobs.len() / BLOB;
        if blobs.len() % BLOB != 0 || commitments.len() != 48 * n || proofs.len() != 48 * n {
            return Err(BackendError::serialization("kzg_verify_blob_proof_batch: need 131072 + 48 + 48 bytes per blob"));
        }
        let mut valid: core::ffi::c_int = 0;
        // SAFETY: every input holds n items of its size; `valid` is a valid out pointer.
        let status = unsafe { sys::b200zk_kzg_verify_blob_proof_batch(self.ctx.as_ptr(), g2_setup, blobs.as_ptr(), commitments.as_ptr(), proofs.as_ptr(), n, &mut valid) };
        check(self, status)?;
        Ok(valid == 1)
    }

    /// c-kzg `compute_cells` for n blobs: n x 128 cells of 2048 bytes, blob-major; the first 64 cells of a blob are the
    /// blob itself.  A blob element >= r is an error.
    pub fn kzg_compute_cells(&mut self, blobs: &[u8]) -> Result<Vec<u8>, BackendError> {
        const BLOB: usize = 4096 * 32;
        let n = blobs.len() / BLOB;
        if blobs.len() % BLOB != 0 {
            return Err(BackendError::serialization("kzg_compute_cells: blobs must be n x 131072 bytes"));
        }
        let mut cells = vec![0u8; 2 * BLOB * n];
        // SAFETY: `blobs` holds n blobs and `cells` 2 x 131072 bytes per blob.
        let status = unsafe { sys::b200zk_kzg_compute_cells(self.ctx.as_ptr(), blobs.as_ptr(), n, cells.as_mut_ptr()) };
        check(self, status)?;
        Ok(cells)
    }

    /// `kzg::blob_to_commitment_and_cell_proofs` for n blobs: (n x 48 commitment bytes, n x 128 x 48 cell-proof bytes,
    /// blob-major with the cell index inner).  `g1_lagrange` is the 4096-point Lagrange setup, `g1_monomial` the setup's
    /// 4096 points [tau^i]1.  A blob element >= r is an error.
    pub fn kzg_blob_to_commitment_and_cell_proofs(&mut self, g1_lagrange: u64, g1_monomial: u64, blobs: &[u8]) -> Result<(Vec<u8>, Vec<u8>), BackendError> {
        const BLOB: usize = 4096 * 32;
        let n = blobs.len() / BLOB;
        if blobs.len() % BLOB != 0 {
            return Err(BackendError::serialization("kzg_blob_to_commitment_and_cell_proofs: blobs must be n x 131072 bytes"));
        }
        let mut commitments = vec![0u8; 48 * n];
        let mut proofs = vec![0u8; 128 * 48 * n];
        // SAFETY: `blobs` holds n blobs, `commitments` 48 bytes and `proofs` 128 x 48 bytes per blob.
        let status = unsafe {
            sys::b200zk_kzg_blob_to_commitment_and_cell_proofs(self.ctx.as_ptr(), g1_lagrange, g1_monomial, blobs.as_ptr(), n, commitments.as_mut_ptr(), proofs.as_mut_ptr())
        };
        check(self, status)?;
        Ok((commitments, proofs))
    }

    /// c-kzg `recover_cells_and_kzg_proofs` for n = `cell_offsets.len() - 1` blobs: blob b's given cells are entries
    /// `cell_offsets[b] .. cell_offsets[b + 1]` of `cell_indices` and `cells` (2048 bytes each), 64 to 128 distinct indices
    /// below 128 in any order.  Returns (n x 128 cells of 2048 bytes, n x 128 x 48 cell-proof bytes), both blob-major with
    /// the cell index inner.  `g1_monomial` is the setup's 4096 points [tau^i]1.  Malformed input, or given cells that do
    /// not all lie on one blob's extension, is an error.
    pub fn kzg_recover_cells_and_cell_proofs(&mut self, g1_monomial: u64, cell_offsets: &[u32], cell_indices: &[u64], cells: &[u8]) -> Result<(Vec<u8>, Vec<u8>), BackendError> {
        const CELL: usize = 64 * 32;
        let n = cell_offsets.len().saturating_sub(1);
        let total = cell_offsets.last().map_or(0, |&t| t as usize);
        if cell_offsets.is_empty() || cell_indices.len() != total || cells.len() != CELL * total {
            return Err(BackendError::serialization("kzg_recover_cells_and_cell_proofs: need n + 1 offsets, and an index and 2048 bytes per given cell"));
        }
        let mut cells_out = vec![0u8; 128 * CELL * n];
        let mut proofs = vec![0u8; 128 * 48 * n];
        // SAFETY: `cell_offsets` holds n + 1 entries, `cell_indices` and `cells` one index and 2048 bytes for each of the
        // `cell_offsets[n]` given cells (the library checks the offsets before reading through them); the outputs hold 128
        // cells and 128 proofs per blob.
        let status = unsafe {
            sys::b200zk_kzg_recover_cells_and_cell_proofs(self.ctx.as_ptr(), g1_monomial, cell_offsets.as_ptr(), cell_indices.as_ptr(), cells.as_ptr(), n,
                                                          cells_out.as_mut_ptr(), proofs.as_mut_ptr())
        };
        check(self, status)?;
        Ok((cells_out, proofs))
    }

    /// `verify_cell_kzg_proof_batch` over whole blobs (every cell, each commitment once per blob, proofs blob-major with
    /// 128 per blob): one answer; malformed input is an error.  `g1_setup` is the 4096-point Lagrange setup, `g2_setup`
    /// the setup's 65 G2 points.
    pub fn kzg_verify_cell_proof_batch(&mut self, g1_setup: u64, g2_setup: u64, blobs: &[u8], commitments: &[u8], proofs: &[u8]) -> Result<bool, BackendError> {
        const BLOB: usize = 4096 * 32;
        let n = blobs.len() / BLOB;
        if blobs.len() % BLOB != 0 || commitments.len() != 48 * n || proofs.len() != 128 * 48 * n {
            return Err(BackendError::serialization("kzg_verify_cell_proof_batch: need 131072 + 48 + 128 x 48 bytes per blob"));
        }
        let mut valid: core::ffi::c_int = 0;
        // SAFETY: every input holds n blobs' worth of its items; `valid` is a valid out pointer.
        let status = unsafe {
            sys::b200zk_kzg_verify_cell_proof_batch(self.ctx.as_ptr(), g1_setup, g2_setup, blobs.as_ptr(), commitments.as_ptr(), proofs.as_ptr(), n, &mut valid)
        };
        check(self, status)?;
        Ok(valid == 1)
    }

    /// c-kzg `verify_cell_kzg_proof_batch(commitments, cell_indices, cells, proofs)` over any n cells without their blobs
    /// (a data column, custody or sampling columns, the cells about to be recovered): 48 bytes of commitment, one index,
    /// 2048 bytes of cell and 48 bytes of proof per cell.  One answer; malformed input is an error.  The handles are those
    /// of `kzg_verify_cell_proof_batch`.
    pub fn kzg_verify_cells(&mut self, g1_setup: u64, g2_setup: u64, commitments: &[u8], cell_indices: &[u64], cells: &[u8], proofs: &[u8]) -> Result<bool, BackendError> {
        const CELL: usize = 64 * 32;
        let n = cell_indices.len();
        if commitments.len() != 48 * n || cells.len() != CELL * n || proofs.len() != 48 * n {
            return Err(BackendError::serialization("kzg_verify_cells: need 48 + 2048 + 48 bytes and one index per cell"));
        }
        let mut valid: core::ffi::c_int = 0;
        // SAFETY: every input holds n cells' worth of its items; `valid` is a valid out pointer.
        let status = unsafe {
            sys::b200zk_kzg_verify_cells(self.ctx.as_ptr(), g1_setup, g2_setup, commitments.as_ptr(), cell_indices.as_ptr(), cells.as_ptr(), proofs.as_ptr(), n,
                                         &mut valid)
        };
        check(self, status)?;
        Ok(valid == 1)
    }
}

impl Drop for B200zk {
    fn drop(&mut self) {
        // SAFETY: ctx came from b200zk_init and is dropped exactly once.
        unsafe { sys::b200zk_destroy(self.ctx.as_ptr()) }
    }
}
