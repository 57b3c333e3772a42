//! `B200Backend`: a `ProverBackend` (`crates/prover/src/backend/mod.rs:81-147`) whose BN254 arithmetic -- the
//! G1/G2 multi-scalar multiplications and Fr NTTs of the Groth16 wrap that the reference reaches only inside
//! third-party SDKs when the coordinator asks for `ProofFormat::Groth16`
//! (`crates/l2/sequencer/proof_coordinator.rs:252-256`, `crates/prover/src/backend/sp1.rs:97-134`) -- runs on
//! an H100 through `libb200zk.so`.
//!
//! Scope (SURVEY.md section 8b): this backend does not introduce a new proof system.  It reports the
//! `ProverType` of the zkVM whose on-chain Groth16 verifier it targets and replaces the *commitment
//! arithmetic* of that zkVM's wrap stage.  The wrap circuit itself (R1CS + proving key) belongs to the
//! zkVM SDK and is injected through [`WrapCircuit`]; without one, `prove` returns
//! `BackendError::NotImplemented` for `ProofFormat::Groth16`, exactly like a backend built without its SDK.
//! Drop this file in as `crates/prover/src/backend/b200.rs` (wiring in INTEGRATION.md).
use std::io::Read;
use std::sync::OnceLock;
use std::time::{Duration, Instant};

use ethrex_common::types::prover::{ProofBytes, ProofFormat, ProverOutput, ProverType};
use ethrex_guest_program::input::ProgramInput;
use rkyv::rancor::Error;
use tracing::info;

use ethrex_prover::backend::{BackendError, ExecBackend, ProverBackend};

use crate::ffi;

/// What the zkVM SDK has to provide for the Groth16 wrap: the witness vector and the proving key in the layout of
/// ark-groth16 / gnark (query columns plus the separate alpha, beta, delta terms).
/// All buffers use the library's native formats (ark-ff Montgomery limbs for points, canonical limbs for
/// scalars), i.e. the in-memory form the arkworks-based wrap provers already hold them in.
pub trait WrapCircuit: Send + Sync {
    /// `ProverType` whose on-chain verifier checks the produced proof (`crates/common/types/prover.rs:7-23`).
    fn prover_type(&self) -> ProverType;
    /// log2 of the evaluation-domain size.
    fn domain_log2(&self) -> u32;
    /// Number of public R1CS variables INCLUDING the leading constant 1: the L column starts behind them.
    fn n_public(&self) -> usize;
    /// Full witness assignment (1, public inputs, private variables), canonical 32-byte little-endian scalars --
    /// one scalar per point of `pk_a_g1`.
    fn witness(&self, serialized_input: &[u8]) -> Result<Vec<u8>, BackendError>;
    /// Proving-key columns as native affine points: A (G1), B (G1), B (G2) with one point per variable; L (G1) with
    /// one point per PRIVATE variable; H (G1) with one point per quotient coefficient (2^k - 1 points).  alpha and
    /// beta are NOT folded into the columns (ark-groth16 `a_query` / `b_g1_query` / `b_g2_query`, gnark `G1.A` ...).
    fn pk_a_g1(&self) -> &[u8];
    fn pk_b_g1(&self) -> &[u8];
    fn pk_b_g2(&self) -> &[u8];
    fn pk_l_g1(&self) -> &[u8];
    fn pk_h_g1(&self) -> &[u8];
    /// The key terms as native affine points: alpha, beta, delta in G1 (64 bytes each), beta, delta in G2 (128 bytes
    /// each).  The device adds them and the blinding r delta1, s delta2, s A + r B1 - r s delta1 to the proof.
    fn pk_alpha_g1(&self) -> &[u8];
    fn pk_beta_g1(&self) -> &[u8];
    fn pk_beta_g2(&self) -> &[u8];
    fn pk_delta_g1(&self) -> &[u8];
    fn pk_delta_g2(&self) -> &[u8];
    /// Evaluations of A*w, B*w, C*w over the domain (Montgomery limbs), from which the library builds the quotient H.
    fn abc_evaluations(&self, witness: &[u8]) -> Result<[Vec<u8>; 3], BackendError>;
    /// Final encoding with the SDK's selector bytes (`sp1.rs:176-194`, `risc0.rs:43-59`); `proof` is the blinded
    /// A | B2 | C the device produced.
    fn assemble(&self, proof: &[u8; 256]) -> Result<Vec<u8>, BackendError>;
    /// The ecpairing calldata of the Groth16 verification equation for `proof`
    /// (`-A | B | alpha | beta | IC(public inputs) | gamma | C | delta`, 4 x 192 bytes), when the SDK exposes its
    /// verifying key; `None` makes `verify` answer "not implemented", like the reference's default.
    fn verifier_calldata(&self, _proof: &[u8]) -> Option<Vec<u8>> {
        None
    }
}

pub struct B200ProveOutput {
    pub prover_type: ProverType,
    pub proof: Vec<u8>,
}

/// The proving key as it lives in HBM across proofs: uploaded and expanded into window tables ONCE per process, like
/// `static PROVER_SETUP: OnceLock<ProverSetup>` in the reference (`sp1.rs:30,93-95`).
struct ResidentKey {
    pk: b200zk_sys::b200zk_groth16_pk,
    g1_terms: u64,
    g2_terms: u64,
}

/// The BN254 group order r, little-endian bytes.
const FR_ORDER_LE: [u8; 32] = [
    0x01, 0x00, 0x00, 0xf0, 0x93, 0xf5, 0xe1, 0x43, 0x91, 0x70, 0xb9, 0x79, 0x48, 0xe8, 0x33, 0x28, 0x5d, 0x58, 0x81, 0x81, 0xb6, 0x45,
    0x50, 0xb8, 0x29, 0xa0, 0x31, 0xe1, 0x72, 0x4e, 0x64, 0x30,
];

fn below_order(x: &[u8; 32]) -> bool {
    for (a, b) in x.iter().rev().zip(FR_ORDER_LE.iter().rev()) {
        if a != b {
            return a < b;
        }
    }
    false
}

/// A uniform blinding scalar in [0, r), canonical little-endian: 254 random bits, drawn again while the value is >= r.
/// Rejection rather than a reduction mod r, which would make the values below 2^254 - r twice as likely; fewer than two
/// draws are needed on average.
fn blinding_scalar(rng: &mut impl Read) -> Result<[u8; 32], BackendError> {
    loop {
        let mut x = [0u8; 32];
        rng.read_exact(&mut x).map_err(BackendError::proving)?;
        if let Some(top) = x.last_mut() {
            *top &= 0x3f;
        }
        if below_order(&x) {
            return Ok(x);
        }
    }
}

#[derive(Default)]
pub struct B200Backend {
    circuit: Option<Box<dyn WrapCircuit>>,
    resident: OnceLock<Result<ResidentKey, String>>,
}

fn count_of(bytes: &[u8], point: usize) -> Result<u64, BackendError> {
    if bytes.len() % point != 0 {
        return Err(BackendError::serialization("proving-key column is not a whole number of points"));
    }
    u64::try_from(bytes.len() / point).map_err(BackendError::serialization)
}

impl B200Backend {
    pub fn new() -> Self {
        Self { circuit: None, resident: OnceLock::new() }
    }

    pub fn with_circuit(circuit: Box<dyn WrapCircuit>) -> Self {
        Self { circuit: Some(circuit), resident: OnceLock::new() }
    }

    /// Upload + precompute the five columns and upload the key terms once; checks the sizes against each other instead
    /// of truncating.
    fn load_key(circuit: &dyn WrapCircuit, gpu: &mut ffi::B200zk) -> Result<ResidentKey, BackendError> {
        let k = circuit.domain_log2();
        let n = 1u64.checked_shl(k).ok_or_else(|| BackendError::serialization("domain too large"))?;
        let n_pub = u64::try_from(circuit.n_public()).map_err(BackendError::serialization)?;
        let m = count_of(circuit.pk_a_g1(), 64)?;
        let (mb1, mb2) = (count_of(circuit.pk_b_g1(), 64)?, count_of(circuit.pk_b_g2(), 128)?);
        let (ml, mh) = (count_of(circuit.pk_l_g1(), 64)?, count_of(circuit.pk_h_g1(), 64)?);
        if mb1 != m || mb2 != m || n_pub > m || ml != m.saturating_sub(n_pub) || mh.saturating_add(1) != n {
            return Err(BackendError::serialization(format!(
                "proving-key columns disagree: A {m}, B1 {mb1}, B2 {mb2} (must be equal), L {ml} (must be A - {n_pub} public), H {mh} (must be 2^{k} - 1)"
            )));
        }
        let g1_sizes = [circuit.pk_alpha_g1().len(), circuit.pk_beta_g1().len(), circuit.pk_delta_g1().len()];
        let g2_sizes = [circuit.pk_beta_g2().len(), circuit.pk_delta_g2().len()];
        if g1_sizes != [64; 3] || g2_sizes != [128; 2] {
            return Err(BackendError::serialization("key terms: alpha, beta, delta in G1 are 64 bytes each, beta and delta in G2 128 bytes each"));
        }
        // plain bases: the key terms are three scalar multiplications' worth of work, not an MSM
        let g1_terms = gpu.g1_bases_upload(&[circuit.pk_alpha_g1(), circuit.pk_beta_g1(), circuit.pk_delta_g1()].concat(), 0)?;
        let g2_terms = gpu.g2_bases_upload(&[circuit.pk_beta_g2(), circuit.pk_delta_g2()].concat(), 0)?;
        let handles = [
            gpu.g1_bases_upload(circuit.pk_a_g1(), 0)?,
            gpu.g1_bases_upload(circuit.pk_b_g1(), 0)?,
            gpu.g2_bases_upload(circuit.pk_b_g2(), 0)?,
            gpu.g1_bases_upload(circuit.pk_l_g1(), 0)?,
            gpu.g1_bases_upload(circuit.pk_h_g1(), 0)?,
        ];
        for h in handles {
            gpu.bases_precompute(h, 0)?;
        }
        Ok(ResidentKey {
            pk: b200zk_sys::b200zk_groth16_pk { log_n: k, reserved: 0, handle: handles, count: [m, m, m, ml, mh], offset: [0, 0, 0, n_pub, 0] },
            g1_terms,
            g2_terms,
        })
    }

    /// The hot path: one call -- 3 iNTT + 3 coset NTT + quotient + 1 coset iNTT, 4 G1 MSMs + 1 G2 MSM over the
    /// resident key (A, B1, B2 share one digit sort), then the key terms and the blinding with fresh r, s from the
    /// OS's random source -- and one synchronisation.
    fn prove_blinded(&self, circuit: &dyn WrapCircuit, serialized: &[u8]) -> Result<[u8; 256], BackendError> {
        let gpu = ffi::global()?;
        let mut gpu = gpu.lock().map_err(|_| BackendError::proving("b200zk context poisoned"))?;
        let key = self
            .resident
            .get_or_init(|| Self::load_key(circuit, &mut gpu).map_err(|e| e.to_string()))
            .as_ref()
            .map_err(BackendError::proving)?;
        let witness = circuit.witness(serialized)?;
        let [mut a, mut b, mut c] = circuit.abc_evaluations(&witness)?;
        let mut urandom = std::fs::File::open("/dev/urandom").map_err(BackendError::proving)?;
        let zk = b200zk_sys::b200zk_groth16_zk {
            g1_terms: key.g1_terms,
            g2_terms: key.g2_terms,
            r: blinding_scalar(&mut urandom)?,
            s: blinding_scalar(&mut urandom)?,
        };
        gpu.groth16_prove(&key.pk, &zk, &witness, &mut a, &mut b, &mut c)
    }
}

impl ProverBackend for B200Backend {
    type ProofOutput = B200ProveOutput;
    type SerializedInput = Vec<u8>;

    fn prover_type(&self) -> ProverType {
        self.circuit.as_ref().map_or(ProverType::Exec, |c| c.prover_type())
    }

    fn serialize_input(&self, input: &ProgramInput) -> Result<Self::SerializedInput, BackendError> {
        // same wire form the zkVM backends feed their guests (sp1.rs:145-150)
        let bytes = rkyv::to_bytes::<Error>(input).map_err(BackendError::serialization)?;
        Ok(bytes.to_vec())
    }

    fn execute(&self, input: ProgramInput) -> Result<(), BackendError> {
        ExecBackend::new().execute(input)
    }

    fn prove(&self, input: ProgramInput, format: ProofFormat) -> Result<Self::ProofOutput, BackendError> {
        let serialized = self.serialize_input(&input)?;
        // the guest program must accept the batch before anything is committed to
        ExecBackend::new().execute(input)?;
        match (format, self.circuit.as_deref()) {
            (ProofFormat::Groth16, Some(circuit)) => {
                let proof = self.prove_blinded(circuit, &serialized)?;
                Ok(B200ProveOutput { prover_type: circuit.prover_type(), proof: circuit.assemble(&proof)? })
            }
            (ProofFormat::Groth16, None) => Err(BackendError::not_implemented(
                "b200 backend built without a wrap circuit: ProofFormat::Groth16 needs a zkVM SDK's proving key",
            )),
            (ProofFormat::Compressed, _) => Err(BackendError::not_implemented(
                "b200 backend accelerates the BN254 wrap only; Compressed (STARK) proofs come from the zkVM backend",
            )),
        }
    }

    /// The pairing check of the Groth16 verification equation, on the device (`b200zk_bn254_pairing_check_batch`).
    fn verify(&self, proof: &Self::ProofOutput) -> Result<(), BackendError> {
        let calldata = self
            .circuit
            .as_ref()
            .and_then(|c| c.verifier_calldata(&proof.proof))
            .ok_or_else(BackendError::verify_not_supported)?;
        let mut gpu = ffi::global()?.lock().map_err(|e| BackendError::verification(e.to_string()))?;
        match gpu.bn254_pairing_check_batch(&[calldata.as_slice()])?.first() {
            Some(Ok(true)) => Ok(()),
            Some(Ok(false)) => Err(BackendError::verification("Groth16 pairing check failed")),
            Some(Err(status)) => Err(BackendError::verification(format!("malformed proof point: {status:?}"))),
            None => Err(BackendError::verification("b200zk returned no result")),
        }
    }

    fn to_proof_bytes(&self, proof: Self::ProofOutput, _format: ProofFormat) -> Result<ProverOutput, BackendError> {
        Ok(ProverOutput::Proof(ProofBytes { prover_type: proof.prover_type, proof: proof.proof }))
    }

    fn prove_timed(&self, input: ProgramInput, format: ProofFormat) -> Result<(Self::ProofOutput, Duration), BackendError> {
        let start = Instant::now();
        let proof = self.prove(input, format)?;
        let elapsed = start.elapsed();
        // the caller (`Prover::poll_endpoints`, crates/prover/src/prover.rs:106-118) logs `proving_time_s` / `proving_time_ms`
        // from this Duration; the backend adds the same two fields for its own share of it
        info!(proving_time_s = elapsed.as_secs(), proving_time_ms = u64::try_from(elapsed.as_millis()).unwrap_or(u64::MAX), "b200 backend proved in {:.2?}", elapsed);
        Ok((proof, elapsed))
    }
}
