//! H100 prover backend for ethrex: safe wrapper over `b200zk-sys` plus the `ProverBackend` implementation.
pub mod b200;
pub mod crypto;
pub mod ffi;
pub use b200::B200Backend;
pub use crypto::B200Crypto;
