//! Safe wrappers over `libb200prover` with the shapes of the upstream calls they replace:
//!
//! | reference call site | upstream call | wrapper |
//! |---|---|---|
//! | `circuit-types/src/traits.rs:850`  | `PlonkKzgSnark::preprocess(&SYSTEM_SRS, &cs)` | [`GpuProver::preprocess`] |
//! | `circuit-types/src/traits.rs:996`  | `PlonkKzgSnark::prove_with_link_hint::<_, _, SolidityTranscript>(rng, &circuit, &pk)` | [`GpuProver::prove_with_link_hint`] |
//! | `circuit-types/src/traits.rs:1012` | `PlonkKzgSnark::verify::<SolidityTranscript>(&vk, pi, &proof, None)` | [`verify`] (host only) |
//! | `circuit-types/src/traits.rs:850`  | the same, keeping the wiring on the device | [`GpuProver::preprocess_wiring`] |
//! | `circuit-types/src/traits.rs:996`  | the same, from `cs.witness()` instead of the 5 x n value table | [`GpuProver::prove_from_witness`] |
//! | `circuit-types/src/traits.rs:996`  | the same for many witnesses of one key, in one pool job | [`GpuProver::prove_from_witness_batch`] |
//! | `proof_linking/intent_only.rs:42-47` | `PlonkKzgSnark::link_proofs::<SolidityTranscript>(a, b, &layout, &ck)` | [`GpuProver::link_proofs`] |
//! | `native_proof_manager.rs:726-782` | the four `link_proofs` calls of `compute_private_settlement_link_proofs` | [`GpuProver::link_proofs_batch`] |
//! | `native_proof_manager.rs:514-660` | a settlement arm: `singleprover_prove_with_hint`, then `link_proofs` against each stored hint | [`GpuProver::prove_settlement`], [`GpuProver::prove_settlement_from_witness`] |
//! | `gossip-server/src/orderbook.rs:180-229` | the order check: two proofs and one link proof per order (`todo!` upstream) | [`GpuProver::submit_verify`], [`GpuProver::submit_verify_combined`] |
//! | `primitives/srs.rs:63-71` | `parse_ptau_file` + `powers_of_g` | [`GpuProver::load_srs`] |
//! | `native_proof_manager.rs:167-178` | the cancel channel: `ProofManagerError::Cancelled` at once | [`GpuProver::cancel_all`], [`GpuProver::shutdown_now`] |
//! | `circuit-types/src/traits.rs:850`  | the same, for domains up to 2^23: round 3 one coset at a time | [`GpuProver::preprocess_wiring_compact`] |
//!
//! Marshalling rules (SURVEY.md §7 "Rust ABI hazards"): `Fr`/`Fq` are `Fp(BigInt<4>, PhantomData)` holding the
//! Montgomery limbs — reading `.0 .0` is the value the C ABI wants; `G1Affine` is `repr(Rust)` {x, y, infinity} and is
//! NEVER passed by pointer — it is marshalled to the packed 64-byte x || y record (the SRS file's own record,
//! srs.rs:172-182).  Errors: non-zero status -> `PlonkError` -> `ProverError::Plonk` (errors.rs:41); the library never
//! panics, aborts or unwinds across the boundary.
//!
//! NOT compiled in the build image (no cargo there).  `mpc_relation::PlonkCircuit` accessors used below
//! (`selector_evals`, `wire_permutation_flat`, `witness_table`, `wire_variables`, `witness`) are thin getters over fields
//! the fork already has.
#![allow(unsafe_code)]
pub mod ffi;
pub mod ffi_settlement;
pub mod ffi_verifyjobs;
pub mod ffi_express;
pub mod ffi_reserved;
pub mod ffi_selftest;
pub mod ffi_cancel;
pub mod ffi_compact;

use ark_bn254::{Bn254, Fq, Fr, G1Affine};
use ark_ff::{BigInt, UniformRand};
use mpc_plonk::errors::PlonkError;
use mpc_plonk::proof_system::structs::{LinkingHint, Proof, ProofEvaluations};
use mpc_relation::proof_linking::GroupLayout;
use mpc_relation::PlonkCircuit;
use std::ffi::CStr;
use std::os::raw::{c_int, c_uint};

fn fr_limbs(x: &Fr) -> [u64; 4] {
    (x.0).0
}
fn fr_from(l: &[u64; 4]) -> Fr {
    Fr::new_unchecked(BigInt(*l)) // already Montgomery, like srs.rs:201-209
}
fn g1_from(xy: &[u64; 8]) -> G1Affine {
    if xy.iter().all(|l| *l == 0) {
        return G1Affine::identity();
    }
    let x = Fq::new_unchecked(BigInt([xy[0], xy[1], xy[2], xy[3]]));
    let y = Fq::new_unchecked(BigInt([xy[4], xy[5], xy[6], xy[7]]));
    G1Affine::new_unchecked(x, y)
}
fn g1_record(p: &G1Affine) -> [u64; 8] {
    if p.infinity {
        return [0; 8];
    }
    let (x, y) = ((p.x.0).0, (p.y.0).0);
    [x[0], x[1], x[2], x[3], y[0], y[1], y[2], y[3]]
}

fn check(rc: c_int) -> Result<(), PlonkError> {
    if rc == ffi::B200_OK {
        return Ok(());
    }
    let msg = unsafe { CStr::from_ptr(ffi::b200_last_error()) }.to_string_lossy().into_owned();
    Err(match rc {
        ffi::B200_ERR_UNSATISFIED => PlonkError::WrongQuotientPolyDegree(0, 0),
        _ => PlonkError::InvalidParameters(msg),  // B200_ERR_CANCELLED too: its message names the code
    })
}

/// One GPU: a prover pool (N proofs in flight, the shape of `NativeProofManager`'s rayon pool,
/// native_proof_manager.rs:187-192) plus the resident SRS.
pub struct GpuProver {
    pool: *mut ffi::b200_pool,
    srs: *mut ffi::b200_bases,
    srs_len: usize,
}
// the library serialises the calls made on one context; the pool hands every job its own context
unsafe impl Send for GpuProver {}
unsafe impl Sync for GpuProver {}

pub struct GpuProvingKey {
    raw: *mut ffi::b200_pk,
    pub num_inputs: usize,
    pub log_n: u32,
}
unsafe impl Send for GpuProvingKey {}
unsafe impl Sync for GpuProvingKey {}

impl GpuProver {
    pub fn new(device: i32, workers: u32) -> Result<Self, PlonkError> {
        let mut pool = std::ptr::null_mut();
        check(unsafe { ffi::b200_pool_create(device, workers, &mut pool) })?;
        Ok(Self { pool, srs: std::ptr::null_mut(), srs_len: 0 })
    }

    /// replaces `parse_ptau_file` + the `powers_of_g` vector (srs.rs:63-71); on-curve check = srs.rs:178-179
    pub fn load_srs(&mut self, ptau_bytes: &[u8], n_points: usize) -> Result<(), PlonkError> {
        let (mut rec, mut n) = (std::ptr::null(), 0usize);
        check(unsafe { ffi::b200_srs_parse_ptau(ptau_bytes.as_ptr(), ptau_bytes.len(), &mut rec, &mut n) })?;
        if n < n_points {
            return Err(PlonkError::InvalidParameters(format!("ptau holds {n} G1 powers, need {n_points}")));
        }
        let ctx = unsafe { ffi::b200_pool_ctx(self.pool, 0) };
        let mut b = std::ptr::null_mut();
        check(unsafe { ffi::b200_bases_load(ctx, rec, n_points, 0, 1, &mut b) })?;
        self.srs = b;
        self.srs_len = n_points;
        Ok(())
    }

    /// replaces `PlonkKzgSnark::preprocess(&SYSTEM_SRS, &cs)` (traits.rs:850); `cs` is finalized
    pub fn preprocess(&self, cs: &PlonkCircuit<Fr>) -> Result<GpuProvingKey, PlonkError> {
        let n = cs.eval_domain_size()?;
        let selectors: Vec<u64> = cs.selector_evals().iter().flat_map(|col| col.iter().flat_map(fr_limbs)).collect(); // 13 x n
        let perm: Vec<u64> = cs.wire_permutation_flat(); // perm[i * n + j] = i' * n + j'
        let k: Vec<u64> = cs.coset_representatives().iter().flat_map(fr_limbs).collect();
        let ctx = unsafe { ffi::b200_pool_ctx(self.pool, 0) };
        let mut pk = std::ptr::null_mut();
        check(unsafe {
            ffi::b200_plonk_preprocess(ctx, self.srs, n.trailing_zeros(), cs.num_inputs(), selectors.as_ptr(), perm.as_ptr(),
                                       k.as_ptr(), &mut pk)
        })?;
        Ok(GpuProvingKey { raw: pk, num_inputs: cs.num_inputs(), log_n: n.trailing_zeros() })
    }

    /// replaces `PlonkKzgSnark::prove_with_link_hint::<_, _, SolidityTranscript>(rng, &circuit, &pk)` (traits.rs:996).
    /// Blocks the calling rayon worker only: the job runs on one of the pool's contexts, other proofs keep the GPU busy.
    pub fn prove_with_link_hint<R: rand::RngCore + rand::CryptoRng>(
        &self, rng: &mut R, cs: &PlonkCircuit<Fr>, pk: &GpuProvingKey,
    ) -> Result<(Proof<Bn254>, LinkingHint<Bn254>), PlonkError> {
        let n = 1usize << pk.log_n;
        let wires: Vec<u64> = cs.witness_table().iter().flat_map(|col| col.iter().flat_map(fr_limbs)).collect(); // 5 x n
        let pub_inputs: Vec<u64> = cs.public_input()?.iter().flat_map(fr_limbs).collect();
        // the 17 draws of the reference prover, in its order: 2 per wire polynomial, 3 for z, 4 for the quotient split
        let blinders: Vec<u64> = (0..17).map(|_| Fr::rand(rng)).flat_map(|f| fr_limbs(&f)).collect();
        let mut raw: ffi::b200_proof = unsafe { std::mem::zeroed() };
        let mut link = vec![0u64; (n + 2) * 4];
        let mut ticket = 0u64;
        check(unsafe {
            ffi::b200_pool_submit_prove(self.pool, pk.raw, wires.as_ptr(), pub_inputs.as_ptr(), pk.num_inputs, blinders.as_ptr(),
                                        &mut raw, link.as_mut_ptr(), &mut ticket)
        })?;
        check(unsafe { ffi::b200_pool_wait(self.pool, ticket) })?; // buffers above stay alive until here
        Ok((proof_from_raw(&raw), hint_from_raw(&raw, &link)))
    }

    /// `preprocess` from the circuit's wiring: the device derives the copy permutation from `cs.wire_variables()` (5 x n
    /// variable indices) and the key keeps them, so that its proofs are made by `prove_from_witness`.  Same verifying key
    /// as a key preprocessed from the permutation whose cycles run through each variable's positions in ascending order.
    pub fn preprocess_wiring(&self, cs: &PlonkCircuit<Fr>) -> Result<GpuProvingKey, PlonkError> {
        let n = cs.eval_domain_size()?;
        let selectors: Vec<u64> = cs.selector_evals().iter().flat_map(|col| col.iter().flat_map(fr_limbs)).collect(); // 13 x n
        let wire_vars: Vec<c_uint> = cs.wire_variables().iter().flat_map(|col| col.iter().map(|v| *v as c_uint)).collect(); // 5 x n
        let k: Vec<u64> = cs.coset_representatives().iter().flat_map(fr_limbs).collect();
        let ctx = unsafe { ffi::b200_pool_ctx(self.pool, 0) };
        let mut pk = std::ptr::null_mut();
        check(unsafe {
            ffi::b200_plonk_preprocess_wiring(ctx, self.srs, n.trailing_zeros(), cs.num_inputs(), selectors.as_ptr(),
                                              wire_vars.as_ptr(), cs.num_vars(), k.as_ptr(), &mut pk)
        })?;
        Ok(GpuProvingKey { raw: pk, num_inputs: cs.num_inputs(), log_n: n.trailing_zeros() })
    }

    /// `preprocess_wiring` making a compact key (b200compact.h): no coset tables in the key, round 3 one coset at a
    /// time, so that 2^23 domains fit one 80 GB GPU.  Same verifying key, same proofs; every prove method takes it.
    /// `b200_plonk_footprint` gives the device bytes of either kind before anything is allocated.
    pub fn preprocess_wiring_compact(&self, cs: &PlonkCircuit<Fr>) -> Result<GpuProvingKey, PlonkError> {
        let n = cs.eval_domain_size()?;
        let selectors: Vec<u64> = cs.selector_evals().iter().flat_map(|col| col.iter().flat_map(fr_limbs)).collect(); // 13 x n
        let wire_vars: Vec<c_uint> = cs.wire_variables().iter().flat_map(|col| col.iter().map(|v| *v as c_uint)).collect(); // 5 x n
        let k: Vec<u64> = cs.coset_representatives().iter().flat_map(fr_limbs).collect();
        let ctx = unsafe { ffi::b200_pool_ctx(self.pool, 0) };
        let mut pk = std::ptr::null_mut();
        check(unsafe {
            ffi_compact::b200_plonk_preprocess_wiring_compact(ctx, self.srs, n.trailing_zeros(), cs.num_inputs(),
                                                              selectors.as_ptr(), wire_vars.as_ptr(), cs.num_vars(), k.as_ptr(),
                                                              &mut pk)
        })?;
        Ok(GpuProvingKey { raw: pk, num_inputs: cs.num_inputs(), log_n: n.trailing_zeros() })
    }

    /// `prove_with_link_hint` for a key made by `preprocess_wiring`: the witness vector (`cs.witness()`, num_vars
    /// elements) is all that crosses the boundary; the 5 x n value table is gathered on the device.
    pub fn prove_from_witness<R: rand::RngCore + rand::CryptoRng>(
        &self, rng: &mut R, cs: &PlonkCircuit<Fr>, pk: &GpuProvingKey,
    ) -> Result<(Proof<Bn254>, LinkingHint<Bn254>), PlonkError> {
        let n = 1usize << pk.log_n;
        let witness: Vec<u64> = cs.witness().iter().flat_map(fr_limbs).collect(); // num_vars
        if witness.len() != 4 * unsafe { ffi::b200_pk_num_vars(pk.raw) } {
            return Err(PlonkError::InvalidParameters("witness length differs from the key's num_vars".into()));
        }
        let blinders: Vec<u64> = (0..17).map(|_| Fr::rand(rng)).flat_map(|f| fr_limbs(&f)).collect();
        let mut raw: ffi::b200_proof = unsafe { std::mem::zeroed() };
        let mut link = vec![0u64; (n + 2) * 4];
        let mut ticket = 0u64;
        check(unsafe {
            ffi::b200_pool_submit_prove_witness(self.pool, pk.raw, witness.as_ptr(), blinders.as_ptr(), &mut raw,
                                                link.as_mut_ptr(), std::ptr::null_mut(), &mut ticket)
        })?;
        check(unsafe { ffi::b200_pool_wait(self.pool, ticket) })?; // buffers above stay alive until here
        Ok((proof_from_raw(&raw), hint_from_raw(&raw, &link)))
    }

    /// `prove_with_link_hint` for many circuits (witnesses) of ONE key, proved by one `b200_plonk_prove_batch` job on one
    /// worker: every kernel launch covers all of them and each commitment round is one batched MSM.  Item i of the result
    /// is `prove_with_link_hint`'s answer for `circuits[i]` with the same blinders: the proof and hint, or
    /// `WrongQuotientPolyDegree` for a witness that does not satisfy the circuit.
    pub fn prove_batch<R: rand::RngCore + rand::CryptoRng>(
        &self, rng: &mut R, circuits: &[&PlonkCircuit<Fr>], pk: &GpuProvingKey,
    ) -> Result<Vec<Result<(Proof<Bn254>, LinkingHint<Bn254>), PlonkError>>, PlonkError> {
        let n = 1usize << pk.log_n;
        let k = circuits.len();
        let mut wires = Vec::with_capacity(k);
        let mut pub_inputs = Vec::with_capacity(k);
        for cs in circuits {
            wires.push(cs.witness_table().iter().flat_map(|col| col.iter().flat_map(fr_limbs)).collect::<Vec<u64>>());
            pub_inputs.push(cs.public_input()?.iter().flat_map(fr_limbs).collect::<Vec<u64>>());
        }
        let blinders: Vec<Vec<u64>> = (0..k).map(|_| (0..17).map(|_| Fr::rand(rng)).flat_map(|f| fr_limbs(&f)).collect()).collect();
        let mut raws: Vec<ffi::b200_proof> = (0..k).map(|_| unsafe { std::mem::zeroed() }).collect();
        let mut links: Vec<Vec<u64>> = (0..k).map(|_| vec![0u64; (n + 2) * 4]).collect();
        let items: Vec<ffi::b200_prove_item> = (0..k).map(|i| ffi::b200_prove_item {
            wires: wires[i].as_ptr(), pub_inputs: pub_inputs[i].as_ptr(), blinders: blinders[i].as_ptr(),
            proof: &mut raws[i], link_poly: links[i].as_mut_ptr(), challenges: std::ptr::null_mut(),
        }).collect();
        let mut statuses: Vec<c_int> = vec![0; k];
        let mut ticket = 0u64;
        check(unsafe {
            ffi::b200_pool_submit_prove_batch(self.pool, pk.raw, items.as_ptr(), k, statuses.as_mut_ptr(), &mut ticket)
        })?;
        let rc = unsafe { ffi::b200_pool_wait(self.pool, ticket) }; // buffers above stay alive until here
        if rc != ffi::B200_ERR_UNSATISFIED {
            check(rc)?;
        }
        Ok((0..k).map(|i| {
            check(statuses[i])?;
            Ok((proof_from_raw(&raws[i]), hint_from_raw(&raws[i], &links[i])))
        }).collect())
    }

    /// `prove_batch` for a key made by `preprocess_wiring`: one `b200_plonk_prove_witness_batch` job on one worker, each
    /// circuit handing over only its witness vector (`cs.witness()`).  Item i of the result is `prove_from_witness`'s
    /// answer for `circuits[i]` with the same blinders, or `WrongQuotientPolyDegree` for an unsatisfied witness.
    pub fn prove_from_witness_batch<R: rand::RngCore + rand::CryptoRng>(
        &self, rng: &mut R, circuits: &[&PlonkCircuit<Fr>], pk: &GpuProvingKey,
    ) -> Result<Vec<Result<(Proof<Bn254>, LinkingHint<Bn254>), PlonkError>>, PlonkError> {
        let n = 1usize << pk.log_n;
        let k = circuits.len();
        let num_vars = unsafe { ffi::b200_pk_num_vars(pk.raw) };
        let witnesses: Vec<Vec<u64>> = circuits.iter().map(|cs| cs.witness().iter().flat_map(fr_limbs).collect()).collect();
        if witnesses.iter().any(|w| w.len() != 4 * num_vars) {
            return Err(PlonkError::InvalidParameters("witness length differs from the key's num_vars".into()));
        }
        let blinders: Vec<Vec<u64>> = (0..k).map(|_| (0..17).map(|_| Fr::rand(rng)).flat_map(|f| fr_limbs(&f)).collect()).collect();
        let mut raws: Vec<ffi::b200_proof> = (0..k).map(|_| unsafe { std::mem::zeroed() }).collect();
        let mut links: Vec<Vec<u64>> = (0..k).map(|_| vec![0u64; (n + 2) * 4]).collect();
        let items: Vec<ffi::b200_witness_item> = (0..k).map(|i| ffi::b200_witness_item {
            witness: witnesses[i].as_ptr(), blinders: blinders[i].as_ptr(), proof: &mut raws[i],
            link_poly: links[i].as_mut_ptr(), challenges: std::ptr::null_mut(), pub_inputs_out: std::ptr::null_mut(),
        }).collect();
        let mut statuses: Vec<c_int> = vec![0; k];
        let mut ticket = 0u64;
        check(unsafe {
            ffi::b200_pool_submit_prove_witness_batch(self.pool, pk.raw, items.as_ptr(), k, statuses.as_mut_ptr(), &mut ticket)
        })?;
        let rc = unsafe { ffi::b200_pool_wait(self.pool, ticket) }; // buffers above stay alive until here
        if rc != ffi::B200_ERR_UNSATISFIED {
            check(rc)?;
        }
        Ok((0..k).map(|i| {
            check(statuses[i])?;
            Ok((proof_from_raw(&raws[i]), hint_from_raw(&raws[i], &links[i])))
        }).collect())
    }

    /// replaces `PlonkKzgSnark::link_proofs::<SolidityTranscript>(lhs, rhs, &layout, &pk.commit_key)`
    /// (proof_linking/intent_only.rs:42-47, intent_and_balance.rs:66-72, output_balance.rs)
    pub fn link_proofs(&self, lhs: &LinkingHint<Bn254>, rhs: &LinkingHint<Bn254>, layout: &GroupLayout)
        -> Result<mpc_plonk::proof_system::structs::LinkingProof<Bn254>, PlonkError> {
        let a1: Vec<u64> = lhs.linking_wire_poly.coeffs.iter().flat_map(fr_limbs).collect();
        let a2: Vec<u64> = rhs.linking_wire_poly.coeffs.iter().flat_map(fr_limbs).collect();
        let (c1, c2) = (g1_record(&lhs.linking_wire_comm.0), g1_record(&rhs.linking_wire_comm.0));
        let mut raw: ffi::b200_link_proof = unsafe { std::mem::zeroed() };
        let mut ticket = 0u64;
        check(unsafe {
            ffi::b200_pool_submit_link(self.pool, self.srs, a1.as_ptr(), a1.len() / 4, a2.as_ptr(), a2.len() / 4, c1.as_ptr(),
                                       c2.as_ptr(), layout.alignment as u32, layout.offset, layout.size, &mut raw, &mut ticket)
        })?;
        check(unsafe { ffi::b200_pool_wait(self.pool, ticket) })?;
        Ok(mpc_plonk::proof_system::structs::LinkingProof {
            quotient_commitment: jf_primitives::pcs::prelude::Commitment(g1_from(&raw.quotient_commitment)),
            opening_proof: jf_primitives::pcs::prelude::UnivariateKzgProof { proof: g1_from(&raw.opening_proof) },
        })
    }

    /// `link_proofs` for many (lhs, rhs, layout) triples, made by one `b200_plonk_link_batch` job on one worker: the
    /// division runs as one launch per step over the items of one transform size, and the quotient and opening
    /// commitments are one batched MSM each.  Item i of the result is `link_proofs`' answer for `links[i]`: the proof, or
    /// `WrongQuotientPolyDegree` when the two polynomials differ on the group.  E.g. the four link proofs of a private
    /// match (`compute_private_settlement_link_proofs`, native_proof_manager.rs:726-782) in one call.
    #[allow(clippy::type_complexity)]
    pub fn link_proofs_batch(&self, links: &[(&LinkingHint<Bn254>, &LinkingHint<Bn254>, &GroupLayout)])
        -> Vec<Result<mpc_plonk::proof_system::structs::LinkingProof<Bn254>, PlonkError>> {
        let k = links.len();
        let polys: Vec<(Vec<u64>, Vec<u64>)> = links.iter().map(|(l, r, _)| (
            l.linking_wire_poly.coeffs.iter().flat_map(fr_limbs).collect(),
            r.linking_wire_poly.coeffs.iter().flat_map(fr_limbs).collect())).collect();
        let comms: Vec<([u64; 8], [u64; 8])> =
            links.iter().map(|(l, r, _)| (g1_record(&l.linking_wire_comm.0), g1_record(&r.linking_wire_comm.0))).collect();
        let mut raws: Vec<ffi::b200_link_proof> = (0..k).map(|_| unsafe { std::mem::zeroed() }).collect();
        let items: Vec<ffi::b200_link_item> = (0..k).map(|i| ffi::b200_link_item {
            a1: polys[i].0.as_ptr(), len1: polys[i].0.len() / 4, a2: polys[i].1.as_ptr(), len2: polys[i].1.len() / 4,
            comm1: comms[i].0.as_ptr(), comm2: comms[i].1.as_ptr(), alignment: links[i].2.alignment as c_uint,
            offset: links[i].2.offset, size: links[i].2.size, proof: &mut raws[i], eta: std::ptr::null_mut(),
        }).collect();
        let mut statuses: Vec<c_int> = vec![0; k];
        let mut ticket = 0u64;
        let submitted = check(unsafe {
            ffi::b200_pool_submit_link_batch(self.pool, self.srs, items.as_ptr(), k, statuses.as_mut_ptr(), &mut ticket)
        });
        let rc = match submitted {
            Ok(()) => unsafe { ffi::b200_pool_wait(self.pool, ticket) }, // buffers above stay alive until here
            Err(e) => return (0..k).map(|_| Err(PlonkError::InvalidParameters(format!("{e:?}")))).collect(),
        };
        if rc != ffi::B200_OK && rc != ffi::B200_ERR_UNSATISFIED {
            let err = check(rc).unwrap_err();
            return (0..k).map(|_| Err(PlonkError::InvalidParameters(format!("{err:?}")))).collect();
        }
        (0..k).map(|i| {
            check(statuses[i])?;
            Ok(mpc_plonk::proof_system::structs::LinkingProof {
                quotient_commitment: jf_primitives::pcs::prelude::Commitment(g1_from(&raws[i].quotient_commitment)),
                opening_proof: jf_primitives::pcs::prelude::UnivariateKzgProof { proof: g1_from(&raws[i].opening_proof) },
            })
        }).collect()
    }

    /// A settlement arm of `NativeProofManager::handle_proof_job` (native_proof_manager.rs:514-660) as ONE pool job
    /// (`b200_pool_submit_settlement`): `singleprover_prove_with_hint` of the settlement statement, then `link_proofs(hint,
    /// &settlement_hint, layout)` for every stored hint the job brings (validity hint first, intent_and_balance.rs:57-72),
    /// as one link batch that reads the settlement hint from device memory.  The proof and link proofs equal
    /// `prove_with_link_hint` + `link_proofs` with the same rng draws.  A stale hint (one that differs from the
    /// settlement on its group) or an unsatisfied witness is `WrongQuotientPolyDegree`; `b200_last_error` names the link.
    pub fn prove_settlement<R: rand::RngCore + rand::CryptoRng>(
        &self, rng: &mut R, cs: &PlonkCircuit<Fr>, pk: &GpuProvingKey, hints: &[(&LinkingHint<Bn254>, &GroupLayout)],
    ) -> Result<(Proof<Bn254>, Vec<mpc_plonk::proof_system::structs::LinkingProof<Bn254>>), PlonkError> {
        let wires: Vec<u64> = cs.witness_table().iter().flat_map(|col| col.iter().flat_map(fr_limbs)).collect(); // 5 x n
        let pub_inputs: Vec<u64> = cs.public_input()?.iter().flat_map(fr_limbs).collect();
        let blinders: Vec<u64> = (0..17).map(|_| Fr::rand(rng)).flat_map(|f| fr_limbs(&f)).collect();
        self.settle(hints, |raw, links, statuses, ticket| unsafe {
            let proof = ffi::b200_bundle_proof { pk: pk.raw, wires: wires.as_ptr(), pub_inputs: pub_inputs.as_ptr(),
                                                 num_inputs: pk.num_inputs, blinders: blinders.as_ptr(), proof: raw,
                                                 link_poly: std::ptr::null_mut() };
            ffi_settlement::b200_pool_submit_settlement(self.pool, self.srs, &proof, links.as_ptr(), links.len(), statuses, ticket)
        })
    }

    /// `prove_settlement` for a key made by `preprocess_wiring`: only the witness vector crosses the boundary
    /// (`b200_pool_submit_settlement_witness`).
    pub fn prove_settlement_from_witness<R: rand::RngCore + rand::CryptoRng>(
        &self, rng: &mut R, cs: &PlonkCircuit<Fr>, pk: &GpuProvingKey, hints: &[(&LinkingHint<Bn254>, &GroupLayout)],
    ) -> Result<(Proof<Bn254>, Vec<mpc_plonk::proof_system::structs::LinkingProof<Bn254>>), PlonkError> {
        let witness: Vec<u64> = cs.witness().iter().flat_map(fr_limbs).collect(); // num_vars
        if witness.len() != 4 * unsafe { ffi::b200_pk_num_vars(pk.raw) } {
            return Err(PlonkError::InvalidParameters("witness length differs from the key's num_vars".into()));
        }
        let blinders: Vec<u64> = (0..17).map(|_| Fr::rand(rng)).flat_map(|f| fr_limbs(&f)).collect();
        self.settle(hints, |raw, links, statuses, ticket| unsafe {
            let proof = ffi::b200_bundle_witness { pk: pk.raw, witness: witness.as_ptr(), blinders: blinders.as_ptr(), proof: raw,
                                                   link_poly: std::ptr::null_mut(), pub_inputs_out: std::ptr::null_mut() };
            ffi_settlement::b200_pool_submit_settlement_witness(self.pool, self.srs, &proof, links.as_ptr(), links.len(), statuses, ticket)
        })
    }

    /// The part both settlement wrappers share: the link array, the submission (`submit`), the wait and the results.
    #[allow(clippy::type_complexity)]
    fn settle(&self, hints: &[(&LinkingHint<Bn254>, &GroupLayout)],
              submit: impl FnOnce(*mut ffi::b200_proof, &[ffi_settlement::b200_settlement_link], *mut c_int, *mut u64) -> c_int)
        -> Result<(Proof<Bn254>, Vec<mpc_plonk::proof_system::structs::LinkingProof<Bn254>>), PlonkError> {
        let k = hints.len();
        let polys: Vec<Vec<u64>> = hints.iter().map(|(h, _)| h.linking_wire_poly.coeffs.iter().flat_map(fr_limbs).collect()).collect();
        let comms: Vec<[u64; 8]> = hints.iter().map(|(h, _)| g1_record(&h.linking_wire_comm.0)).collect();
        let mut raws: Vec<ffi::b200_link_proof> = (0..k).map(|_| unsafe { std::mem::zeroed() }).collect();
        let links: Vec<ffi_settlement::b200_settlement_link> = (0..k).map(|i| ffi_settlement::b200_settlement_link {
            hint_poly: polys[i].as_ptr(), hint_len: polys[i].len() / 4, hint_comm: comms[i].as_ptr(),
            alignment: hints[i].1.alignment as c_uint, offset: hints[i].1.offset, size: hints[i].1.size, proof: &mut raws[i],
            eta: std::ptr::null_mut(),
        }).collect();
        let mut raw: ffi::b200_proof = unsafe { std::mem::zeroed() };
        let mut statuses: Vec<c_int> = vec![0; k + 1];
        let mut ticket = 0u64;
        check(submit(&mut raw, &links, statuses.as_mut_ptr(), &mut ticket))?;
        check(unsafe { ffi::b200_pool_wait(self.pool, ticket) })?; // buffers above stay alive until here
        let proofs = raws.iter().map(|r| mpc_plonk::proof_system::structs::LinkingProof {
            quotient_commitment: jf_primitives::pcs::prelude::Commitment(g1_from(&r.quotient_commitment)),
            opening_proof: jf_primitives::pcs::prelude::UnivariateKzgProof { proof: g1_from(&r.opening_proof) },
        }).collect();
        Ok((proof_from_raw(&raw), proofs))
    }

    /// Many `verify` / `verify_link_proof` checks with ONE pairing on this GPU (`b200_plonk_batch_verify`).
    /// `proofs[i] = (index into vks, public inputs, proof)`; `links[i] = (comm_a, comm_b, link proof, layout)`.
    /// Returns every item's verdict, proofs first, then links: exactly what the single verifiers answer.
    #[allow(clippy::type_complexity)]
    pub fn batch_verify(&self, vks: &[BatchVerifyingKey], proofs: &[(usize, &[Fr], &Proof<Bn254>)],
                        links: &[(&G1Affine, &G1Affine, &mpc_plonk::proof_system::structs::LinkingProof<Bn254>, &GroupLayout)],
                        g2_h: &[u64; 16], g2_tau_h: &[u64; 16]) -> Result<Vec<bool>, PlonkError> {
        let mut verdicts = vec![0u8; proofs.len() + links.len()];
        let mut all: c_int = 0;
        with_batch(vks, proofs, links, |c_vks, c_proofs, c_links| check(unsafe {
            ffi::b200_plonk_batch_verify(ffi::b200_pool_ctx(self.pool, 0), c_vks.as_ptr(), c_vks.len(), c_proofs.as_ptr(),
                                         c_proofs.len(), c_links.as_ptr(), c_links.len(), g2_h.as_ptr(), g2_tau_h.as_ptr(),
                                         &mut all, verdicts.as_mut_ptr())
        }))?;
        Ok(verdicts.into_iter().map(|v| v == 1).collect())
    }

    /// The same verdicts as `batch_verify`, each item checked on its own with its own pairing on this GPU
    /// (`b200_plonk_verify_each`): no bisection, so the cost does not depend on how many items fail.
    #[allow(clippy::type_complexity)]
    pub fn verify_each(&self, vks: &[BatchVerifyingKey], proofs: &[(usize, &[Fr], &Proof<Bn254>)],
                       links: &[(&G1Affine, &G1Affine, &mpc_plonk::proof_system::structs::LinkingProof<Bn254>, &GroupLayout)],
                       g2_h: &[u64; 16], g2_tau_h: &[u64; 16]) -> Result<Vec<bool>, PlonkError> {
        let mut verdicts = vec![0u8; proofs.len() + links.len()];
        with_batch(vks, proofs, links, |c_vks, c_proofs, c_links| check(unsafe {
            ffi::b200_plonk_verify_each(ffi::b200_pool_ctx(self.pool, 0), c_vks.as_ptr(), c_vks.len(), c_proofs.as_ptr(),
                                        c_proofs.len(), c_links.as_ptr(), c_links.len(), g2_h.as_ptr(), g2_tau_h.as_ptr(),
                                        verdicts.as_mut_ptr())
        }))?;
        Ok(verdicts.into_iter().map(|v| v == 1).collect())
    }

    /// `verify_each` as ONE job on this GPU's pool (`b200_pool_submit_verify`, mode 0): a worker runs it on its own
    /// context next to the proofs, so a caller that verifies while the pool proves needs no context of its own.  Every
    /// input is copied at submit; the ticket owns the verdict buffer.  `wait_verify` returns the verdicts.
    #[allow(clippy::type_complexity)]
    pub fn submit_verify(&self, vks: &[BatchVerifyingKey], proofs: &[(usize, &[Fr], &Proof<Bn254>)],
                         links: &[(&G1Affine, &G1Affine, &mpc_plonk::proof_system::structs::LinkingProof<Bn254>, &GroupLayout)],
                         g2_h: &[u64; 16], g2_tau_h: &[u64; 16]) -> Result<VerifyTicket<'_>, PlonkError> {
        self.submit_verify_mode(0, vks, proofs, links, g2_h, g2_tau_h)
    }

    /// `batch_verify` as ONE pool job (`b200_pool_submit_verify`, mode 1): one combined pairing, the failing items found
    /// by bisection inside the job.  `wait_verify` returns the verdicts and whether every item was accepted.
    #[allow(clippy::type_complexity)]
    pub fn submit_verify_combined(&self, vks: &[BatchVerifyingKey], proofs: &[(usize, &[Fr], &Proof<Bn254>)],
                                  links: &[(&G1Affine, &G1Affine, &mpc_plonk::proof_system::structs::LinkingProof<Bn254>, &GroupLayout)],
                                  g2_h: &[u64; 16], g2_tau_h: &[u64; 16]) -> Result<VerifyTicket<'_>, PlonkError> {
        self.submit_verify_mode(1, vks, proofs, links, g2_h, g2_tau_h)
    }

    #[allow(clippy::type_complexity)]
    fn submit_verify_mode(&self, mode: c_int, vks: &[BatchVerifyingKey], proofs: &[(usize, &[Fr], &Proof<Bn254>)],
                          links: &[(&G1Affine, &G1Affine, &mpc_plonk::proof_system::structs::LinkingProof<Bn254>, &GroupLayout)],
                          g2_h: &[u64; 16], g2_tau_h: &[u64; 16]) -> Result<VerifyTicket<'_>, PlonkError> {
        let mut t = VerifyTicket { pool: self.pool, ticket: 0, waited: true, combined: mode == 1, all: Box::new(0),
                                   verdicts: vec![0u8; proofs.len() + links.len()].into_boxed_slice(),
                                   _prover: std::marker::PhantomData };
        let (all, verdicts): (*mut c_int, *mut u8) = (&mut *t.all, t.verdicts.as_mut_ptr());
        with_batch(vks, proofs, links, |c_vks, c_proofs, c_links| check(unsafe {
            ffi_verifyjobs::b200_pool_submit_verify(self.pool, mode, c_vks.as_ptr(), c_vks.len(), c_proofs.as_ptr(),
                                                    c_proofs.len(), c_links.as_ptr(), c_links.len(), g2_h.as_ptr(),
                                                    g2_tau_h.as_ptr(), all, verdicts, &mut t.ticket)
        }))?;
        t.waited = false;
        Ok(t)
    }

    /// Waits for a verification job: (every item accepted, verdicts proofs first, then links).  The first value is
    /// the combined check's answer for `submit_verify_combined`, and whether every verdict is true for `submit_verify`.
    pub fn wait_verify(&self, mut t: VerifyTicket<'_>) -> Result<(bool, Vec<bool>), PlonkError> {
        t.waited = true;
        check(unsafe { ffi::b200_pool_wait(self.pool, t.ticket) })?;
        let verdicts: Vec<bool> = t.verdicts.iter().map(|v| *v == 1).collect();
        let all = if t.combined { *t.all == 1 } else { verdicts.iter().all(|v| *v) };
        Ok((all, verdicts))
    }

    /// Checks the first `n` powers of the loaded SRS against `(g2_h, g2_tau_h)` on this GPU (`b200_srs_check`): one
    /// batch-2 MSM and one pairing, with weights drawn from `seed`, which must be unknown to whoever made the file.
    /// With `locate`, a failed check also names the failing pairs (P_i, P_{i+1}).  Valid exactly when
    /// `consistent && g1_generator && g2_subgroup`.
    pub fn check_srs(&self, n: usize, g2_h: &[u64; 16], g2_tau_h: &[u64; 16], seed: &[u8; 32], locate: bool)
        -> Result<ffi::b200_srs_report, PlonkError> {
        if self.srs.is_null() {
            return Err(PlonkError::InvalidParameters("check_srs: no SRS loaded".into()));
        }
        let mut report: ffi::b200_srs_report = unsafe { std::mem::zeroed() };
        check(unsafe {
            ffi::b200_srs_check(ffi::b200_pool_ctx(self.pool, 0), self.srs, n, g2_h.as_ptr(), g2_tau_h.as_ptr(), seed.as_ptr(),
                                locate as c_int, &mut report)
        })?;
        Ok(report)
    }

    /// Cancels a pool job by ticket (`b200_pool_cancel`): its queued jobs are dropped and never run, a running one stops
    /// at its next abort point (a host round trip; no kernel is interrupted).  Returns how many queued jobs were dropped.
    /// Its wait then fails with `B200_ERR_CANCELLED` (or returns its real status if it finished first); the job's outputs
    /// must not be read.  A finished or already cancelled ticket is `Ok(0)`.
    pub fn cancel(&self, ticket: u64) -> Result<usize, PlonkError> {
        let mut dropped = 0usize;
        check(unsafe { ffi_cancel::b200_pool_cancel(self.pool, ticket, &mut dropped) })?;
        Ok(dropped)
    }

    /// `cancel` for every job the pool holds (`b200_pool_cancel_all`).  Jobs submitted afterwards run as usual.
    pub fn cancel_all(&self) -> Result<usize, PlonkError> {
        let mut dropped = 0usize;
        check(unsafe { ffi_cancel::b200_pool_cancel_all(self.pool, &mut dropped) })?;
        Ok(dropped)
    }

    /// Stops now: cancels every job, then destroys the pool (dropping `self`), which waits at most for each worker's
    /// next abort point instead of draining the queue.  The shape of the reference's cancel channel
    /// (native_proof_manager.rs:167-178): on the signal the coordinator returns `ProofManagerError::Cancelled`; the
    /// threads still blocked in a wait see `B200_ERR_CANCELLED` once `cancel_all` runs, so their tickets are gone
    /// before this is called:
    ///
    /// ```ignore
    /// if cancel_channel.has_changed()? {
    ///     prover.cancel_all()?;                 // every waiting job thread returns its error now
    ///     pool_threads.join();                  // the borrows of `prover` end
    ///     Arc::try_unwrap(prover).ok().unwrap().shutdown_now()?;
    ///     return Err(ProofManagerError::Cancelled("received cancel signal".to_string()));
    /// }
    /// ```
    pub fn shutdown_now(self) -> Result<(), PlonkError> {
        let r = self.cancel_all().map(|_| ());
        drop(self);  // b200_pool_destroy: nothing is left queued
        r
    }
}

/// replaces `read_ptau_section3` (srs.rs:147-157): `(h, beta_h)`, the two G2 records of the ptau's section 3 in the
/// layout `verify` takes; both are checked to lie on the twist.  Host only.
pub fn parse_ptau_g2(ptau_bytes: &[u8]) -> Result<([u64; 16], [u64; 16]), PlonkError> {
    let (mut h, mut beta_h) = ([0u64; 16], [0u64; 16]);
    check(unsafe { ffi::b200_srs_parse_ptau_g2(ptau_bytes.as_ptr(), ptau_bytes.len(), h.as_mut_ptr(), beta_h.as_mut_ptr()) })?;
    Ok((h, beta_h))
}

/// The C structs of a batch of `verify` / `verify_link_proof` items, alive while `f` runs.
#[allow(clippy::type_complexity)]
fn with_batch<R>(vks: &[BatchVerifyingKey], proofs: &[(usize, &[Fr], &Proof<Bn254>)],
                 links: &[(&G1Affine, &G1Affine, &mpc_plonk::proof_system::structs::LinkingProof<Bn254>, &GroupLayout)],
                 f: impl FnOnce(&[ffi::b200_verifying_key], &[ffi::b200_batch_proof], &[ffi::b200_batch_link]) -> R) -> R {
    let flat: Vec<(Vec<u64>, Vec<u64>, Vec<u64>)> = vks.iter().map(|v| (
        v.k.iter().flat_map(fr_limbs).collect(),
        v.selector_comms.iter().flat_map(g1_record).collect(),
        v.sigma_comms.iter().flat_map(g1_record).collect())).collect();
    let c_vks: Vec<ffi::b200_verifying_key> = vks.iter().zip(&flat).map(|(v, (k, sel, sig))| ffi::b200_verifying_key {
        log_n: v.log_n, num_inputs: v.num_inputs, k: k.as_ptr(), selector_comms: sel.as_ptr(), sigma_comms: sig.as_ptr(),
    }).collect();
    let pis: Vec<Vec<u64>> = proofs.iter().map(|(_, pi, _)| pi.iter().flat_map(fr_limbs).collect()).collect();
    let raws: Vec<ffi::b200_proof> = proofs.iter().map(|(_, _, p)| proof_to_raw(p)).collect();
    let c_proofs: Vec<ffi::b200_batch_proof> = proofs.iter().zip(pis.iter().zip(&raws)).map(|((vk, _, _), (pi, raw))| {
        ffi::b200_batch_proof { vk: *vk as c_uint, pub_inputs: pi.as_ptr(), proof: raw }
    }).collect();
    let lflat: Vec<([u64; 8], [u64; 8], ffi::b200_link_proof)> = links.iter().map(|(a, b, lp, _)| (g1_record(a), g1_record(b),
        ffi::b200_link_proof { quotient_commitment: g1_record(&lp.quotient_commitment.0), opening_proof: g1_record(&lp.opening_proof.proof) })).collect();
    let c_links: Vec<ffi::b200_batch_link> = links.iter().zip(&lflat).map(|((_, _, _, lay), (a, b, lp))| ffi::b200_batch_link {
        comm1: a.as_ptr(), comm2: b.as_ptr(), alignment: lay.alignment as c_uint, offset: lay.offset, size: lay.size, proof: lp,
    }).collect();
    f(&c_vks, &c_proofs, &c_links)
}

/// A queued verification job: it owns the buffers the worker writes (the verdicts, the combined answer), so it waits
/// for its job when dropped unwaited; it cannot outlive the `GpuProver` whose pool runs the job.
pub struct VerifyTicket<'a> {
    pool: *mut ffi::b200_pool,
    ticket: u64,
    waited: bool,
    combined: bool,
    all: Box<c_int>,
    verdicts: Box<[u8]>,
    _prover: std::marker::PhantomData<&'a GpuProver>,
}
unsafe impl Send for VerifyTicket<'_> {}

impl VerifyTicket<'_> {
    /// The pool ticket, for [`GpuProver::cancel`].
    pub fn id(&self) -> u64 {
        self.ticket
    }
}

impl Drop for VerifyTicket<'_> {
    fn drop(&mut self) {
        if !self.waited {
            unsafe { ffi::b200_pool_wait(self.pool, self.ticket) };
        }
    }
}

/// The flat verifying key of one circuit, as `verify` takes it.
pub struct BatchVerifyingKey<'a> {
    pub log_n: u32,
    pub num_inputs: usize,
    pub k: &'a [Fr; 5],
    pub selector_comms: &'a [G1Affine; 13],
    pub sigma_comms: &'a [G1Affine; 5],
}

impl Drop for GpuProver {
    fn drop(&mut self) {
        unsafe {
            if !self.srs.is_null() {
                ffi::b200_bases_free(ffi::b200_pool_ctx(self.pool, 0), self.srs);
            }
            ffi::b200_pool_destroy(self.pool);
        }
    }
}

/// replaces `PlonkKzgSnark::verify::<SolidityTranscript>(&vk, public_inputs, &proof, None)` (traits.rs:1012-1018).
/// Host only: `g2_h` / `g2_tau_h` are the ptau G2 records of `open_key.h` / `open_key.beta_h` (srs.rs:185-199).
#[allow(clippy::too_many_arguments)]
pub fn verify(log_n: u32, k: &[Fr; 5], selector_comms: &[G1Affine; 13], sigma_comms: &[G1Affine; 5], public_inputs: &[Fr],
              proof: &Proof<Bn254>, g2_h: &[u64; 16], g2_tau_h: &[u64; 16]) -> Result<(), PlonkError> {
    let kk: Vec<u64> = k.iter().flat_map(fr_limbs).collect();
    let sel: Vec<u64> = selector_comms.iter().flat_map(g1_record).collect();
    let sig: Vec<u64> = sigma_comms.iter().flat_map(g1_record).collect();
    let pi: Vec<u64> = public_inputs.iter().flat_map(fr_limbs).collect();
    let raw = proof_to_raw(proof);
    let mut accepted: c_int = 0;
    check(unsafe {
        ffi::b200_plonk_verify(log_n, public_inputs.len(), kk.as_ptr(), sel.as_ptr(), sig.as_ptr(), pi.as_ptr(), &raw,
                               g2_h.as_ptr(), g2_tau_h.as_ptr(), &mut accepted)
    })?;
    if accepted == 1 { Ok(()) } else { Err(PlonkError::WrongProof) }
}

// ---- field-by-field copies between the flat C structs and the upstream types (plonk_proof_def.rs:168-222) -----------
fn proof_from_raw(r: &ffi::b200_proof) -> Proof<Bn254> {
    use jf_primitives::pcs::prelude::{Commitment, UnivariateKzgProof};
    Proof {
        wires_poly_comms: r.wires_poly_comms.iter().map(|c| Commitment(g1_from(c))).collect(),
        prod_perm_poly_comm: Commitment(g1_from(&r.prod_perm_poly_comm)),
        split_quot_poly_comms: r.split_quot_poly_comms.iter().map(|c| Commitment(g1_from(c))).collect(),
        opening_proof: Commitment(g1_from(&r.opening_proof)),
        shifted_opening_proof: Commitment(g1_from(&r.shifted_opening_proof)),
        poly_evals: ProofEvaluations {
            wires_evals: r.wires_evals.iter().map(fr_from).collect(),
            wire_sigma_evals: r.wire_sigma_evals.iter().map(fr_from).collect(),
            perm_next_eval: fr_from(&r.perm_next_eval),
        },
        plookup_proof: None,
    }
    .tap_kzg::<UnivariateKzgProof<Bn254>>()
}
fn proof_to_raw(p: &Proof<Bn254>) -> ffi::b200_proof {
    let mut r: ffi::b200_proof = unsafe { std::mem::zeroed() };
    for i in 0..5 {
        r.wires_poly_comms[i] = g1_record(&p.wires_poly_comms[i].0);
        r.split_quot_poly_comms[i] = g1_record(&p.split_quot_poly_comms[i].0);
        r.wires_evals[i] = fr_limbs(&p.poly_evals.wires_evals[i]);
    }
    for i in 0..4 {
        r.wire_sigma_evals[i] = fr_limbs(&p.poly_evals.wire_sigma_evals[i]);
    }
    r.prod_perm_poly_comm = g1_record(&p.prod_perm_poly_comm.0);
    r.opening_proof = g1_record(&p.opening_proof.0);
    r.shifted_opening_proof = g1_record(&p.shifted_opening_proof.0);
    r.perm_next_eval = fr_limbs(&p.poly_evals.perm_next_eval);
    r
}
fn hint_from_raw(r: &ffi::b200_proof, link: &[u64]) -> LinkingHint<Bn254> {
    use ark_poly::{univariate::DensePolynomial, DenseUVPolynomial};
    let coeffs: Vec<Fr> = link.chunks_exact(4).map(|c| fr_from(&[c[0], c[1], c[2], c[3]])).collect();
    LinkingHint {
        linking_wire_poly: DensePolynomial::from_coefficients_vec(coeffs),
        linking_wire_comm: jf_primitives::pcs::prelude::Commitment(g1_from(&r.wires_poly_comms[0])),
    }
}

/// Adapter kept next to the conversion it documents: the fork's `Proof` stores opening proofs as `Commitment`s.
trait TapKzg: Sized {
    fn tap_kzg<T>(self) -> Self {
        self
    }
}
impl TapKzg for Proof<Bn254> {}
