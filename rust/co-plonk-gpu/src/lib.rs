//! `Plonk::plain_prove`, `Rep3CoPlonk::prove` and `ShamirCoPlonk::prove` with the signatures of co-plonk
//! (co-circom/co-plonk/src/lib.rs:222-260, 271-281), executed by the library: the device-resident key is built
//! once from the snarkjs `.zkey`, a proof is one FFI call (`cs_plonk_prove_plain`) or, for an MPC party, one
//! `cs_plonk_rep3_prove` / `cs_plonk_shamir_prove` -- step sequence, Keccak transcript, openings and (Shamir) the
//! double sharings run inside libcosnarks_gpu.so over the caller's `mpc_net::Network` through the callback transport.  SOURCE ONLY: never compiled (no rustc in the build
//! image); the same entry points are exercised from C++ (`include/co_plonk.hpp`) and Python in `tests/`.
use ark_bn254::{Bn254, Fr};
use circom_types::plonk::PlonkProof;
use co_circom_types::{Rep3SharedWitness, ShamirSharedWitness, SharedWitness};
use cosnarks_gpu_sys as sys;
use mpc_net::Network;
use std::ffi::CString;
use std::os::raw::{c_int, c_void};

/// Device-resident proving key (`circom_types::plonk::Zkey` uploaded once).
pub struct GpuZkey { ctx: *mut sys::cs_ctx, pk: *mut sys::cs_plonk_pk, n_public: usize, n_witness: usize }

impl GpuZkey {
    /// `Zkey::from_reader` (co-circom.rs:1053-1060) straight into the device layout.
    pub fn from_file(device: i32, path: &str) -> eyre::Result<Self> {
        let (mut ctx, mut pk) = (std::ptr::null_mut(), std::ptr::null_mut());
        let (mut n_public, mut n_witness) = (0usize, 0usize);
        let c = CString::new(path)?;
        check(unsafe { sys::cs_ctx_create(device, std::ptr::null_mut(), &mut ctx) })?;
        check(unsafe { sys::cs_plonk_pk_from_zkey(ctx, c.as_ptr(), &mut pk, &mut n_public, &mut n_witness) })?;
        Ok(Self { ctx, pk, n_public, n_witness })
    }
    fn check_lengths(&self, n_pub: usize, n_wit: usize) -> eyre::Result<()> {
        eyre::ensure!(n_pub == self.n_public + 1 && n_wit == self.n_witness, "witness does not match the circuit");
        Ok(())
    }
}
impl Drop for GpuZkey {
    fn drop(&mut self) { unsafe { sys::cs_plonk_pk_free(self.pk); sys::cs_ctx_destroy(self.ctx) } }
}

fn check(rc: c_int) -> eyre::Result<()> { sys::check(rc).map_err(|e| eyre::eyre!(e)) }

/// `&N: Network` as a `cs_net` (the same adapter as in co-groth16-gpu).
struct NetAdapter<'a, N: Network> { _net: &'a N, h: *mut sys::cs_net }
unsafe extern "C" fn send_cb<N: Network>(u: *mut c_void, to: c_int, data: *const c_void, bytes: usize) -> c_int {
    let net = &*(u as *const N);
    if net.send(to as usize, std::slice::from_raw_parts(data as *const u8, bytes)).is_ok() { 0 } else { -1 }
}
unsafe extern "C" fn recv_cb<N: Network>(u: *mut c_void, from: c_int, data: *mut c_void, bytes: usize) -> c_int {
    let net = &*(u as *const N);
    match net.recv(from as usize) {
        Ok(v) if v.len() == bytes => { std::ptr::copy_nonoverlapping(v.as_ptr(), data as *mut u8, bytes); 0 }
        Ok(_) => -2,
        Err(_) => -1,
    }
}
impl<'a, N: Network> NetAdapter<'a, N> {
    fn new(net: &'a N) -> eyre::Result<Self> { Self::with_parties(net, 3) }
    fn with_parties(net: &'a N, parties: usize) -> eyre::Result<Self> {
        let cb = sys::cs_net_callbacks { user: net as *const N as *mut c_void, send: send_cb::<N>, recv: recv_cb::<N> };
        let mut h = std::ptr::null_mut();
        check(unsafe { sys::cs_net_from_callbacks(net.id() as c_int, parties as c_int, &cb, &mut h) })?;
        Ok(Self { _net: net, h })
    }
}
impl<N: Network> Drop for NetAdapter<'_, N> { fn drop(&mut self) { unsafe { sys::cs_net_free(self.h) } } }

/// 9 points (A B C Z T1 T2 T3 Wxi Wxiw, affine Montgomery limbs) + 6 evaluations -> `PlonkProof<Bn254>`
fn proof_from(points: &[[u64; 8]; 9], evals: &[[u64; 4]; 6]) -> PlonkProof<Bn254> {
    // limbs are arkworks' internal representation: Fq::new_unchecked(BigInt(limbs)), (0, 0) = the point at infinity
    circom_types::plonk::PlonkProof::from_montgomery_limbs(points, evals)
}

pub struct Plonk;
pub struct Rep3CoPlonk;
pub struct ShamirCoPlonk;

impl Plonk {
    /// `Plonk::plain_prove(zkey, private_witness)` (lib.rs:271-281); the eleven round-1 blinders are drawn here
    /// (Round1Challenges::random, round1.rs:82-92).
    pub fn plain_prove(zkey: &GpuZkey, witness: SharedWitness<Fr, Fr>) -> eyre::Result<PlonkProof<Bn254>> {
        zkey.check_lengths(witness.public_inputs.len(), witness.witness.len())?;
        let blinders: [Fr; 11] = core::array::from_fn(|_| ark_ff::UniformRand::rand(&mut rand::thread_rng()));
        let (mut pts, mut evs) = ([[0u64; 8]; 9], [[0u64; 4]; 6]);
        check(unsafe {
            sys::cs_plonk_prove_plain(zkey.ctx, zkey.pk, witness.public_inputs.as_ptr().cast(), witness.public_inputs.len(),
                                      witness.witness.as_ptr().cast(), witness.witness.len(), blinders.as_ptr().cast(),
                                      pts.as_mut_ptr().cast(), evs.as_mut_ptr().cast())
        })?;
        Ok(proof_from(&pts, &evs))
    }
}

impl Rep3CoPlonk {
    /// `Rep3CoPlonk::prove(net, zkey, witness)` (lib.rs:222-240) for this party.  Parties on the GPUs of one box
    /// additionally exchange the IPC handles of their session arenas / out-vectors and call
    /// `cs_plonk_rep3_connect` / `cs_plonk_rep3_connect_io`; without that every exchange goes through `net`.
    pub fn prove<N: Network>(net: &N, zkey: &GpuZkey, witness: Rep3SharedWitness<Fr>) -> eyre::Result<PlonkProof<Bn254>> {
        zkey.check_lengths(witness.public_inputs.len(), witness.witness.len())?;
        let adapter = NetAdapter::new(net)?;
        let (mut state, mut sess) = (std::ptr::null_mut(), std::ptr::null_mut());
        check(unsafe { sys::cs_rep3_state_create(adapter.h, &mut state) })?; // Rep3State::new: OS-entropy seeds over the net
        check(unsafe { sys::cs_plonk_rep3_create(zkey.ctx, zkey.pk, net.id() as c_int, &mut sess) })?;
        let (mut pts, mut evs) = ([[0u64; 8]; 9], [[0u64; 4]; 6]);
        let rc = unsafe {
            sys::cs_plonk_rep3_prove(sess, adapter.h, state, witness.public_inputs.as_ptr().cast(), witness.public_inputs.len(),
                                     witness.witness.as_ptr().cast(), witness.witness.len(), std::ptr::null(),
                                     pts.as_mut_ptr().cast(), evs.as_mut_ptr().cast())
        };
        unsafe { sys::cs_plonk_rep3_free(sess); sys::cs_rep3_state_free(state) };
        check(rc)?;
        Ok(proof_from(&pts, &evs))
    }
}

impl ShamirCoPlonk {
    /// `ShamirCoPlonk::prove(nets, num_parties, threshold, zkey, witness)` (lib.rs:237-260) for this party.  The
    /// reference's eight networks become the one `net`; instead of preprocessing `222 domain_size + 15` pairs up front,
    /// the library makes the 58 domain_size + 2 double sharings the proof consumes on the device when rounds 2 and 3
    /// start, and draws the eleven blinder shares with ShamirState::rand.
    pub fn prove<N: Network>(net: &N, num_parties: usize, threshold: usize, zkey: &GpuZkey,
                             witness: ShamirSharedWitness<Fr>) -> eyre::Result<PlonkProof<Bn254>> {
        zkey.check_lengths(witness.public_inputs.len(), witness.witness.len())?;
        let adapter = NetAdapter::with_parties(net, num_parties)?;
        let mut sess = std::ptr::null_mut();
        check(unsafe {
            sys::cs_plonk_shamir_create(zkey.ctx, zkey.pk, num_parties as c_int, threshold as c_int, net.id() as c_int, &mut sess)
        })?;
        let (mut pts, mut evs) = ([[0u64; 8]; 9], [[0u64; 4]; 6]);
        let rc = unsafe {
            sys::cs_plonk_shamir_prove(sess, adapter.h, witness.public_inputs.as_ptr().cast(), witness.public_inputs.len(),
                                       witness.witness.as_ptr().cast(), witness.witness.len(), std::ptr::null(),
                                       pts.as_mut_ptr().cast(), evs.as_mut_ptr().cast(), std::ptr::null_mut())
        };
        unsafe { sys::cs_plonk_shamir_free(sess) };
        check(rc)?;
        Ok(proof_from(&pts, &evs))
    }
}
