//! Raw declarations of the C ABI in `include/cosnarks_gpu.h`.  Field elements are `[u64; N]` Montgomery limbs
//! (byte-identical to arkworks' `Fp<MontBackend<_, N>>`), points are packed `x || y` limb arrays with the
//! all-zero encoding for infinity, Rep3 shares are `a || b`.  Every function returns 0 or a negative code;
//! `cs_last_error()` holds the message for the calling thread.
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_int, c_uint, c_void};

macro_rules! opaque { ($($n:ident),*) => { $( #[repr(C)] pub struct $n { _p: [u8; 0] } )* } }
opaque!(cs_ctx, cs_bases, cs_domain, cs_groth16_pk, cs_plonk_pk, cs_plonk_rep3, cs_plonk_shamir, cs_net, cs_rep3_state, cs_shamir_state);

pub const CS_BN254: c_int = 0;
pub const CS_BLS12_381: c_int = 1;
pub const CS_G1: c_int = 0;
pub const CS_G2: c_int = 1;
pub const CS_PLAIN: c_int = 0;
pub const CS_REP3: c_int = 1;

#[repr(C)]
pub struct cs_net_callbacks {
    pub user: *mut c_void,
    pub send: unsafe extern "C" fn(user: *mut c_void, to: c_int, data: *const c_void, bytes: usize) -> c_int,
    pub recv: unsafe extern "C" fn(user: *mut c_void, from: c_int, data: *mut c_void, bytes: usize) -> c_int,
}

#[repr(C)]
pub struct cs_rep3_prf {
    pub seed1: [u8; 32],
    pub word_pos1: u64,
    pub seed2: [u8; 32],
    pub word_pos2: u64,
    pub rounds: c_uint,
}

/// Device pointers to the polynomials of the UltraArithmeticRelation (witness columns: values or Rep3 shares).
#[repr(C)]
pub struct cs_honk_arith_polys {
    pub w_l: *const u64, pub w_r: *const u64, pub w_o: *const u64, pub w_4: *const u64,
    pub w_l_shift: *const u64, pub w_4_shift: *const u64,
    pub q_m: *const u64, pub q_l: *const u64, pub q_r: *const u64, pub q_o: *const u64, pub q_4: *const u64,
    pub q_c: *const u64, pub q_arith: *const u64,
}

#[repr(C)]
pub struct cs_groth16_key_desc {
    pub curve: c_int,
    pub num_constraints: usize,
    pub num_instance_variables: usize,
    pub num_witness_variables: usize,
    pub a_row_ptr: *const u32, pub a_col: *const u32, pub a_coeff: *const u64, pub a_nnz: usize,
    pub b_row_ptr: *const u32, pub b_col: *const u32, pub b_coeff: *const u64, pub b_nnz: usize,
    pub c_row_ptr: *const u32, pub c_col: *const u32, pub c_coeff: *const u64, pub c_nnz: usize,
    pub alpha_g1: *const u64, pub beta_g1: *const u64, pub beta_g2: *const u64,
    pub delta_g1: *const u64, pub delta_g2: *const u64,
    pub a_query: *const u64, pub a_query_len: usize,
    pub b_g1_query: *const u64, pub b_g1_query_len: usize,
    pub b_g2_query: *const u64, pub b_g2_query_len: usize,
    pub l_query: *const u64, pub l_query_len: usize,
    pub h_query: *const u64, pub h_query_len: usize,
    pub window_bits: c_int,
}

extern "C" {
    pub fn cs_last_error() -> *const c_char;
    pub fn cs_ctx_create(device: c_int, stream: *mut c_void, out: *mut *mut cs_ctx) -> c_int;
    pub fn cs_ctx_destroy(ctx: *mut cs_ctx);
    pub fn cs_os_random(out: *mut u8, bytes: usize) -> c_int;
    // --- msm / fft (seam 1)
    pub fn cs_bases_upload(ctx: *mut cs_ctx, curve: c_int, group: c_int, pts: *const u64, n: usize,
                           window_bits: c_int, out: *mut *mut cs_bases) -> c_int;
    pub fn cs_bases_free(b: *mut cs_bases);
    pub fn cs_bases_info(b: *const cs_bases, window_bits: *mut c_uint, windows: *mut c_uint, table_rows: *mut c_uint,
                         device_bytes: *mut usize) -> c_int;
    pub fn cs_ctx_set_table_budget(ctx: *mut cs_ctx, bytes: usize) -> c_int;
    pub fn cs_msm(ctx: *mut cs_ctx, b: *const cs_bases, offset: usize, scalars: *const u64, n: usize,
                  scalars_montgomery: c_int, out_affine: *mut u64, out_is_inf: *mut c_int) -> c_int;
    pub fn cs_domain_create(ctx: *mut cs_ctx, curve: c_int, log_n: c_uint, gen: *const u64,
                            out: *mut *mut cs_domain) -> c_int;
    pub fn cs_domain_free(d: *mut cs_domain);
    pub fn cs_ifft_in_to_out_host(ctx: *mut cs_ctx, d: *const cs_domain, data: *mut u64, batch: c_uint) -> c_int;
    pub fn cs_fft_out_to_in_host(ctx: *mut cs_ctx, d: *const cs_domain, data: *mut u64, batch: c_uint) -> c_int;
    // --- Groth16 (seams 2, 3)
    pub fn cs_groth16_pk_create(ctx: *mut cs_ctx, d: *const cs_groth16_key_desc, out: *mut *mut cs_groth16_pk) -> c_int;
    pub fn cs_groth16_pk_free(pk: *mut cs_groth16_pk);
    pub fn cs_groth16_domain_size(pk: *const cs_groth16_pk) -> usize;
    pub fn cs_groth16_pk_table_info(pk: *const cs_groth16_pk, table_rows: *mut c_uint, table_bytes: *mut usize) -> c_int;
    pub fn cs_groth16_witness_map(ctx: *mut cs_ctx, pk: *mut cs_groth16_pk, kind: c_int, party: c_int,
                                  public_inputs: *const u64, witness: *const u64, mask1: *const u64,
                                  mask2: *const u64, h_out: *mut u64) -> c_int;
    pub fn cs_groth16_prove_plain(ctx: *mut cs_ctx, pk: *mut cs_groth16_pk, public_inputs: *const u64,
                                  witness: *const u64, r: *const u64, s: *const u64, out_a: *mut u64,
                                  out_b: *mut u64, out_c: *mut u64) -> c_int;
    pub fn cs_groth16_prove_plain_batch(ctx: *mut cs_ctx, pk: *mut cs_groth16_pk, num_proofs: usize,
                                        public_inputs: *const u64, num_public: usize, h_witness: *const u64,
                                        d_witness: *const u64, num_witness: usize, r: *const u64, s: *const u64,
                                        out_a: *mut u64, out_b: *mut u64, out_c: *mut u64) -> c_int;
    // --- transport + Rep3 / Shamir parties inside the library
    pub fn cs_net_from_callbacks(id: c_int, n_parties: c_int, cb: *const cs_net_callbacks, out: *mut *mut cs_net) -> c_int;
    pub fn cs_net_free(net: *mut cs_net);
    pub fn cs_rep3_state_create(net: *mut cs_net, out: *mut *mut cs_rep3_state) -> c_int;
    pub fn cs_rep3_state_from_seeds(party: c_int, own: *const u8, pos_own: u64, prev: *const u8, pos_prev: u64,
                                    out: *mut *mut cs_rep3_state) -> c_int;
    pub fn cs_rep3_state_free(st: *mut cs_rep3_state);
    pub fn cs_groth16_rep3_prove(ctx: *mut cs_ctx, pk: *mut cs_groth16_pk, net0: *mut cs_net, net1: *mut cs_net,
                                 state: *mut cs_rep3_state, public_inputs: *const u64, h_witness_shares: *const u64,
                                 d_witness_shares: *const u64, out_a: *mut u64, out_b: *mut u64, out_c: *mut u64,
                                 out_rs: *mut u64) -> c_int;
    pub fn cs_groth16_shamir_prove(ctx: *mut cs_ctx, pk: *mut cs_groth16_pk, net0: *mut cs_net, net1: *mut cs_net,
                                   num_parties: c_int, threshold: c_int, public_inputs: *const u64,
                                   witness_shares: *const u64, out_a: *mut u64, out_b: *mut u64, out_c: *mut u64,
                                   out_rs: *mut u64) -> c_int;
    // --- mailbox transport in GPU memory (parties on the GPUs of one box)
    pub fn cs_net_peer_create(ctx: *mut cs_ctx, id: c_int, n_parties: c_int, out: *mut *mut cs_net) -> c_int;
    pub fn cs_net_peer_handle(net: *mut cs_net, out_handle64: *mut u8) -> c_int;
    pub fn cs_net_peer_connect(net: *mut cs_net, handles: *const u8) -> c_int;
    pub fn cs_net_send(net: *mut cs_net, to: c_int, data: *const c_void, bytes: usize) -> c_int;
    pub fn cs_net_recv(net: *mut cs_net, from: c_int, data: *mut c_void, bytes: usize) -> c_int;
    pub fn cs_net_sendrecv(net: *mut cs_net, to: c_int, sdata: *const c_void, sbytes: usize, from: c_int,
                           rdata: *mut c_void, rbytes: usize) -> c_int;
    pub fn cs_net_bytes_sent(net: *const cs_net) -> u64;
    pub fn cs_ipc_export(ctx: *mut cs_ctx, d_ptr: *const c_void, out_handle64: *mut u8) -> c_int;
    pub fn cs_ipc_open(ctx: *mut cs_ctx, handle64: *const u8, out_peer_ptr: *mut *mut c_void) -> c_int;
    pub fn cs_ipc_close(ctx: *mut cs_ctx, peer_ptr: *mut c_void) -> c_int;
    // --- file formats straight to the device layout
    pub fn cs_groth16_pk_from_zkey(ctx: *mut cs_ctx, zkey_path: *const c_char, window_bits: c_int,
                                   out: *mut *mut cs_groth16_pk, out_n_public: *mut usize) -> c_int;
    pub fn cs_plonk_pk_from_zkey(ctx: *mut cs_ctx, path: *const c_char, out: *mut *mut cs_plonk_pk,
                                 out_n_public: *mut usize, out_n_witness: *mut usize) -> c_int;
    pub fn cs_bases_from_crs_file(ctx: *mut cs_ctx, path: *const c_char, offset: usize, n: usize, window_bits: c_int,
                                  out: *mut *mut cs_bases) -> c_int;
    pub fn cs_rep3_witness_read(path: *const c_char, curve: c_int, out_public: *mut u64, public_capacity: usize,
                                out_shares: *mut u64, shares_capacity_elems: usize, out_n_public: *mut usize,
                                out_n_witness: *mut usize, out_kind: *mut c_int) -> c_int;
    // --- co-Plonk (co-plonk/src/lib.rs:222-281)
    pub fn cs_plonk_pk_free(pk: *mut cs_plonk_pk);
    pub fn cs_plonk_prove_plain(ctx: *mut cs_ctx, pk: *mut cs_plonk_pk, public_inputs: *const u64, n_public_inputs: usize,
                                witness: *const u64, n_witness: usize, blinders: *const u64, out_points: *mut u64,
                                out_evals: *mut u64) -> c_int;
    pub fn cs_plonk_rep3_create(ctx: *mut cs_ctx, pk: *mut cs_plonk_pk, party: c_int, out: *mut *mut cs_plonk_rep3) -> c_int;
    pub fn cs_plonk_rep3_free(s: *mut cs_plonk_rep3);
    pub fn cs_plonk_rep3_arena(s: *mut cs_plonk_rep3, d_arena: *mut *mut c_void, slot_bytes: *mut usize, n_slots: *mut c_uint) -> c_int;
    pub fn cs_plonk_rep3_io(s: *mut cs_plonk_rep3, d_additive_out: *mut *mut c_void, d_opened_in: *mut *mut c_void) -> c_int;
    pub fn cs_plonk_rep3_connect(s: *mut cs_plonk_rep3, d_next_arena: *mut c_void) -> c_int;
    pub fn cs_plonk_rep3_connect_io(s: *mut cs_plonk_rep3, d_prev_out: *mut c_void, d_next_out: *mut c_void) -> c_int;
    pub fn cs_plonk_rep3_prove(s: *mut cs_plonk_rep3, net: *mut cs_net, state: *mut cs_rep3_state, public_inputs: *const u64,
                               n_public_inputs: usize, witness_shares: *const u64, n_witness: usize,
                               blinder_shares: *const u64, out_points: *mut u64, out_evals: *mut u64) -> c_int;
    // --- Shamir co-Plonk: one session per party of a Shamir(n, t) sharing, the whole proof over one cs_net
    pub fn cs_plonk_shamir_create(ctx: *mut cs_ctx, pk: *mut cs_plonk_pk, num_parties: c_int, threshold: c_int, party: c_int,
                                  out: *mut *mut cs_plonk_shamir) -> c_int;
    pub fn cs_plonk_shamir_free(s: *mut cs_plonk_shamir);
    pub fn cs_plonk_shamir_prove(s: *mut cs_plonk_shamir, net: *mut cs_net, public_inputs: *const u64, n_public_inputs: usize,
                                 witness_shares: *const u64, n_witness: usize, blinder_shares: *const u64,
                                 out_points: *mut u64, out_evals: *mut u64, out_blinder_shares: *mut u64) -> c_int;
    pub fn cs_plonk_shamir_pairs(s: *const cs_plonk_shamir) -> usize;
    pub fn cs_plonk_shamir_pair_ms(s: *const cs_plonk_shamir) -> f64;
    pub fn cs_plonk_shamir_device_bytes(s: *const cs_plonk_shamir) -> usize;
    pub fn cs_shamir_double_sharings(ctx: *mut cs_ctx, st: *mut cs_shamir_state, net: *mut cs_net, count: usize,
                                     d_rt: *mut u64, d_r2t: *mut u64) -> c_int;
    // --- large-vector Rep3 products, batched VM opcodes, Honk commitments and sumcheck kernels
    pub fn cs_rep3_mul_vec_reshare(ctx: *mut cs_ctx, curve: c_int, d_a: *const u64, d_b: *const u64, n: usize,
                                   prf: *const cs_rep3_prf, d_out: *mut u64, d_next_out: *mut u64) -> c_int;
    pub fn cs_rep3_batch(ctx: *mut cs_ctx, curve: c_int, op: c_int, party: c_int, d_x: *const u64, d_y: *const u64,
                         d_out: *mut u64, n: usize) -> c_int;
    pub fn cs_honk_commit_batch(ctx: *mut cs_ctx, crs: *const cs_bases, kind: c_int, d_polys: *const *const u64,
                                lens: *const usize, k: c_uint, out_points: *mut u64) -> c_int;
    pub fn cs_sumcheck_gate_separator(ctx: *mut cs_ctx, curve: c_int, betas: *const u64, log_n: c_uint, d_out: *mut u64) -> c_int;
    pub fn cs_sumcheck_fold(ctx: *mut cs_ctx, curve: c_int, d_in: *const *const u64, d_out: *const *mut u64, n_polys: usize,
                            shared: c_int, len: usize, challenge: *const u64) -> c_int;
    pub fn cs_sumcheck_arith_round(ctx: *mut cs_ctx, curve: c_int, kind: c_int, party: c_int, d_polys: *const cs_honk_arith_polys,
                                   round_size: usize, d_beta_products: *const u64, periodicity: usize,
                                   prf: *const cs_rep3_prf, r0: *mut u64, r1: *mut u64) -> c_int;
    pub fn cs_groth16_prove_with_shamir_bridge(ctx: *mut cs_ctx, pk: *mut cs_groth16_pk, net0: *mut cs_net,
                                               net1: *mut cs_net, public_inputs: *const u64,
                                               witness_rep3_shares: *const u64, out_a: *mut u64, out_b: *mut u64,
                                               out_c: *mut u64, out_rs: *mut u64) -> c_int;
}

/// `Err(message)` for a non-zero return code.
pub fn check(rc: c_int) -> Result<(), String> {
    if rc == 0 {
        return Ok(());
    }
    let msg = unsafe { std::ffi::CStr::from_ptr(cs_last_error()) }.to_string_lossy().into_owned();
    Err(format!("cosnarks_gpu ({rc}): {msg}"))
}
