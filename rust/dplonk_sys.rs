//! `extern "C"` view of include/dplonk.h (the subset the worker needs; one line per symbol, same order as the header).
//! Every function returns 0 (DP_OK) or a negative DP_E_* code and never unwinds; `dp_last_error` gives the text.
#![allow(non_camel_case_types, dead_code)]
use std::ffi::CStr;
use std::os::raw::{c_char, c_int, c_void};

#[repr(C)]
pub struct dp_ctx {
    _private: [u8; 0],
}

/// FftWorkload of utils.rs:3-9 as it crosses the ABI (include/dplonk.h: dp_fft_workload)
#[repr(C)]
#[derive(Clone, Copy)]
pub struct dp_fft_workload {
    pub row_start: u64,
    pub row_end: u64,
    pub col_start: u64,
    pub col_end: u64,
}

pub const DP_IPC_HANDLE_BYTES: usize = 64;

/// the 25 coset-evaluation arrays and the challenges of round 3 (include/dplonk.h: dp_quotient_args)
#[repr(C)]
pub struct dp_quotient_args {
    pub selectors: [*const c_void; 13],
    pub sigmas: [*const c_void; 5],
    pub wires: [*const c_void; 5],
    pub perm: *const c_void,
    pub pub_input: *const c_void,
    pub k: *const u8,
    pub alpha: *const u8,
    pub beta: *const u8,
    pub gamma: *const u8,
}

/// coefficients n, n+1, ... of each blinded wire and of z, device pointers, at most 3 each (include/dplonk.h: dp_quotient_tails)
#[repr(C)]
pub struct dp_quotient_tails {
    pub wires: [*const c_void; 5],
    pub wire_len: [usize; 5],
    pub perm: *const c_void,
    pub perm_len: usize,
}

extern "C" {
    pub fn dp_create(cuda_device: c_int, me: u64, n_workers: u64, out: *mut *mut dp_ctx) -> c_int;
    pub fn dp_destroy(ctx: *mut dp_ctx) -> c_int;
    pub fn dp_last_error(ctx: *const dp_ctx) -> *const c_char;
    pub fn dp_init(ctx: *mut dp_ctx, bases: *const u8, n_bases: usize, domain_size: u64, quot_domain_size: u64) -> c_int;
    pub fn dp_srs_powers_of_tau(ctx: *mut dp_ctx, tau32: *const u8, n: usize, out104: *mut c_void) -> c_int;
    pub fn dp_g1_decompress(ctx: *mut dp_ctx, in48: *const u8, n: usize, check_subgroup: c_int, out104: *mut u8,
                            bad_index: *mut usize, why: *mut c_int) -> c_int;
    pub fn dp_msm_points(ctx: *mut dp_ctx, points104: *const u8, scalars32: *const u8, n: usize, out144: *mut u8) -> c_int;
    pub fn dp_srs_open_key(ctx: *mut dp_ctx, tau32: *const u8, out400: *mut u8) -> c_int;
    pub fn dp_multi_pairing(ctx: *mut dp_ctx, g1_104: *const u8, g2_200: *const u8, k: usize, out576: *mut u8) -> c_int;
    pub fn dp_srs_update(ctx: *mut dp_ctx, s32: *const u8, g2_400: *const u8, out48: *mut c_void, out400: *mut c_void) -> c_int;
    pub fn dp_msm(ctx: *mut dp_ctx, start: u64, end: u64, scalars: *const u8, n_scalars: usize, out144: *mut u8) -> c_int;
    pub fn dp_msm_submit(ctx: *mut dp_ctx, id: u64, start: u64, end: u64, scalars: *const u8, n_scalars: usize) -> c_int;
    pub fn dp_msm_collect(ctx: *mut dp_ctx, id: u64, out144: *mut u8) -> c_int;
    pub fn dp_commit(ctx: *mut dp_ctx, coeffs: *const u8, n: usize, out144: *mut u8) -> c_int;
    pub fn dp_fft_init(ctx: *mut dp_ctx, id: u64, workloads: *const dp_fft_workload, n_workloads: usize,
                       is_quot: c_int, is_inv: c_int, is_coset: c_int) -> c_int;
    pub fn dp_fft1(ctx: *mut dp_ctx, id: u64, i: u64, row: *const u8, len: usize) -> c_int;
    pub fn dp_fft1_rows(ctx: *mut dp_ctx, id: u64, i_first: u64, n_rows: u64, rows: *const u8) -> c_int;
    pub fn dp_fft1_rows_short(ctx: *mut dp_ctx, id: u64, i_first: u64, n_rows: u64, rows: *const u8, row_len: usize) -> c_int;
    pub fn dp_fft2_prepare(ctx: *mut dp_ctx, id: u64) -> c_int;
    pub fn dp_fft_exchange_begin(ctx: *mut dp_ctx, id: u64, send_dev: *mut *mut c_void, recv_dev: *mut *mut c_void,
                                 block_elems: *mut u64) -> c_int;
    pub fn dp_fft_exchange_begin_async(ctx: *mut dp_ctx, id: u64, send_dev: *mut *mut c_void, recv_dev: *mut *mut c_void,
                                       block_elems: *mut u64) -> c_int;
    pub fn dp_compute_stream(ctx: *mut dp_ctx, stream: *mut *mut c_void) -> c_int;
    pub fn dp_fft_exchange_end(ctx: *mut dp_ctx, id: u64) -> c_int;
    pub fn dp_fft2(ctx: *mut dp_ctx, id: u64, out: *mut u8, out_bytes: usize) -> c_int;
    pub fn dp_round1(ctx: *mut dp_ctx, evals: *const u8, n: usize, blind_2fr: *const u8, out144: *mut u8) -> c_int;
    pub fn dp_get_wire(ctx: *mut dp_ctx, out: *mut u8, out_bytes: usize, n_coeffs: *mut usize) -> c_int;
    pub fn dp_quotient_evals_dev(ctx: *mut dp_ctx, dev_arrays: *const dp_quotient_args, out_dev: *mut c_void) -> c_int;
    pub fn dp_ntt_dev_quot_slice(ctx: *mut dp_ctx, coeffs_dev: *const c_void, n_valid: usize, slice: u32, out_dev: *mut c_void,
                                 wait: c_int) -> c_int;
    pub fn dp_quotient_evals_slice_dev(ctx: *mut dp_ctx, slice_arrays: *const dp_quotient_args, slice: u32,
                                       out_dev: *mut c_void) -> c_int;
    pub fn dp_quotient_evals_tail_dev(ctx: *mut dp_ctx, dev_arrays: *const dp_quotient_args, tails: *const dp_quotient_tails,
                                      out_dev: *mut c_void) -> c_int;
    pub fn dp_quotient_evals_slice_tail_dev(ctx: *mut dp_ctx, slice_arrays: *const dp_quotient_args, tails: *const dp_quotient_tails,
                                            slice: u32, out_dev: *mut c_void) -> c_int;
    /// out_dev += scale * quotient: round 3 of a batch proof; tails may be null (unblinded)
    pub fn dp_quotient_evals_acc_dev(ctx: *mut dp_ctx, dev_arrays: *const dp_quotient_args, tails: *const dp_quotient_tails,
                                     scale_fr: *const u8, out_dev: *mut c_void) -> c_int;
    pub fn dp_quotient_evals_slice_acc_dev(ctx: *mut dp_ctx, slice_arrays: *const dp_quotient_args, tails: *const dp_quotient_tails,
                                           slice: u32, scale_fr: *const u8, out_dev: *mut c_void) -> c_int;
    pub fn dp_poly_blind_dev(ctx: *mut dp_ctx, coeffs_dev: *mut c_void, n: usize, k: u32, blind_kfr: *const u8) -> c_int;
    pub fn dp_wire_permutation_scratch_bytes(num_wire_types: usize, n: usize, num_vars: u64, bytes: *mut usize) -> c_int;
    pub fn dp_wire_permutation_dev(ctx: *mut dp_ctx, vars_dev: *const u32, num_wire_types: usize, n: usize, num_vars: u64,
                                   scratch_dev: *mut c_void, scratch_bytes: usize, succ_out_dev: *mut u32) -> c_int;
    pub fn dp_perm_evals_dev(ctx: *mut dp_ctx, succ_dev: *const u32, num_wire_types: usize, n: usize, k: *const u8,
                             id_out_dev: *mut c_void, sigma_out_dev: *mut c_void) -> c_int;
    pub fn dp_witness_gather_dev(ctx: *mut dp_ctx, witness_dev: *const c_void, num_vars: u64, vars_dev: *const u32,
                                 num_wire_types: usize, n: usize, num_inputs: usize, wires_out_dev: *mut c_void,
                                 pub_out_dev: *mut c_void) -> c_int;
    pub fn dp_commit_dev_batch(ctx: *mut dp_ctx, n_jobs: usize, coeffs_dev: *const *mut c_void, lens: *const usize,
                               outs144: *mut u8) -> c_int;
    pub fn dp_peer_arena_create(ctx: *mut dp_ctx, arena_bytes: u64, handle_out: *mut u8) -> c_int;
    pub fn dp_peer_attach(ctx: *mut dp_ctx, peer: u64, handle: *const u8) -> c_int;
    pub fn dp_peer_ready(ctx: *const dp_ctx) -> c_int;
    pub fn dp_sync(ctx: *mut dp_ctx) -> c_int;
}

/// non-zero return code -> the capnp error the caller of the RPC sees (the reference `unwrap()`s and panics instead)
pub fn check(ctx: *const dp_ctx, rc: c_int) -> Result<(), capnp::Error> {
    if rc == 0 {
        return Ok(());
    }
    let msg = unsafe { CStr::from_ptr(dp_last_error(ctx)) }.to_string_lossy().into_owned();
    Err(capnp::Error::failed(format!("dplonk error {}: {}", rc, msg)))
}
