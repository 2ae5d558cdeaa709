"""ctypes binding of the C ABI declared in include/dplonk.h (one Python method per entry point)."""
from __future__ import annotations

import ctypes as C

import numpy as np

DP_OK, DP_E_ARG, DP_E_STATE, DP_E_OOM, DP_E_CUDA, DP_E_COMM = 0, -1, -2, -3, -4, -5
FR_BYTES, G1_AFFINE_BYTES, G1_PROJECTIVE_BYTES = 32, 104, 144
G1_COMPRESSED_BYTES, G2_AFFINE_BYTES, FQ12_BYTES = 48, 200, 576
G2_COMPRESSED_BYTES = 96
LINCOMB_MAX = 32                 # operands of one dp_poly_lincomb call (RND_MAX_POLYS)
FR_MODULUS = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001

EXPORTS = [
    "dp_create", "dp_destroy", "dp_last_error", "dp_version", "dp_init", "dp_msm", "dp_commit", "dp_fft_init",
    "dp_fft1", "dp_fft1_rows", "dp_fft2_prepare", "dp_fft_exchange_begin", "dp_fft_exchange_end", "dp_fft2",
    "dp_ntt", "dp_round1", "dp_get_wire", "dp_peer_arena_create", "dp_peer_attach", "dp_last_timing",
    "dp_launch_count", "dp_sync", "dp_msm_dev", "dp_ntt_dev", "dp_fft_dev", "dp_debug_set_limits",
    "dp_last_msm_breakdown", "dp_msm_tuning", "dp_msm_tuning_all", "dp_debug_gen_bases", "dp_fft_dev_rows", "dp_fft_dev_cols", "dp_peer_ready", "dp_fft_dev_rows_p2p", "dp_fft_dev_p2p", "dp_msm_dev_batch", "dp_perm_product", "dp_msm_batch", "dp_perm_product_dev",
    "dp_quotient_evals", "dp_quotient_evals_dev", "dp_poly_eval", "dp_poly_eval_dev", "dp_poly_lincomb", "dp_poly_lincomb_dev",
    "dp_poly_div_linear", "dp_poly_div_linear_dev", "dp_init_compressed", "dp_get_bases",
    "dp_msm_submit", "dp_msm_collect", "dp_poly_put", "dp_poly_ptr", "dp_poly_get", "dp_poly_free", "dp_commit_dev",
    "dp_fft_exchange_begin_async", "dp_compute_stream", "dp_fft_dev_p2p_async", "dp_fft1_rows_short", "dp_fft_dev_hint_valid_cols", "dp_ntt_dev_padded", "dp_debug_set_three_pass",
    "dp_ntt_dev_quot_slice", "dp_quotient_evals_slice_dev",
    "dp_poly_blind_dev", "dp_quotient_evals_tail_dev", "dp_quotient_evals_slice_tail_dev",
    "dp_wire_permutation_scratch_bytes", "dp_wire_permutation_dev", "dp_perm_evals_dev", "dp_witness_gather_dev", "dp_commit_dev_batch",
    "dp_srs_powers_of_tau",
    "dp_g1_decompress", "dp_msm_points", "dp_srs_open_key", "dp_multi_pairing",
    "dp_g1_compress", "dp_get_bases_compressed", "dp_g2_compress", "dp_g2_decompress", "dp_srs_check", "dp_last_srs_check",
    "dp_srs_update", "dp_debug_srs_update_plain",
    "dp_quotient_evals_acc_dev", "dp_quotient_evals_slice_acc_dev",
]


class DpError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"dplonk error {code}: {msg}")
        self.code = code
        self.msg = msg


class FftWorkload(C.Structure):
    """utils.rs:3-19 / hello_world.capnp:8-13"""
    _fields_ = [("row_start", C.c_uint64), ("row_end", C.c_uint64), ("col_start", C.c_uint64), ("col_end", C.c_uint64)]


class QuotientArgs(C.Structure):
    """dp_quotient_args (include/dplonk.h): 25 polynomial-sized arrays + the challenges"""
    _fields_ = [("selectors", C.c_void_p * 13), ("sigmas", C.c_void_p * 5), ("wires", C.c_void_p * 5), ("perm", C.c_void_p),
                ("pub_input", C.c_void_p), ("k", C.c_void_p), ("alpha", C.c_void_p), ("beta", C.c_void_p), ("gamma", C.c_void_p)]


class QuotientTails(C.Structure):
    """dp_quotient_tails (include/dplonk.h): coefficients n, n+1, ... of each blinded wire and of z (device pointers)"""
    _fields_ = [("wires", C.c_void_p * 5), ("wire_len", C.c_size_t * 5), ("perm", C.c_void_p), ("perm_len", C.c_size_t)]


def bind(cdll: C.CDLL) -> C.CDLL:
    u64, vp, i, sz, u32 = C.c_uint64, C.c_void_p, C.c_int, C.c_size_t, C.c_uint32
    sig = {
        "dp_create": (i, [i, u64, u64, C.POINTER(vp)]),
        "dp_destroy": (i, [vp]),
        "dp_last_error": (C.c_char_p, [vp]),
        "dp_version": (C.c_char_p, []),
        "dp_init": (i, [vp, vp, sz, u64, u64]),
        "dp_msm": (i, [vp, u64, u64, vp, sz, vp]),
        "dp_commit": (i, [vp, vp, sz, vp]),
        "dp_fft_init": (i, [vp, u64, C.POINTER(FftWorkload), sz, i, i, i]),
        "dp_fft1": (i, [vp, u64, u64, vp, sz]),
        "dp_fft1_rows": (i, [vp, u64, u64, u64, vp]),
        "dp_fft1_rows_short": (i, [vp, u64, u64, u64, vp, sz]),
        "dp_fft2_prepare": (i, [vp, u64]),
        "dp_fft_exchange_begin": (i, [vp, u64, C.POINTER(vp), C.POINTER(vp), C.POINTER(u64)]),
        "dp_fft_exchange_end": (i, [vp, u64]),
        "dp_fft_exchange_begin_async": (i, [vp, u64, C.POINTER(vp), C.POINTER(vp), C.POINTER(u64)]),
        "dp_compute_stream": (i, [vp, C.POINTER(vp)]),
        "dp_fft2": (i, [vp, u64, vp, sz]),
        "dp_ntt": (i, [vp, vp, sz, u32, i, i]),
        "dp_round1": (i, [vp, vp, sz, vp, vp]),
        "dp_get_wire": (i, [vp, vp, sz, C.POINTER(sz)]),
        "dp_peer_arena_create": (i, [vp, u64, vp]),
        "dp_peer_attach": (i, [vp, u64, vp]),
        "dp_last_timing": (i, [vp, C.POINTER(C.c_float), C.POINTER(u64)]),
        "dp_launch_count": (u64, [vp]),
        "dp_sync": (i, [vp]),
        "dp_msm_dev": (i, [vp, u64, u64, vp, sz, vp]),
        "dp_ntt_dev": (i, [vp, vp, u32, i, i]),
        "dp_ntt_dev_padded": (i, [vp, vp, sz, C.c_uint32, i, i, i]),
        "dp_fft_dev": (i, [vp, vp, vp, i, i, i]),
        "dp_debug_set_limits": (i, [vp, u32, u32, i]),
        "dp_last_msm_breakdown": (i, [vp, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float)]),
        "dp_msm_tuning": (i, [vp, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
        "dp_msm_tuning_all": (i, [vp, C.POINTER(C.c_float)]),
        "dp_debug_gen_bases": (i, [vp, u64, sz, vp]),
        "dp_fft_dev_rows": (i, [vp, vp, i, i, i, C.POINTER(vp), C.POINTER(vp), C.POINTER(u64)]),
        "dp_fft_dev_cols": (i, [vp, vp]),
        "dp_peer_ready": (i, [vp]),
        "dp_perm_product": (i, [vp, vp, vp, vp, sz, sz, vp, vp, vp]),
        "dp_perm_product_dev": (i, [vp, vp, vp, vp, sz, sz, vp, vp, vp]),
        "dp_msm_batch": (i, [vp, sz, C.POINTER(u64), C.POINTER(u64), C.POINTER(vp), C.POINTER(sz), C.POINTER(vp)]),
        "dp_msm_dev_batch": (i, [vp, sz, C.POINTER(u64), C.POINTER(u64), C.POINTER(vp), C.POINTER(sz), C.POINTER(vp)]),
        "dp_fft_dev_rows_p2p": (i, [vp, vp, i, i, i]),
        "dp_fft_dev_p2p": (i, [vp, vp, vp, i, i, i]),
        "dp_fft_dev_p2p_async": (i, [vp, vp, vp, i, i, i]),
        "dp_fft_dev_hint_valid_cols": (i, [vp, i, u64]),
        "dp_debug_set_three_pass": (i, [vp, C.c_uint32]),
        "dp_poly_put": (i, [vp, u64, vp, sz, sz]),
        "dp_poly_ptr": (i, [vp, u64, C.POINTER(vp), C.POINTER(sz)]),
        "dp_poly_get": (i, [vp, u64, sz, sz, vp]),
        "dp_poly_free": (i, [vp, u64]),
        "dp_commit_dev": (i, [vp, vp, sz, vp]),
        "dp_msm_submit": (i, [vp, u64, u64, u64, vp, sz]),
        "dp_msm_collect": (i, [vp, u64, vp]),
        "dp_init_compressed": (i, [vp, vp, sz, u64, u64, i]),
        "dp_get_bases": (i, [vp, u64, sz, vp]),
        "dp_quotient_evals": (i, [vp, C.POINTER(QuotientArgs), vp]),
        "dp_quotient_evals_dev": (i, [vp, C.POINTER(QuotientArgs), vp]),
        "dp_quotient_evals_slice_dev": (i, [vp, C.POINTER(QuotientArgs), u32, vp]),
        "dp_ntt_dev_quot_slice": (i, [vp, vp, sz, u32, vp, i]),
        "dp_quotient_evals_tail_dev": (i, [vp, C.POINTER(QuotientArgs), C.POINTER(QuotientTails), vp]),
        "dp_quotient_evals_slice_tail_dev": (i, [vp, C.POINTER(QuotientArgs), C.POINTER(QuotientTails), u32, vp]),
        "dp_quotient_evals_acc_dev": (i, [vp, C.POINTER(QuotientArgs), C.POINTER(QuotientTails), vp, vp]),
        "dp_quotient_evals_slice_acc_dev": (i, [vp, C.POINTER(QuotientArgs), C.POINTER(QuotientTails), u32, vp, vp]),
        "dp_poly_blind_dev": (i, [vp, vp, sz, u32, vp]),
        "dp_wire_permutation_scratch_bytes": (i, [sz, sz, u64, C.POINTER(sz)]),
        "dp_wire_permutation_dev": (i, [vp, vp, sz, sz, u64, vp, sz, vp]),
        "dp_perm_evals_dev": (i, [vp, vp, sz, sz, vp, vp, vp]),
        "dp_witness_gather_dev": (i, [vp, vp, u64, vp, sz, sz, sz, vp, vp]),
        "dp_commit_dev_batch": (i, [vp, sz, C.POINTER(vp), C.POINTER(sz), vp]),
        "dp_srs_powers_of_tau": (i, [vp, vp, sz, vp]),
        "dp_g1_decompress": (i, [vp, vp, sz, i, vp, C.POINTER(sz), C.POINTER(i)]),
        "dp_msm_points": (i, [vp, vp, vp, sz, vp]),
        "dp_srs_open_key": (i, [vp, vp, vp]),
        "dp_multi_pairing": (i, [vp, vp, vp, sz, vp]),
        "dp_g1_compress": (i, [vp, vp, sz, vp]),
        "dp_get_bases_compressed": (i, [vp, u64, sz, vp]),
        "dp_g2_compress": (i, [vp, vp, sz, vp]),
        "dp_g2_decompress": (i, [vp, vp, sz, i, vp, C.POINTER(sz), C.POINTER(i)]),
        "dp_srs_check": (i, [vp, vp, vp, C.POINTER(i)]),
        "dp_last_srs_check": (i, [vp, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float), vp]),
        "dp_srs_update": (i, [vp, vp, vp, vp, vp]),
        "dp_debug_srs_update_plain": (i, [vp, vp, vp, vp, vp]),
        "dp_poly_eval": (i, [vp, vp, sz, vp, vp]),
        "dp_poly_eval_dev": (i, [vp, vp, sz, vp, vp]),
        "dp_poly_lincomb": (i, [vp, C.POINTER(vp), C.POINTER(sz), vp, sz, vp, sz]),
        "dp_poly_lincomb_dev": (i, [vp, C.POINTER(vp), C.POINTER(sz), vp, sz, vp, sz]),
        "dp_poly_div_linear": (i, [vp, vp, sz, vp, vp, vp]),
        "dp_poly_div_linear_dev": (i, [vp, vp, sz, vp, vp, vp]),
    }
    assert set(sig) == set(EXPORTS)
    for name, (res, args) in sig.items():
        f = getattr(cdll, name)  # AttributeError here = the library does not export what dplonk.h declares
        f.restype = res
        f.argtypes = args
    return cdll


def _addr(buf) -> int:
    """host address of a numpy array / bytes-like / raw int address."""
    if isinstance(buf, int):
        return buf
    if isinstance(buf, np.ndarray):
        assert buf.flags["C_CONTIGUOUS"]
        return buf.ctypes.data
    return C.addressof(C.c_char.from_buffer(buf))


class Context:
    """One dp_ctx (one GPU).  Thin: arguments are numpy arrays in the reference's raw layouts."""

    def __init__(self, cdll: C.CDLL, device: int = 0, me: int = 0, n_workers: int = 1):
        self.lib = cdll
        self.me, self.n_workers = me, n_workers
        h = C.c_void_p()
        rc = cdll.dp_create(device, me, n_workers, C.byref(h))
        if rc != DP_OK:
            raise DpError(rc, (cdll.dp_last_error(None) or b"").decode())
        self.h = h

    def close(self):
        if self.h:
            self.lib.dp_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc: int):
        if rc != DP_OK:
            raise DpError(rc, (self.lib.dp_last_error(self.h) or b"").decode())

    # ---- PlonkSlave surface
    def init(self, bases: np.ndarray, domain_size: int, quot_domain_size: int):
        bases = np.ascontiguousarray(bases, dtype=np.uint8)
        n = bases.size // G1_AFFINE_BYTES
        self._ck(self.lib.dp_init(self.h, _addr(bases) if n else None, n, domain_size, quot_domain_size))

    def msm(self, start: int, end: int, scalars: np.ndarray) -> np.ndarray:
        scalars = np.ascontiguousarray(scalars)
        n = scalars.nbytes // 32
        out = np.zeros(G1_PROJECTIVE_BYTES, dtype=np.uint8)
        self._ck(self.lib.dp_msm(self.h, start, end, _addr(scalars) if n else None, n, _addr(out)))
        return out

    def commit(self, coeffs: np.ndarray) -> np.ndarray:
        coeffs = np.ascontiguousarray(coeffs)
        n = coeffs.nbytes // 32
        out = np.zeros(G1_PROJECTIVE_BYTES, dtype=np.uint8)
        self._ck(self.lib.dp_commit(self.h, _addr(coeffs) if n else None, n, _addr(out)))
        return out

    def fft_init(self, task_id: int, workloads, is_quot: bool, is_inv: bool, is_coset: bool):
        arr = (FftWorkload * len(workloads))(*[FftWorkload(*w) for w in workloads])
        self._ck(self.lib.dp_fft_init(self.h, task_id, arr, len(workloads), int(is_quot), int(is_inv), int(is_coset)))

    def fft1(self, task_id: int, i: int, row: np.ndarray):
        row = np.ascontiguousarray(row)
        self._ck(self.lib.dp_fft1(self.h, task_id, i, _addr(row), row.nbytes // 32))

    def fft1_rows(self, task_id: int, i_first: int, rows: np.ndarray, n_rows: int):
        rows = np.ascontiguousarray(rows)
        self._ck(self.lib.dp_fft1_rows(self.h, task_id, i_first, n_rows, _addr(rows)))

    def fft1_rows_short(self, task_id: int, i_first: int, rows, n_rows: int, row_len: int):
        """n_rows rows of row_len leading entries each (compact array or host address); the tails are implicit zeros"""
        self._ck(self.lib.dp_fft1_rows_short(self.h, task_id, i_first, n_rows, _addr(rows), row_len))

    def fft2_prepare(self, task_id: int):
        self._ck(self.lib.dp_fft2_prepare(self.h, task_id))

    def fft_exchange_begin(self, task_id: int):
        s, r, n = C.c_void_p(), C.c_void_p(), C.c_uint64()
        self._ck(self.lib.dp_fft_exchange_begin(self.h, task_id, C.byref(s), C.byref(r), C.byref(n)))
        return s.value, r.value, n.value

    def fft_exchange_begin_async(self, task_id: int):
        """like fft_exchange_begin, without waiting: the buffers are valid for work on compute_stream()"""
        s, r, n = C.c_void_p(), C.c_void_p(), C.c_uint64()
        self._ck(self.lib.dp_fft_exchange_begin_async(self.h, task_id, C.byref(s), C.byref(r), C.byref(n)))
        return s.value, r.value, n.value

    def compute_stream(self) -> int:
        st = C.c_void_p()
        self._ck(self.lib.dp_compute_stream(self.h, C.byref(st)))
        return st.value or 0

    def fft_exchange_end(self, task_id: int):
        self._ck(self.lib.dp_fft_exchange_end(self.h, task_id))

    def fft2(self, task_id: int, n_cols: int, r: int) -> np.ndarray:
        out = np.empty((n_cols, r, 4), dtype=np.uint64)
        self._ck(self.lib.dp_fft2(self.h, task_id, _addr(out), out.nbytes))
        return out

    def ntt(self, data: np.ndarray, log_n: int, is_inv: bool, is_coset: bool) -> np.ndarray:
        n = data.nbytes // 32
        buf = np.zeros((1 << log_n, 4), dtype=np.uint64)
        buf.reshape(-1)[: n * 4] = np.ascontiguousarray(data).view(np.uint64).reshape(-1)
        self._ck(self.lib.dp_ntt(self.h, _addr(buf), n, log_n, int(is_inv), int(is_coset)))
        return buf

    def round1(self, evals: np.ndarray, blind: np.ndarray | None) -> np.ndarray:
        evals = np.ascontiguousarray(evals)
        out = np.zeros(G1_PROJECTIVE_BYTES, dtype=np.uint8)
        b = np.ascontiguousarray(blind) if blind is not None else None
        self._ck(self.lib.dp_round1(self.h, _addr(evals), evals.nbytes // 32, _addr(b) if b is not None else None, _addr(out)))
        return out

    def perm_product(self, wires: np.ndarray, id_perm: np.ndarray, sigma_perm: np.ndarray, beta: np.ndarray, gamma: np.ndarray) -> np.ndarray:
        """round-2 grand product (dispatcher2.rs:329-345); inputs [n_types, n, 4] u64 raw Fr"""
        a = [np.ascontiguousarray(x, dtype=np.uint64) for x in (wires, id_perm, sigma_perm, beta, gamma)]
        n_types, n = a[0].shape[0], a[0].shape[1]
        out = np.empty((n, 4), dtype=np.uint64)
        self._ck(self.lib.dp_perm_product(self.h, _addr(a[0]), _addr(a[1]), _addr(a[2]), n_types, n, _addr(a[3]), _addr(a[4]), _addr(out)))
        return out

    def perm_product_dev(self, wires_ptr: int, id_ptr: int, sigma_ptr: int, n_types: int, n: int, beta: np.ndarray, gamma: np.ndarray, out_ptr: int):
        b, g = np.ascontiguousarray(beta, dtype=np.uint64), np.ascontiguousarray(gamma, dtype=np.uint64)
        self._ck(self.lib.dp_perm_product_dev(self.h, wires_ptr, id_ptr, sigma_ptr, n_types, n, _addr(b), _addr(g), out_ptr))

    # ---- worker-resident polynomials
    def poly_put(self, poly_id: int, coeffs: np.ndarray, capacity: int = 0) -> int:
        """store [n,4] raw Fr under poly_id (zero-extended to `capacity`); returns the device address"""
        a = np.ascontiguousarray(coeffs, dtype=np.uint64)
        self._ck(self.lib.dp_poly_put(self.h, poly_id, _addr(a) if a.size else None, a.size // 4, capacity))
        return self.poly_ptr(poly_id)[0]

    def poly_ptr(self, poly_id: int):
        d, cap = C.c_void_p(), C.c_size_t()
        self._ck(self.lib.dp_poly_ptr(self.h, poly_id, C.byref(d), C.byref(cap)))
        return d.value, cap.value

    def poly_get(self, poly_id: int, n: int | None = None, offset: int = 0) -> np.ndarray:
        if n is None:
            n = self.poly_ptr(poly_id)[1] - offset
        out = np.empty((n, 4), dtype=np.uint64)
        self._ck(self.lib.dp_poly_get(self.h, poly_id, offset, n, _addr(out) if n else None))
        return out

    def poly_free(self, poly_id: int):
        self._ck(self.lib.dp_poly_free(self.h, poly_id))

    def commit_dev(self, coeffs_ptr: int, n: int) -> np.ndarray:
        out = np.zeros(G1_PROJECTIVE_BYTES, dtype=np.uint8)
        self._ck(self.lib.dp_commit_dev(self.h, coeffs_ptr, n, _addr(out)))
        return out

    def msm_submit(self, job_id: int, start: int, end: int, scalars, n: int | None = None):
        """asynchronous varMsm: scalars = [n,4] host array (kept alive by the caller) or a host pointer + n"""
        if isinstance(scalars, int):
            self._ck(self.lib.dp_msm_submit(self.h, job_id, start, end, scalars, n))
        else:
            a = np.ascontiguousarray(scalars)
            self._keep = getattr(self, "_keep", {})
            self._keep[job_id] = a
            self._ck(self.lib.dp_msm_submit(self.h, job_id, start, end, _addr(a) if a.size else None, a.nbytes // 32))

    def msm_collect(self, job_id: int) -> np.ndarray:
        out = np.zeros(G1_PROJECTIVE_BYTES, dtype=np.uint8)
        try:
            self._ck(self.lib.dp_msm_collect(self.h, job_id, _addr(out)))
        finally:
            getattr(self, "_keep", {}).pop(job_id, None)
        return out

    def init_compressed(self, bases48: np.ndarray, domain_size: int, quot_domain_size: int, check_subgroup: bool = True):
        """dp_init from ark-serialize compressed points ([n, 48] uint8)"""
        b = np.ascontiguousarray(bases48, dtype=np.uint8)
        self._ck(self.lib.dp_init_compressed(self.h, _addr(b) if b.size else None, b.size // 48, domain_size, quot_domain_size, int(check_subgroup)))

    def get_bases(self, start: int, n: int) -> np.ndarray:
        out = np.zeros((n, 104), dtype=np.uint8)
        self._ck(self.lib.dp_get_bases(self.h, start, n, _addr(out) if n else None))
        return out

    # ---- rounds 3-5 ("next" row 1): plain = host arrays, *_dev = device pointers (ints)
    @staticmethod
    def _quotient_args(selectors, sigmas, wires, perm, pub_input, k, alpha, beta, gamma, keep):
        """pointers may be ints (device) or numpy arrays (host; kept alive in `keep`)"""
        def ptr(x):
            if isinstance(x, int):
                return x
            a = np.ascontiguousarray(x, dtype=np.uint64)
            keep.append(a)
            return a.ctypes.data
        q = QuotientArgs()
        for j in range(13):
            q.selectors[j] = ptr(selectors[j])
        for j in range(5):
            q.sigmas[j] = ptr(sigmas[j])
            q.wires[j] = ptr(wires[j])
        q.perm, q.pub_input = ptr(perm), ptr(pub_input)
        q.k, q.alpha, q.beta, q.gamma = ptr(np.asarray(k)), ptr(np.asarray(alpha)), ptr(np.asarray(beta)), ptr(np.asarray(gamma))
        return q

    def quotient_evals(self, selectors, sigmas, wires, perm, pub_input, k, alpha, beta, gamma) -> np.ndarray:
        """round 3 (dispatcher2.rs:434-504) on host arrays: selectors [13][m,4], sigmas / wires [5][m,4], ..."""
        keep = []
        q = self._quotient_args(selectors, sigmas, wires, perm, pub_input, k, alpha, beta, gamma, keep)
        out = np.empty((np.asarray(perm).shape[0], 4), dtype=np.uint64)
        self._ck(self.lib.dp_quotient_evals(self.h, C.byref(q), _addr(out)))
        return out

    def quotient_evals_dev(self, selectors, sigmas, wires, perm, pub_input, k, alpha, beta, gamma, out_ptr: int):
        keep = []
        q = self._quotient_args(selectors, sigmas, wires, perm, pub_input, k, alpha, beta, gamma, keep)
        self._ck(self.lib.dp_quotient_evals_dev(self.h, C.byref(q), out_ptr))

    def quotient_evals_slice_dev(self, selectors, sigmas, wires, perm, pub_input, k, alpha, beta, gamma, slice_: int, out_ptr: int):
        """round 3 for slice `slice_` of the quotient coset: the 25 arrays hold n points each (ntt_dev_quot_slice); writes
        out[slice_ + (m/n) i], i < n, of the m-point output"""
        keep = []
        q = self._quotient_args(selectors, sigmas, wires, perm, pub_input, k, alpha, beta, gamma, keep)
        self._ck(self.lib.dp_quotient_evals_slice_dev(self.h, C.byref(q), slice_, out_ptr))

    @staticmethod
    def _quotient_tails(tails) -> QuotientTails:
        """tails: 6 (device pointer or None, length) pairs, the five wires then z"""
        t = QuotientTails()
        for j, (ptr, ln) in enumerate(tails[:5]):
            t.wires[j], t.wire_len[j] = ptr, ln
        t.perm, t.perm_len = tails[5]
        return t

    def quotient_evals_tail_dev(self, selectors, sigmas, wires, perm, pub_input, k, alpha, beta, gamma, tails, out_ptr: int):
        """quotient_evals_dev of blinded wires and z: the arrays hold the evaluations of their first n coefficients, `tails`
        gives coefficients n, n+1, ... of each (6 (pointer, length) pairs, wires then z, lengths <= 3)"""
        keep = []
        q = self._quotient_args(selectors, sigmas, wires, perm, pub_input, k, alpha, beta, gamma, keep)
        t = self._quotient_tails(tails)
        self._ck(self.lib.dp_quotient_evals_tail_dev(self.h, C.byref(q), C.byref(t), out_ptr))

    def quotient_evals_slice_tail_dev(self, selectors, sigmas, wires, perm, pub_input, k, alpha, beta, gamma, tails, slice_: int,
                                      out_ptr: int):
        """quotient_evals_slice_dev of blinded wires and z (quotient_evals_tail_dev)"""
        keep = []
        q = self._quotient_args(selectors, sigmas, wires, perm, pub_input, k, alpha, beta, gamma, keep)
        t = self._quotient_tails(tails)
        self._ck(self.lib.dp_quotient_evals_slice_tail_dev(self.h, C.byref(q), C.byref(t), slice_, out_ptr))

    def quotient_evals_acc_dev(self, selectors, sigmas, wires, perm, pub_input, k, alpha, beta, gamma, tails, scale, out_ptr: int,
                               slice_: int | None = None):
        """out[pt] += scale * quotient(pt) (a batch proof's round 3): over the whole coset (slice_ None, arrays of m points)
        or over slice slice_ (arrays of n points); tails as in quotient_evals_tail_dev, or None (unblinded); scale raw Fr"""
        keep = []
        q = self._quotient_args(selectors, sigmas, wires, perm, pub_input, k, alpha, beta, gamma, keep)
        t = C.byref(self._quotient_tails(tails)) if tails is not None else None
        sc = np.ascontiguousarray(scale, dtype=np.uint64)
        if slice_ is None:
            self._ck(self.lib.dp_quotient_evals_acc_dev(self.h, C.byref(q), t, _addr(sc), out_ptr))
        else:
            self._ck(self.lib.dp_quotient_evals_slice_acc_dev(self.h, C.byref(q), t, slice_, _addr(sc), out_ptr))

    def poly_blind_dev(self, coeffs_ptr: int, n: int, k: int, blind: np.ndarray | None = None):
        """coeffs += b(X) * (X^n - 1) in place (n + k Fr on the device); blind = [k,4] raw Fr, or None: the library draws
        the k scalars from the OS entropy pool and they never leave it"""
        b = np.ascontiguousarray(blind, dtype=np.uint64) if blind is not None else None
        self._ck(self.lib.dp_poly_blind_dev(self.h, coeffs_ptr, n, k, _addr(b) if b is not None else None))

    # ---- circuit preprocessing and the witness gather (device pointers; slot s = wire type * n + gate)
    def wire_permutation_scratch_bytes(self, num_wire_types: int, n: int, num_vars: int) -> int:
        b = C.c_size_t()
        self._ck(self.lib.dp_wire_permutation_scratch_bytes(num_wire_types, n, num_vars, C.byref(b)))
        return b.value

    def wire_permutation_dev(self, vars_ptr: int, num_wire_types: int, n: int, num_vars: int, scratch_ptr: int, scratch_bytes: int,
                             succ_ptr: int):
        """succ[s] = the next slot holding the same variable (wrapping to its first); u32 arrays of num_wire_types * n"""
        self._ck(self.lib.dp_wire_permutation_dev(self.h, vars_ptr, num_wire_types, n, num_vars, scratch_ptr, scratch_bytes, succ_ptr))

    def perm_evals_dev(self, succ_ptr, num_wire_types: int, n: int, k: np.ndarray, id_ptr: int, sigma_ptr: int):
        """id[i n + j] = k_i omega^j, sigma[s] = id[succ[s]] (succ_ptr None: sigma = id); k = [num_wire_types, 4] raw Fr"""
        kk = np.ascontiguousarray(k, dtype=np.uint64)
        self._ck(self.lib.dp_perm_evals_dev(self.h, succ_ptr, num_wire_types, n, _addr(kk), id_ptr, sigma_ptr))

    def witness_gather_dev(self, witness_ptr: int, num_vars: int, vars_ptr: int, num_wire_types: int, n: int, num_inputs: int,
                           wires_ptr: int, pub_ptr: int):
        """wires[s] = witness[vars[s]]; pub[j] = the last wire type's value at gate j < num_inputs, 0 up to n"""
        self._ck(self.lib.dp_witness_gather_dev(self.h, witness_ptr, num_vars, vars_ptr, num_wire_types, n, num_inputs, wires_ptr, pub_ptr))

    def commit_dev_batch(self, ptrs, lens) -> list:
        """commit_dev of several device polynomials as one MSM batch; returns [144-byte arrays]"""
        k = len(ptrs)
        out = np.zeros((k, G1_PROJECTIVE_BYTES), dtype=np.uint8)
        self._ck(self.lib.dp_commit_dev_batch(self.h, k, (C.c_void_p * k)(*ptrs), (C.c_size_t * k)(*lens), _addr(out) if k else None))
        return list(out)

    def poly_eval(self, coeffs, point: np.ndarray, n: int | None = None) -> np.ndarray:
        """round 4: p(point); coeffs = [n,4] host array, or a device pointer with n given"""
        pt, out = np.ascontiguousarray(point, dtype=np.uint64), np.empty(4, dtype=np.uint64)
        if isinstance(coeffs, int):
            self._ck(self.lib.dp_poly_eval_dev(self.h, coeffs, n, _addr(pt), _addr(out)))
        else:
            c = np.ascontiguousarray(coeffs, dtype=np.uint64)
            self._ck(self.lib.dp_poly_eval(self.h, _addr(c) if c.size else None, c.shape[0], _addr(pt), _addr(out)))
        return out

    def poly_div_linear(self, coeffs, point: np.ndarray, n: int | None = None, out_ptr: int | None = None):
        """round 5: (quotient of p / (X - point), remainder p(point)); device form writes the quotient to out_ptr"""
        pt, rem = np.ascontiguousarray(point, dtype=np.uint64), np.empty(4, dtype=np.uint64)
        if isinstance(coeffs, int):
            self._ck(self.lib.dp_poly_div_linear_dev(self.h, coeffs, n, _addr(pt), out_ptr, _addr(rem)))
            return None, rem
        c = np.ascontiguousarray(coeffs, dtype=np.uint64)
        out = np.empty((max(c.shape[0] - 1, 0), 4), dtype=np.uint64)
        self._ck(self.lib.dp_poly_div_linear(self.h, _addr(c) if c.size else None, c.shape[0], _addr(pt), _addr(out) if out.size else None, _addr(rem)))
        return out, rem

    def poly_lincomb(self, polys, coeffs: np.ndarray, out_len: int | None = None, lens=None, out_ptr: int | None = None):
        """round 5: sum_i coeffs[i] * polys[i]; polys = host arrays, or device pointers with lens and out_ptr given"""
        cf = np.ascontiguousarray(coeffs, dtype=np.uint64)
        k = len(polys)
        if out_ptr is not None:
            # more than LINCOMB_MAX operands: the output accumulates in place, [out] + the next 31 with coefficient 1
            head = min(k, LINCOMB_MAX)
            ptrs, ln = (C.c_void_p * head)(*polys[:head]), (C.c_size_t * head)(*lens[:head])
            self._ck(self.lib.dp_poly_lincomb_dev(self.h, ptrs, ln, _addr(np.ascontiguousarray(cf[:head])), head, out_ptr, out_len))
            one = np.frombuffer(((1 << 256) % FR_MODULUS).to_bytes(32, "little"), dtype=np.uint64)
            for s in range(head, k, LINCOMB_MAX - 1):
                e = min(k, s + LINCOMB_MAX - 1)
                ptrs = (C.c_void_p * (1 + e - s))(out_ptr, *polys[s:e])
                ln = (C.c_size_t * (1 + e - s))(out_len, *lens[s:e])
                c2 = np.ascontiguousarray(np.concatenate([one[None], cf[s:e]]))
                self._ck(self.lib.dp_poly_lincomb_dev(self.h, ptrs, ln, _addr(c2), 1 + e - s, out_ptr, out_len))
            return None
        ps = [np.ascontiguousarray(x, dtype=np.uint64) for x in polys]
        ln = [x.shape[0] for x in ps]
        n_out = max(ln) if out_len is None else out_len
        out = np.empty((n_out, 4), dtype=np.uint64)
        ptrs = (C.c_void_p * k)(*[x.ctypes.data if x.size else None for x in ps])
        self._ck(self.lib.dp_poly_lincomb(self.h, ptrs, (C.c_size_t * k)(*ln), _addr(cf), k, _addr(out) if n_out else None, n_out))
        return out

    def get_wire(self) -> np.ndarray:
        n = C.c_size_t()
        self._ck(self.lib.dp_get_wire(self.h, None, 0, C.byref(n)))
        out = np.empty((n.value, 4), dtype=np.uint64)
        self._ck(self.lib.dp_get_wire(self.h, _addr(out), out.nbytes, C.byref(n)))
        return out

    # ---- device-pointer variants (bench)
    def msm_dev(self, start, end, scalars_ptr: int, n: int, out_ptr: int):
        self._ck(self.lib.dp_msm_dev(self.h, start, end, scalars_ptr, n, out_ptr))

    def msm_batch(self, jobs):
        """jobs: list of (start, end, scalars ndarray | host address, n_scalars); returns [144-byte arrays]"""
        k = len(jobs)
        outs = [np.zeros(G1_PROJECTIVE_BYTES, dtype=np.uint8) for _ in range(k)]
        st = (C.c_uint64 * k)(*[j[0] for j in jobs])
        en = (C.c_uint64 * k)(*[j[1] for j in jobs])
        sc = (C.c_void_p * k)(*[_addr(j[2]) for j in jobs])
        ns = (C.c_size_t * k)(*[j[3] for j in jobs])
        ou = (C.c_void_p * k)(*[_addr(o) for o in outs])
        self._ck(self.lib.dp_msm_batch(self.h, k, st, en, sc, ns, ou))
        return outs

    def msm_dev_batch(self, jobs):
        """jobs: list of (start, end, scalars_ptr, n_scalars, out_ptr)"""
        k = len(jobs)
        st = (C.c_uint64 * k)(*[j[0] for j in jobs])
        en = (C.c_uint64 * k)(*[j[1] for j in jobs])
        sc = (C.c_void_p * k)(*[j[2] for j in jobs])
        ns = (C.c_size_t * k)(*[j[3] for j in jobs])
        ou = (C.c_void_p * k)(*[j[4] for j in jobs])
        self._ck(self.lib.dp_msm_dev_batch(self.h, k, st, en, sc, ns, ou))

    def ntt_dev(self, data_ptr: int, log_n: int, is_inv: bool, is_coset: bool):
        self._ck(self.lib.dp_ntt_dev(self.h, data_ptr, log_n, int(is_inv), int(is_coset)))

    def ntt_dev_padded(self, data_ptr: int, n_valid: int, log_n: int, is_inv: bool, is_coset: bool, wait: bool = True):
        """in place on 2^log_n Fr at data_ptr whose entries from n_valid on are zero"""
        self._ck(self.lib.dp_ntt_dev_padded(self.h, data_ptr, n_valid, log_n, int(is_inv), int(is_coset), int(wait)))

    def ntt_dev_quot_slice(self, coeffs_ptr: int, n_valid: int, slice_: int, out_ptr: int, wait: bool = True):
        """p(s * omega_n^i), i < n, s = g * omega_m^slice_: slice slice_ of the coset evaluation on the quotient domain, of the
        n_valid coefficients at coeffs_ptr (only read), into the n Fr at out_ptr"""
        self._ck(self.lib.dp_ntt_dev_quot_slice(self.h, coeffs_ptr, n_valid, slice_, out_ptr, int(wait)))

    def fft_dev(self, rows_ptr: int, cols_ptr: int, is_quot: bool, is_inv: bool, is_coset: bool):
        self._ck(self.lib.dp_fft_dev(self.h, rows_ptr, cols_ptr, int(is_quot), int(is_inv), int(is_coset)))

    def fft_dev_hint_valid_cols(self, is_quot: bool, valid_cols: int):
        self._ck(self.lib.dp_fft_dev_hint_valid_cols(self.h, int(is_quot), valid_cols))

    def fft_dev_rows(self, rows_ptr: int, is_quot: bool, is_inv: bool, is_coset: bool):
        s, r, n = C.c_void_p(), C.c_void_p(), C.c_uint64()
        self._ck(self.lib.dp_fft_dev_rows(self.h, rows_ptr, int(is_quot), int(is_inv), int(is_coset),
                                          C.byref(s), C.byref(r), C.byref(n)))
        return s.value, r.value, n.value

    def peer_arena_create(self, arena_bytes: int) -> bytes:
        h = C.create_string_buffer(64)
        self._ck(self.lib.dp_peer_arena_create(self.h, arena_bytes, h))
        return h.raw

    def peer_attach(self, peer: int, handle: bytes):
        self._ck(self.lib.dp_peer_attach(self.h, peer, C.create_string_buffer(handle, 64)))

    def peer_ready(self) -> bool:
        return bool(self.lib.dp_peer_ready(self.h))

    def fft_dev_rows_p2p(self, rows_ptr: int, is_quot: bool, is_inv: bool, is_coset: bool):
        self._ck(self.lib.dp_fft_dev_rows_p2p(self.h, rows_ptr, int(is_quot), int(is_inv), int(is_coset)))

    def fft_dev_p2p(self, rows_ptr: int, cols_ptr: int, is_quot: bool, is_inv: bool, is_coset: bool):
        self._ck(self.lib.dp_fft_dev_p2p(self.h, rows_ptr, cols_ptr, int(is_quot), int(is_inv), int(is_coset)))

    def fft_dev_p2p_async(self, rows_ptr: int, cols_ptr: int, is_quot: bool, is_inv: bool, is_coset: bool):
        self._ck(self.lib.dp_fft_dev_p2p_async(self.h, rows_ptr, cols_ptr, int(is_quot), int(is_inv), int(is_coset)))

    def fft_dev_cols(self, cols_ptr: int):
        self._ck(self.lib.dp_fft_dev_cols(self.h, cols_ptr))

    def debug_set_limits(self, max_contig_log_k=11, max_strided_log_k=9, msm_window_bits=0):
        self._ck(self.lib.dp_debug_set_limits(self.h, max_contig_log_k, max_strided_log_k, msm_window_bits))

    def debug_set_three_pass(self, min_log_n: int):
        self._ck(self.lib.dp_debug_set_three_pass(self.h, min_log_n))

    def msm_breakdown(self):
        a, b, c = C.c_float(), C.c_float(), C.c_float()
        self.lib.dp_last_msm_breakdown(self.h, C.byref(a), C.byref(b), C.byref(c))
        return a.value, b.value, c.value

    def msm_tuning(self):
        """dp_init's choice between the plain MSM pipeline and batched-affine tree levels:
        {"plain_ms", "affine_ms", "levels", "equal"} (equal: 1 same result, 0 different, -1 not run)"""
        a, b, lv, eq = C.c_float(), C.c_float(), C.c_int(), C.c_int()
        self._ck(self.lib.dp_msm_tuning(self.h, C.byref(a), C.byref(b), C.byref(lv), C.byref(eq)))
        out = {"plain_ms": a.value, "affine_ms": b.value, "levels": lv.value, "equal": eq.value}
        allms = (C.c_float * 4)()
        self._ck(self.lib.dp_msm_tuning_all(self.h, allms))
        if any(v > 0 for v in allms):
            out["ms_by_levels"] = [round(float(v), 4) for v in allms]
        return out

    def gen_bases(self, seed: int, n: int) -> np.ndarray:
        out = np.zeros((n, G1_AFFINE_BYTES), dtype=np.uint8)
        self._ck(self.lib.dp_debug_gen_bases(self.h, seed, n, _addr(out) if n else None))
        return out

    def gen_bases_into(self, seed: int, n: int, out_ptr: int):
        """the same, written to `out_ptr` (n * 104 B of host or device memory)"""
        self._ck(self.lib.dp_debug_gen_bases(self.h, seed, n, out_ptr))

    @staticmethod
    def _tau_bytes(tau: int) -> bytes:
        if not 0 <= int(tau) < 1 << 256:
            raise ValueError("tau must be an integer in [0, 2^256); the library accepts 0 < tau < r")
        return int(tau).to_bytes(32, "little")

    def srs_powers_of_tau(self, tau: int, n: int) -> np.ndarray:
        """[n, 104] raw G1Affine: row i = tau^i * G1 (tau a canonical integer, 0 < tau < r)"""
        out = np.zeros((n, G1_AFFINE_BYTES), dtype=np.uint8)
        self._ck(self.lib.dp_srs_powers_of_tau(self.h, self._tau_bytes(tau), n, _addr(out) if n else None))
        return out

    def srs_powers_of_tau_into(self, tau: int, n: int, out_ptr: int):
        """the same, written to `out_ptr` (n * 104 B of host or device memory)"""
        self._ck(self.lib.dp_srs_powers_of_tau(self.h, self._tau_bytes(tau), n, out_ptr))

    # ---- verifier (none of these needs init)
    def g1_decompress(self, points48, check_subgroup: bool = True) -> np.ndarray:
        """[n, 48] ark-serialize compressed points -> [n, 104] raw G1Affine.  A rejected point raises DpError with
        `index` (the first bad point) and `why` (1 x >= p, 2 both flags, 3 no such point, 4 outside the subgroup)"""
        b = np.ascontiguousarray(points48, dtype=np.uint8).reshape(-1, G1_COMPRESSED_BYTES)
        n = b.shape[0]
        out = np.zeros((n, G1_AFFINE_BYTES), dtype=np.uint8)
        idx, why = C.c_size_t(), C.c_int()
        rc = self.lib.dp_g1_decompress(self.h, _addr(b) if n else None, n, int(check_subgroup), _addr(out) if n else None,
                                       C.byref(idx), C.byref(why))
        if rc != DP_OK:
            err = DpError(rc, (self.lib.dp_last_error(self.h) or b"").decode())
            err.index, err.why = idx.value, why.value
            raise err
        return out

    def msm_points(self, points104, scalars) -> np.ndarray:
        """sum scalars[i] * points[i]: [n, 104] raw G1Affine, [n, 4] u64 canonical scalars -> 144 B normalised Jacobian"""
        pts = np.ascontiguousarray(points104, dtype=np.uint8).reshape(-1, G1_AFFINE_BYTES)
        sc = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, 4)
        if pts.shape[0] != sc.shape[0]:
            raise ValueError(f"{pts.shape[0]} points but {sc.shape[0]} scalars")
        n = pts.shape[0]
        out = np.zeros(G1_PROJECTIVE_BYTES, dtype=np.uint8)
        self._ck(self.lib.dp_msm_points(self.h, _addr(pts) if n else None, _addr(sc) if n else None, n, _addr(out)))
        return out

    def srs_open_key(self, tau: int) -> np.ndarray:
        """[2, 200] raw G2Affine: H and tau * H (tau a canonical integer, 0 < tau < r)"""
        out = np.zeros((2, G2_AFFINE_BYTES), dtype=np.uint8)
        self._ck(self.lib.dp_srs_open_key(self.h, self._tau_bytes(tau), _addr(out)))
        return out

    def multi_pairing(self, g1_104, g2_200) -> np.ndarray:
        """prod e(P_i, Q_i) over [k, 104] raw G1Affine and [k, 200] raw G2Affine -> 576 B Fq12 (12 Montgomery Fq)"""
        p = np.ascontiguousarray(g1_104, dtype=np.uint8).reshape(-1, G1_AFFINE_BYTES)
        q = np.ascontiguousarray(g2_200, dtype=np.uint8).reshape(-1, G2_AFFINE_BYTES)
        if p.shape[0] != q.shape[0]:
            raise ValueError(f"{p.shape[0]} G1 points but {q.shape[0]} G2 points")
        k = p.shape[0]
        out = np.zeros(FQ12_BYTES, dtype=np.uint8)
        self._ck(self.lib.dp_multi_pairing(self.h, _addr(p) if k else None, _addr(q) if k else None, k, _addr(out)))
        return out

    # ---- setup files (only get_bases_compressed and srs_check need init)
    def g1_compress(self, points104) -> np.ndarray:
        """[n, 104] raw G1Affine -> [n, 48] ark-serialize compressed points (the inverse of g1_decompress)"""
        p = np.ascontiguousarray(points104, dtype=np.uint8).reshape(-1, G1_AFFINE_BYTES)
        n = p.shape[0]
        out = np.zeros((n, G1_COMPRESSED_BYTES), dtype=np.uint8)
        self._ck(self.lib.dp_g1_compress(self.h, _addr(p) if n else None, n, _addr(out) if n else None))
        return out

    def get_bases_compressed(self, start: int, n: int, out: np.ndarray | None = None) -> np.ndarray:
        """bases [start, start + n) as [n, 48] compressed points, into `out` when given"""
        if out is None:
            out = np.zeros((n, G1_COMPRESSED_BYTES), dtype=np.uint8)
        assert out.dtype == np.uint8 and out.size == n * G1_COMPRESSED_BYTES
        self._ck(self.lib.dp_get_bases_compressed(self.h, start, n, _addr(out) if n else None))
        return out

    def g2_compress(self, points200) -> np.ndarray:
        """[n, 200] raw G2Affine -> [n, 96] ark-serialize compressed points"""
        q = np.ascontiguousarray(points200, dtype=np.uint8).reshape(-1, G2_AFFINE_BYTES)
        n = q.shape[0]
        out = np.zeros((n, G2_COMPRESSED_BYTES), dtype=np.uint8)
        self._ck(self.lib.dp_g2_compress(self.h, _addr(q) if n else None, n, _addr(out) if n else None))
        return out

    def g2_decompress(self, points96, check_subgroup: bool = True) -> np.ndarray:
        """[n, 96] compressed points -> [n, 200] raw G2Affine.  A rejected point raises DpError with `index` and `why`
        (1 a coordinate >= p, 2 both flags, 3 no such point, 4 outside the subgroup), as g1_decompress does"""
        b = np.ascontiguousarray(points96, dtype=np.uint8).reshape(-1, G2_COMPRESSED_BYTES)
        n = b.shape[0]
        out = np.zeros((n, G2_AFFINE_BYTES), dtype=np.uint8)
        idx, why = C.c_size_t(), C.c_int()
        rc = self.lib.dp_g2_decompress(self.h, _addr(b) if n else None, n, int(check_subgroup), _addr(out) if n else None,
                                       C.byref(idx), C.byref(why))
        if rc != DP_OK:
            err = DpError(rc, (self.lib.dp_last_error(self.h) or b"").decode())
            err.index, err.why = idx.value, why.value
            raise err
        return out

    def srs_check(self, g2_400, seed: bytes | None = None) -> bool:
        """are the context's bases the powers of the tau of the open key (h, beta h: [2, 200] raw G2Affine)?  seed: 32 bytes
        that make the random scalars reproducible; None lets the library draw them from the operating system"""
        q = np.ascontiguousarray(g2_400, dtype=np.uint8).reshape(2, G2_AFFINE_BYTES)
        if seed is not None and len(seed) != 32:
            raise ValueError("the seed is 32 bytes")
        ok = C.c_int()
        self._ck(self.lib.dp_srs_check(self.h, _addr(q), bytes(seed) if seed is not None else None, C.byref(ok)))
        return bool(ok.value)

    def last_srs_check(self) -> dict:
        """the last srs_check: {"scalars_ms", "msm_ms", "pairing_ms"} and its two MSM results "A", "B" (144 B each)"""
        a, b, c = C.c_float(), C.c_float(), C.c_float()
        ab = np.zeros((2, G1_PROJECTIVE_BYTES), dtype=np.uint8)
        self._ck(self.lib.dp_last_srs_check(self.h, C.byref(a), C.byref(b), C.byref(c), _addr(ab)))
        return {"scalars_ms": a.value, "msm_ms": b.value, "pairing_ms": c.value, "A": ab[0], "B": ab[1]}

    def srs_update(self, g2_400, n: int, secret: int | None = None, out48=None, plain: bool = False):
        """one ceremony contribution over the n resident bases (dp_srs_update): returns (the [n, 48] compressed points
        s^i P_i, [2, 200] raw G2Affine s h, s beta h).  g2_400 = h, beta h.  secret None lets the library draw s; out48:
        an [n, 48] uint8 array (a memory map of a file, say) or a device address to write the points to instead.  plain:
        dp_debug_srs_update_plain, the reference method"""
        q = np.ascontiguousarray(g2_400, dtype=np.uint8).reshape(2, G2_AFFINE_BYTES)
        g2 = np.zeros((2, G2_AFFINE_BYTES), dtype=np.uint8)
        if out48 is None:
            out48 = np.zeros((n, G1_COMPRESSED_BYTES), dtype=np.uint8)
        elif not isinstance(out48, int):
            assert out48.dtype == np.uint8 and out48.size == n * G1_COMPRESSED_BYTES and out48.flags["C_CONTIGUOUS"]
        s = self._tau_bytes(secret) if secret is not None else None
        f = self.lib.dp_debug_srs_update_plain if plain else self.lib.dp_srs_update
        self._ck(f(self.h, s, _addr(q), _addr(out48), _addr(g2)))
        return out48, g2

    def init_ptr(self, bases_ptr: int, n_bases: int, domain_size: int, quot_domain_size: int):
        """PlonkSlave.init with the raw GroupAffine array at `bases_ptr` (host or device memory)"""
        self._ck(self.lib.dp_init(self.h, bases_ptr if n_bases else None, n_bases, domain_size, quot_domain_size))

    def sync(self):
        self._ck(self.lib.dp_sync(self.h))

    def last_timing(self):
        ms, n = C.c_float(), C.c_uint64()
        self.lib.dp_last_timing(self.h, C.byref(ms), C.byref(n))
        return ms.value, n.value

    def launch_count(self) -> int:
        return int(self.lib.dp_launch_count(self.h))
