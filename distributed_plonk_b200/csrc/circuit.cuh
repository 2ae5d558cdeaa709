// Circuit preprocessing and the witness gather on the GPU: what jf-plonk's preprocessing and the reference's dispatcher
// build on the CPU from a circuit before round 1.
//
// A slot is s = i * n + j: wire type i, gate j (wire_permutation[i * n + j], dispatcher2.rs:340).
//   wire permutation  succ(s) = the next slot, in increasing slot order, holding the same variable; the last slot of a
//                     variable wraps to its first.  These are the cycles of jf-relation's compute_wire_permutation
//                     (variable_wires_map[var].push((wire, gate)) wire-major, then windows(2) with the first element
//                     re-appended) [3P-recall].  Built by a stable LSD radix sort of (variable, slot) keyed by the
//                     variable - 8-bit digits, only as many passes as the bit width of num_vars - 1 needs - then one
//                     successor kernel.  Every pass is reduce-then-scan (block histograms, an exclusive scan of them,
//                     a stable scatter with in-block ranks): no block ever waits for another.
//   perm evals        id[i n + j] = k_i * omega_n^j,  sigma[s] = id[succ(s)]   (dispatcher2.rs:340-342)
//   witness gather    wires[s] = witness[vars[s]],  pub[j] = wires[(T - 1) n + j] for j < num_inputs, else 0
//                     (dispatcher2.rs:299, 337; the output wire of the first num_inputs gates [3P-recall])
#pragma once
#include "msm.cuh"
#include "ntt.cuh"

namespace dp {

constexpr int CIRC_TPB = 256;                       // threads per block; also the radix (one digit per thread)
constexpr int CIRC_ITEMS = 8;
constexpr int CIRC_TILE = CIRC_TPB * CIRC_ITEMS;    // elements per sort block
constexpr uint32_t CIRC_RADIX_BITS = 8;
constexpr uint32_t CIRC_RADIX = 1u << CIRC_RADIX_BITS;
static_assert(CIRC_RADIX == CIRC_TPB, "one digit per thread in the histogram and offset steps");

// *flag |= 1 when some ids[i] >= bound (variable ids against num_vars, successor slots against the slot count)
__global__ void circ_check_ids_kernel(const uint32_t *ids, uint64_t count, uint64_t bound, uint32_t *flag) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (uint64_t)gridDim.x * blockDim.x)
        if (ids[i] >= bound) atomicOr(flag, 1u);
}

// digit counts of one tile: hist[d * n_blocks + block] (digit-major, so that the exclusive scan of the whole array gives
// each (digit, block) its first output position, blocks of one digit in order: the scatter is stable)
__global__ void __launch_bounds__(CIRC_TPB) circ_radix_hist_kernel(const uint32_t *keys, uint64_t count, uint32_t shift,
                                                                    uint32_t n_blocks, uint32_t *hist) {
    __shared__ uint32_t h[CIRC_RADIX];
    h[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t base = (uint64_t)blockIdx.x * CIRC_TILE;
    for (int r = 0; r < CIRC_ITEMS; r++) {
        const uint64_t idx = base + (uint64_t)r * CIRC_TPB + threadIdx.x;
        if (idx < count) atomicAdd(&h[(keys[idx] >> shift) & (CIRC_RADIX - 1)], 1u);
    }
    __syncthreads();
    hist[(uint64_t)threadIdx.x * n_blocks + blockIdx.x] = h[threadIdx.x];
}

// exclusive scan of n u32 in place: block sums (scan_block_sums_kernel of msm.cuh), one block scans those
// (circ_scan_offsets_kernel), then every block rescans its tile from its offset
__global__ void __launch_bounds__(CIRC_TPB) circ_scan_offsets_kernel(uint32_t *block_sums, uint32_t n_blocks) {
    __shared__ uint32_t sh[CIRC_TPB];
    uint32_t run = 0;
    for (uint32_t base = 0; base < n_blocks; base += CIRC_TPB) {
        const uint32_t i = base + threadIdx.x;
        uint32_t total;
        const uint32_t e = block_exclusive_scan(i < n_blocks ? block_sums[i] : 0u, sh, total);
        if (i < n_blocks) block_sums[i] = run + e;
        run += total;
    }
}

__global__ void __launch_bounds__(SCAN_TPB) circ_scan_write_kernel(uint32_t *x, uint32_t n, const uint32_t *block_offsets) {
    __shared__ uint32_t sh[SCAN_TPB];
    const uint32_t base = blockIdx.x * SCAN_BLOCK + threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS], a = 0;
    for (int k = 0; k < SCAN_ITEMS; k++) {
        v[k] = base + k < n ? x[base + k] : 0u;
        a += v[k];
    }
    uint32_t total;
    uint32_t run = block_offsets[blockIdx.x] + block_exclusive_scan(a, sh, total);
    for (int k = 0; k < SCAN_ITEMS; k++)
        if (base + k < n) {
            x[base + k] = run;
            run += v[k];
        }
}

// Stable scatter of one tile by the digit at `shift`.  The tile is walked in CIRC_ITEMS rounds of CIRC_TPB consecutive
// elements; inside a round an element's rank is the number of lower lanes of its warp with the same digit (32 broadcast
// reads of shared memory) plus the counts of that digit in the lower warps, on top of what earlier rounds placed.
// vals == nullptr: the values are the element indices (the slots of the first pass).
__global__ void __launch_bounds__(CIRC_TPB) circ_radix_scatter_kernel(const uint32_t *keys_in, const uint32_t *vals_in, uint64_t count,
                                                                       uint32_t shift, const uint32_t *offsets, uint32_t n_blocks,
                                                                       uint32_t *keys_out, uint32_t *vals_out) {
    constexpr int WARPS = CIRC_TPB / 32;
    __shared__ uint32_t run[CIRC_RADIX];             // next output position of each digit
    __shared__ uint32_t wcnt[WARPS][CIRC_RADIX];     // this round: elements of each digit in each warp
    __shared__ uint32_t dig[CIRC_TPB];
    const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    run[tid] = offsets[(uint64_t)tid * n_blocks + blockIdx.x];
    for (int w = 0; w < WARPS; w++) wcnt[w][tid] = 0;
    const uint64_t base = (uint64_t)blockIdx.x * CIRC_TILE;
    for (int r = 0; r < CIRC_ITEMS; r++) {
        const uint64_t idx = base + (uint64_t)r * CIRC_TPB + tid;
        const bool valid = idx < count;
        const uint32_t key = valid ? keys_in[idx] : 0u;
        const uint32_t val = valid ? (vals_in ? vals_in[idx] : (uint32_t)idx) : 0u;
        const uint32_t d = valid ? (key >> shift) & (CIRC_RADIX - 1) : CIRC_RADIX;   // CIRC_RADIX: no element
        dig[tid] = d;
        __syncthreads();
        uint32_t rank = 0;
        bool last = true;
        for (uint32_t l = 0; l < 32; l++) {
            if (dig[(warp << 5) + l] != d) continue;
            if (l < lane) rank++;
            else if (l > lane) last = false;
        }
        if (valid && last) wcnt[warp][d] = rank + 1;
        __syncthreads();
        if (valid) {
            uint32_t pos = run[d] + rank;
            for (uint32_t w = 0; w < warp; w++) pos += wcnt[w][d];
            keys_out[pos] = key;
            vals_out[pos] = val;
        }
        __syncthreads();
        uint32_t tot = 0;
        for (int w = 0; w < WARPS; w++) {
            tot += wcnt[w][tid];
            wcnt[w][tid] = 0;
        }
        run[tid] += tot;
        __syncthreads();
    }
}

// succ[vals[p]] = vals[p + 1] inside a group of equal keys, and the group's first value for its last element (found by a
// binary search for the first occurrence of the key).  vals == nullptr: the identity (no sort pass ran: one variable).
__global__ void circ_successor_kernel(const uint32_t *keys, const uint32_t *vals, uint64_t count, uint32_t *succ) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= count) return;
    const uint32_t k = keys[p];
    uint64_t q;
    if (p + 1 < count && keys[p + 1] == k) {
        q = p + 1;
    } else {
        uint64_t lo = 0, hi = p;
        while (lo < hi) {
            const uint64_t mid = (lo + hi) >> 1;
            if (keys[mid] < k) lo = mid + 1;
            else hi = mid;
        }
        q = lo;
    }
    succ[vals ? vals[p] : p] = vals ? vals[q] : (uint32_t)q;
}

struct CircK {
    Fr k[5];
};

// omega_n^j from the half table H (omega^e, e < n/2; omega^(n/2) = -1)
DP_D Fr circ_omega_pow(const Fr *H, uint64_t n, uint64_t j) {
    const uint64_t half = n >> 1;
    if (half == 0) return Fr::one();
    return j < half ? gmem_ld(H + j) : Fr::zero() - gmem_ld(H + (j - half));
}

// id[s] = k_(s / n) * omega^(s mod n); sigma[s] = id[succ[s]] (= id[s] without succ).  succ entries are checked < count
// before the launch.
__global__ void circ_perm_evals_kernel(const uint32_t *succ, uint64_t count, uint32_t log_n, const Fr *H, CircK k, Fr *id_out,
                                       Fr *sigma_out) {
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= count) return;
    const uint64_t n = (uint64_t)1 << log_n;
    const Fr id = k.k[s >> log_n] * circ_omega_pow(H, n, s & (n - 1));
    gmem_st(id_out + s, id);
    if (succ) {
        const uint64_t t = succ[s];
        gmem_st(sigma_out + s, k.k[t >> log_n] * circ_omega_pow(H, n, t & (n - 1)));
    } else {
        gmem_st(sigma_out + s, id);
    }
}

// wires[s] = witness[vars[s]] (s < count); pub[j] = witness[vars[pub_first + j]] for j < num_inputs, 0 for
// num_inputs <= j < n.  Variable ids are checked < num_vars before the launch.
__global__ void circ_gather_kernel(const Fr *witness, const uint32_t *vars, uint64_t count, uint64_t n, uint64_t pub_first,
                                   uint64_t num_inputs, Fr *wires, Fr *pub) {
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s < count) gmem_st(wires + s, gmem_ld(witness + vars[s]));
    if (s < n) gmem_st(pub + s, s < num_inputs ? gmem_ld(witness + vars[pub_first + s]) : Fr::zero());
}

// canonical -> Montgomery in place (undoes fr_into_repr_kernel)
__global__ void fr_to_mont_kernel(Fr *x, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) gmem_st(x + i, gmem_ld(x + i).to_mont());
}

}  // namespace dp
