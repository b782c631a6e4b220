// jslpsolver_b200/csrc/jslp_sensitivity.cuh -- ratio-test bounds of a solved LP for its sensitivity report
// (included by jslp_api.cu).  DESIGN.md section 2b gives the definitions; the host applies the signs of the objective
// sense and of each row.  With P the tableau precision and only rows 1 .. H-1 read:
//
//   column c (a non-basic variable), over rows r whose basic variable is restricted:
//     col_lo[c] = max of -M[r,0] / M[r,c] over M[r,c] >  P        col_hi[c] = min of the same over M[r,c] < -P
//   row r (a basic variable), over columns c >= 1:
//     row_lo[r] = max of  M[0,c] / M[r,c] over M[r,c] >  P        row_hi[r] = min of the same over M[r,c] < -P
//     for restricted columns; an unrestricted column with |M[r,c]| > P offers 0 to both.
//
// Every quotient is one IEEE division, normalised to +0 when it is -0 (a NaN one, from non-finite entries, takes no
// part), and reduced as an order-preserving integer key (dkey) with max / min, which do not depend on the order rows
// and columns are visited in: the result is the same for every grid.  An empty set leaves the identity key, read back as -inf (lo) / +inf (hi).
#pragma once

namespace jslp {

static constexpr int SENS_PAIRS = 4;                 // column pairs per lane
static constexpr int SENS_COLS = 2 * 32 * SENS_PAIRS;  // columns per warp pass over a row (one grid column)
static constexpr unsigned long long SENS_LO_NONE = 0ull, SENS_HI_NONE = ~0ull;

__device__ __forceinline__ unsigned long long warp_max_key(unsigned long long k) {
    const unsigned int hi = __reduce_max_sync(0xffffffffu, (unsigned int)(k >> 32));
    const unsigned int lo = __reduce_max_sync(0xffffffffu, (unsigned int)(k >> 32) == hi ? (unsigned int)k : 0u);
    return ((unsigned long long)hi << 32) | lo;
}
__device__ __forceinline__ unsigned long long warp_min_key(unsigned long long k) {
    const unsigned int hi = __reduce_min_sync(0xffffffffu, (unsigned int)(k >> 32));
    const unsigned int lo = __reduce_min_sync(0xffffffffu, (unsigned int)(k >> 32) == hi ? (unsigned int)k : 0xffffffffu);
    return ((unsigned long long)hi << 32) | lo;
}

// Grid (row blocks, column blocks of SENS_COLS).  Warp w of CTA b reads rows 1 + 8 b + w, stepping by 8 gridDim.x, over
// the columns of blockIdx.y with 128-bit no-allocate loads (lane l: column pairs l + 32 j); each entry is read once.
// Row keys are reduced over the warp and merged across column blocks with atomics; column keys are merged over the
// CTA in shared memory, then across row blocks with atomics.  keys_lo / keys_hi: [0, W) columns, [W, W + H) rows,
// set to SENS_LO_NONE / SENS_HI_NONE before the launch.
__global__ void __launch_bounds__(256) k_sensitivity(const TabDev *Tp, unsigned long long *keys_lo,
                                                     unsigned long long *keys_hi) {
    __shared__ unsigned long long s_lo[SENS_COLS], s_hi[SENS_COLS];
    const TabDev T = *Tp;
    const int W = T.W, H = T.H;
    const double P = T.prec;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int pair0 = blockIdx.y * (SENS_COLS / 2) + lane;
    for (int i = threadIdx.x; i < SENS_COLS; i += blockDim.x) { s_lo[i] = SENS_LO_NONE; s_hi[i] = SENS_HI_NONE; }

    double cost[2 * SENS_PAIRS];
    bool live[2 * SENS_PAIRS], unr[2 * SENS_PAIRS];
    unsigned long long clo[2 * SENS_PAIRS], chi[2 * SENS_PAIRS];
#pragma unroll
    for (int k = 0; k < 2 * SENS_PAIRS; k++) {
        const int c = 2 * (pair0 + 32 * (k >> 1)) + (k & 1);
        live[k] = c >= 1 && c < W;
        cost[k] = live[k] ? T.M[c] : 0.0;
        unr[k] = live[k] && is_unres(T, T.vcol[c]);
        clo[k] = SENS_LO_NONE;
        chi[k] = SENS_HI_NONE;
    }
    __syncthreads();

    for (int r = 1 + blockIdx.x * nwarps + warp; r < H; r += gridDim.x * nwarps) {
        const double *row = T.M + (size_t)r * T.stride;
        double2 v[SENS_PAIRS];
#pragma unroll
        for (int j = 0; j < SENS_PAIRS; j++) {
            const int p = pair0 + 32 * j;
            v[j] = 2 * p < W ? ld_v2_dead(row + 2 * p) : make_double2(0.0, 0.0);
        }
        const double nrhs = -row[0];
        const bool restricted_row = !is_unres(T, T.vrow[r]);
        unsigned long long rlo = SENS_LO_NONE, rhi = SENS_HI_NONE;
#pragma unroll
        for (int k = 0; k < 2 * SENS_PAIRS; k++) {
            const double x = (k & 1) ? v[k >> 1].y : v[k >> 1].x;
            const bool pos = x > P, neg = x < -P;
            if (!live[k] || !(pos || neg)) continue;
            if (restricted_row) {
                const double q = __ddiv_rn(nrhs, x);
                if (q == q) {
                    if (pos) clo[k] = max(clo[k], dkey(q)); else chi[k] = min(chi[k], dkey(q));
                }
            }
            if (unr[k]) {
                const unsigned long long z = dkey(0.0);
                rlo = max(rlo, z);
                rhi = min(rhi, z);
            } else {
                const double q = __ddiv_rn(cost[k], x);
                if (q == q) {
                    if (pos) rlo = max(rlo, dkey(q)); else rhi = min(rhi, dkey(q));
                }
            }
        }
        rlo = warp_max_key(rlo);
        rhi = warp_min_key(rhi);
        if (lane == 0) {
            if (rlo != SENS_LO_NONE) atomicMax(keys_lo + W + r, rlo);
            if (rhi != SENS_HI_NONE) atomicMin(keys_hi + W + r, rhi);
        }
    }

#pragma unroll
    for (int k = 0; k < 2 * SENS_PAIRS; k++) {
        const int i = 2 * (lane + 32 * (k >> 1)) + (k & 1);
        if (clo[k] != SENS_LO_NONE) atomicMax(s_lo + i, clo[k]);
        if (chi[k] != SENS_HI_NONE) atomicMin(s_hi + i, chi[k]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < SENS_COLS; i += blockDim.x) {
        const int c = blockIdx.y * SENS_COLS + i;
        if (c >= W) break;
        if (s_lo[i] != SENS_LO_NONE) atomicMax(keys_lo + c, s_lo[i]);
        if (s_hi[i] != SENS_HI_NONE) atomicMin(keys_hi + c, s_hi[i]);
    }
}

}  // namespace jslp

static double sens_key_value(unsigned long long k, double none) {
    if (k == jslp::SENS_LO_NONE || k == jslp::SENS_HI_NONE) return none;
    const unsigned long long b = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;  // dkey_inv
    double v;
    memcpy(&v, &b, sizeof v);
    return v;
}

extern "C" int jslp_sensitivity(jslp_tab *t, double *col_lo, double *col_hi, double *row_lo, double *row_hi) {
    if (!t || !col_lo || !col_hi || !row_lo || !row_hi) return fail(JSLP_E_INVALID, "NULL argument");
    CK(cudaSetDevice(t->ctx->device));
    cudaStream_t s = t->ctx->stream;
    const int W = t->W, H = t->H;
    const size_t n = (size_t)W + H;
    if (n > t->sens_cap) {
        cudaFree(t->d_sens);
        t->d_sens = nullptr;
        t->sens_cap = 0;
        CK(cudaMalloc(&t->d_sens, 2 * n * sizeof(unsigned long long)));
        t->sens_cap = n;
    }
    unsigned long long *lo = t->d_sens, *hi = t->d_sens + n;
    CK(cudaMemsetAsync(lo, 0x00, n * sizeof(unsigned long long), s));  // SENS_LO_NONE
    CK(cudaMemsetAsync(hi, 0xff, n * sizeof(unsigned long long), s));  // SENS_HI_NONE
    // about two CTAs per SM over the whole grid, never more row blocks than there are 8-row groups
    const int col_blocks = (W + SENS_COLS - 1) / SENS_COLS;
    const int row_groups = std::max(1, (H - 1 + 7) / 8);
    const int row_blocks = std::max(1, std::min(row_groups, t->ctx->num_sms * 2 / col_blocks));
    k_sensitivity<<<dim3(row_blocks, col_blocks), 256, 0, s>>>(t->d_T, lo, hi);
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    std::vector<unsigned long long> keys(2 * n);
    CK(cudaMemcpyAsync(keys.data(), t->d_sens, 2 * n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    for (int c = 0; c < W; c++) {
        col_lo[c] = sens_key_value(keys[c], -INFINITY);
        col_hi[c] = sens_key_value(keys[n + c], INFINITY);
    }
    for (int r = 0; r < H; r++) {
        row_lo[r] = sens_key_value(keys[W + r], -INFINITY);
        row_hi[r] = sens_key_value(keys[n + W + r], INFINITY);
    }
    return JSLP_OK;
}
