// jslpsolver_b200/csrc/jslp_elastic.cuh -- the elastic tableau of an infeasible LP: every relaxable row gets a
// violation variable of its own, the rows that start infeasible are crashed onto it, and row 0 is the weighted total
// violation priced against that crash basis (included by jslp_api.cu after jslp_lex.cuh; no reference counterpart).
// DESIGN.md section 2k is the contract; in short, with M the uploaded, never pivoted tableau (H x W), P its precision,
// r_1 < ... < r_k the relaxable rows with weights w_j > 0 and l* = max(n_index, lastElementIndex):
//
//   column W+j is e_j; it enters row r_j as -1, relaxing the stored row s.a.x <= s.rhs to s.a.x <= s.rhs + e_j
//   row r_j is crashed iff M[r_j,0] < -P: E[r_j,c] = M[r_j,c] with the sign bit flipped (column 0 included), its
//     elastic entry stays -1, vrow'[r_j] = l*+j and vcol'[W+j] = vrow[r_j] (e_j basic, the slack non-basic)
//   every other row is M's row bit for bit; elastic entries are -1 on the row's own column and +0 elsewhere
//   vcol'[W+j] = l*+j for a row that is not crashed; padding +0
//   E[0,c] = sum over crashed j of w_j * E[r_j,c] for every column but the elastic columns of rows not crashed, which
//     get -w_j: one IEEE multiply per term, added in row order within tiles of ELASTIC_TILE_ROWS rows (rows 1.. on)
//     from +0, then the tile partials added in tile order from +0
//
// E starts primal feasible wherever every row that starts below -P may be relaxed, so minimising the violation is a
// phase 2 from the crash basis.  k_elastic_rows writes rows 1..H-1, the labels and one row-0 partial per row tile and
// column; k_elastic_cost adds the partials in tile order into row 0.  Only the crash count leaves the device.
#pragma once

namespace jslp {

static constexpr int ELASTIC_TILE_ROWS = 32;  // rows per CTA of k_elastic_rows, and the terms of one row-0 partial
static constexpr int ELASTIC_COLS = 256;      // columns of E's stride per CTA (one thread per column)

// What the two kernels read besides the parent: jof[r] = j for row r_j, -1 for a row that may not be relaxed (H
// entries); rows[j] = r_j and w[j] (k entries); and what they write on the side: crashed[j] (k entries), the crash
// count and the row-0 partials (tiles x estride).
struct ElasticArgs {
    const int *jof, *rows;
    const double *w;
    int *crashed, *count;
    double *part;
    double *E;
    int *vrow, *vcol;
    int k, estride, label;
};

// Rows 1..H-1 of E, vrow' and vcol' and the row-0 partials.  Grid: (estride / ELASTIC_COLS, row tiles); tile y covers
// rows 1 + y*ELASTIC_TILE_ROWS .. on.  Every element of those rows, the padding included, is written once, and each
// partial is one thread's running sum in row order, so the grid does not change a bit of the result.
__global__ void __launch_bounds__(ELASTIC_COLS) k_elastic_rows(const TabDev *Tp, ElasticArgs a) {
    __shared__ int s_j[ELASTIC_TILE_ROWS];
    __shared__ double s_w[ELASTIC_TILE_ROWS];   // w_j of a crashed row, 0 for any other
    __shared__ unsigned s_flip[ELASTIC_TILE_ROWS];
    const TabDev &T = *Tp;
    const int W = T.W, H = T.H;
    const size_t stride = (size_t)T.stride;
    const double *M = T.M;  // whichever ping-pong buffer the device calls current
    const int tid = threadIdx.x;
    const int r0 = 1 + blockIdx.y * ELASTIC_TILE_ROWS;
    const int nr = min(ELASTIC_TILE_ROWS, H - r0);
    if (tid < nr) {
        const int r = r0 + tid;
        const int j = a.jof[r];
        const bool crash = j >= 0 && ldg_cg(M + (size_t)r * stride) < -T.prec;
        s_j[tid] = j;
        s_w[tid] = crash ? a.w[j] : 0.0;
        s_flip[tid] = crash;
        if (blockIdx.x == 0) {
            a.vrow[r] = crash ? a.label + j : T.vrow[r];
            if (j >= 0) a.crashed[j] = crash;
            if (crash) atomicAdd(a.count, 1);
        }
    }
    __syncthreads();
    const int c = blockIdx.x * ELASTIC_COLS + tid;
    if (c >= a.estride) return;
    const int je = c - W;  // the elastic column's j, when W <= c < W + k
    double acc = 0.0;
    for (int i = 0; i < nr; i++) {
        const int r = r0 + i;
        double v;
        if (c < W) {
            v = ldg_cg(M + (size_t)r * stride + c);
            if (s_flip[i])  // the IEEE sign flip itself, so no NaN is quietened or rewritten on the way
                v = __longlong_as_double(__double_as_longlong(v) ^ (long long)(1ull << 63));
        } else {
            v = (je < a.k && s_j[i] == je) ? -1.0 : 0.0;
        }
        a.E[(size_t)r * a.estride + c] = v;
        if (s_flip[i] && c < W + a.k) acc = acc + s_w[i] * v;
    }
    a.part[(size_t)blockIdx.y * a.estride + c] = acc;
    if (blockIdx.y == 0) {
        if (c == 0) a.vrow[0] = T.vrow[0];
        if (c < W) {
            a.vcol[c] = T.vcol[c];
        } else if (je < a.k) {
            const int r = a.rows[je];
            const bool crash = ldg_cg(M + (size_t)r * stride) < -T.prec;
            a.vcol[c] = crash ? T.vrow[r] : a.label + je;
        }
    }
}

// Row 0 of E: the partials of column c added in tile order from +0, -w_j at the elastic column of a row that is not
// crashed, +0 in the padding.  One thread per column of the stride.
__global__ void __launch_bounds__(ELASTIC_COLS) k_elastic_cost(int W, int tiles, ElasticArgs a) {
    const int c = blockIdx.x * ELASTIC_COLS + threadIdx.x;
    if (c >= a.estride) return;
    const int je = c - W;
    double v = 0.0;
    if (je >= a.k) {
        v = 0.0;
    } else if (je >= 0 && !a.crashed[je]) {
        v = -a.w[je];
    } else {
        for (int y = 0; y < tiles; y++) v = v + a.part[(size_t)y * a.estride + c];
    }
    a.E[c] = v;
}

}  // namespace jslp

extern "C" int jslp_elastic_create(jslp_tab *t, const int32_t *rows, const double *weights, int n_rows,
                                   jslp_tab **out, int32_t *n_crashed) {
    if (!t || !out || !n_crashed || (n_rows > 0 && (!rows || !weights))) return fail(JSLP_E_INVALID, "NULL argument");
    *out = nullptr;
    *n_crashed = 0;
    if (n_rows < 0) return fail(JSLP_E_INVALID, "elastic_create: negative row count");
    if (t->nOpt > 0) return fail(JSLP_E_INVALID, "elastic_create: optional objectives are not supported");
    const int W = t->W, H = t->H, k = n_rows;
    for (int j = 0; j < k; j++) {
        if (rows[j] < 1 || rows[j] >= H || (j > 0 && rows[j] <= rows[j - 1]))
            return fail(JSLP_E_INVALID, "elastic_create: rows must be increasing and within 1..H-1");
        if (!(weights[j] > 0.0) || std::isinf(weights[j]))
            return fail(JSLP_E_INVALID, "elastic_create: every weight must be finite and > 0");
    }
    jslp_ctx *ctx = t->ctx;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    // a relaxable row must still hold its own constraint: its basic label is the one it was uploaded with
    std::vector<int> vrow((size_t)H);
    CK(cudaMemcpyAsync(vrow.data(), t->hd.vrow, sizeof(int) * (size_t)H, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    for (int j = 0; j < k; j++) {
        const int r = rows[j];
        if (r >= (int)t->h_vrow_upload.size() || vrow[r] != t->h_vrow_upload[r])
            return fail(JSLP_E_INVALID, "elastic_create: row " + std::to_string(r) +
                                            " does not have its own slack basic (the tab must be as uploaded)");
    }
    const int label = first_free_label(t);
    const int tiles = (H - 1 + ELASTIC_TILE_ROWS - 1) / ELASTIC_TILE_ROWS;
    TabOwner e;
    int rc = sibling_create(t, W + k, H, k, e);  // cut rows would take labels after l*+k-1
    if (rc) return rc;
    const int estride = e->stride;
    // one scratch block: w[k] and part[tiles x estride] (doubles), then jof[H], rows[k], crashed[k], count (ints)
    const size_t n_dbl = (size_t)k + (size_t)std::max(tiles, 1) * estride;
    const size_t n_int = (size_t)H + 2 * (size_t)k + 1;
    void *d_buf = nullptr;
    CK(cudaMalloc(&d_buf, sizeof(double) * n_dbl + sizeof(int) * n_int));
    const std::unique_ptr<void, DevFree> buf(d_buf);
    ElasticArgs a;
    double *d_w = (double *)d_buf;
    a.w = d_w;
    a.part = d_w + k;
    int *d_jof = (int *)(d_w + n_dbl);
    a.jof = d_jof;
    a.rows = d_jof + H;
    a.crashed = d_jof + H + k;
    a.count = d_jof + H + 2 * k;
    a.E = e->hd.M; a.vrow = e->hd.vrow; a.vcol = e->hd.vcol;
    a.k = k; a.estride = estride; a.label = label;
    std::vector<int> ints(n_int, -1);
    for (int j = 0; j < k; j++) {
        ints[(size_t)rows[j]] = j;
        ints[(size_t)H + j] = rows[j];
    }
    ints[n_int - 1] = 0;
    CK(cudaMemcpyAsync(d_jof, ints.data(), sizeof(int) * n_int, cudaMemcpyHostToDevice, s));
    if (k > 0) CK(cudaMemcpyAsync(d_w, weights, sizeof(double) * (size_t)k, cudaMemcpyHostToDevice, s));
    if (tiles > 0) {
        const dim3 grid((unsigned)(estride / ELASTIC_COLS + (estride % ELASTIC_COLS != 0)), (unsigned)tiles);
        k_elastic_rows<<<grid, ELASTIC_COLS, 0, s>>>(t->d_T, a);
        ctx->launches += 1;
        CK(cudaGetLastError());
    } else {  // no row below the cost row: only the labels of row 0 and the columns
        CK(cudaMemcpyAsync(e->hd.vrow, t->hd.vrow, sizeof(int), cudaMemcpyDeviceToDevice, s));
        CK(cudaMemcpyAsync(e->hd.vcol, t->hd.vcol, sizeof(int) * (size_t)W, cudaMemcpyDeviceToDevice, s));
    }
    k_elastic_cost<<<(estride + ELASTIC_COLS - 1) / ELASTIC_COLS, ELASTIC_COLS, 0, s>>>(W, tiles, a);
    ctx->launches += 1;
    CK(cudaGetLastError());
    int crashed = 0;  // *n_crashed stays 0 unless the call succeeds
    CK(cudaMemcpyAsync(&crashed, a.count, sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    *n_crashed = crashed;
    *out = e.release();
    return JSLP_OK;
}
