// jslpsolver_b200/csrc/jslp_cone.cuh -- the recession cone of an uploaded LP and batched solves of its column
// subsets (included by jslp_api.cu after jslp_elastic.cuh; no reference counterpart).  DESIGN.md section 2l is the
// contract; in short, with M the uploaded, never pivoted tableau (H x W) and l* = max(n_index, lastElementIndex):
//
//   K ((H+1) x W, M's stride rounded as jslp_tab_create rounds it): rows 0..H-1 = M's rows bit for bit, except that
//     column 0 is +0 in every one of them; row H = 1.0 at column 0 and at every column 1..W-1, +0 padding
//   vrow' = (vrow..., l*), vcol' = vcol; l* restricted and not integer
//
// Row H is the normalisation sum_j d_j <= 1, so K is a bounded LP whose slack basis is primal feasible: its phase 1
// finds no leaving row, and its phase 2 finds an improving direction d >= 0 of M (every row's activity rate at most 0
// towards its bound, objective rate > 0) exactly when the optimum M[0,0] is non-zero.  Capping the variables of a set
// S is dropping their columns: jslp_column_batch writes +0 over them in every row, row 0 included, so they price at 0
// and never enter.  Rows 0..H-1 are one device-to-device copy; k_cone_rows writes column 0, row H and the new label.
#pragma once

namespace jslp {

static constexpr int CONE_THREADS = 256;

// Column 0 of rows 0..H-1 (+0) and row H of K (1.0 at columns 0..W-1, +0 padding), and vrow'[H].  Grid: max(H,
// kstride) threads, so every element written here is written exactly once.
__global__ void __launch_bounds__(CONE_THREADS) k_cone_rows(double *K, int kstride, int W, int H, int *vrow_out,
                                                            int label) {
    const int i = blockIdx.x * CONE_THREADS + threadIdx.x;
    if (i < H) K[(size_t)i * kstride] = 0.0;
    if (i < kstride) K[(size_t)H * kstride + i] = i < W ? 1.0 : 0.0;
    if (i == 0) vrow_out[H] = label;
}

// +0 over every column 1..W-1 whose bit is clear in keep, in every row of the current buffer (the HBM path of
// jslp_column_batch).  One CTA per row, grid-strided.
__global__ void __launch_bounds__(CONE_THREADS) k_zero_columns(const TabDev *Tp, const uint32_t *keep) {
    const TabDev &T = *Tp;
    for (int r = blockIdx.x; r < T.H; r += gridDim.x) {
        double *row = T.M + (size_t)r * T.stride;
        for (int c = 1 + threadIdx.x; c < T.W; c += CONE_THREADS)
            if (!((keep[c >> 5] >> (c & 31)) & 1u)) row[c] = 0.0;
    }
}

}  // namespace jslp

extern "C" int jslp_cone_create(jslp_tab *t, jslp_tab **out) {
    if (!t || !out) return fail(JSLP_E_INVALID, "NULL argument");
    *out = nullptr;
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, "cone_create: optional objectives are not supported");
    jslp_ctx *ctx = t->ctx;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const int W = t->W, H = t->H;
    const int label = first_free_label(t);
    TabOwner k;
    int rc = sibling_create(t, W, H + 1, 1, k);
    if (rc) return rc;
    rc = sibling_copy_rows(t, k.get(), 0);
    if (rc) return rc;
    const int n = std::max(H, k->stride);
    k_cone_rows<<<(n + CONE_THREADS - 1) / CONE_THREADS, CONE_THREADS, 0, s>>>(k->hd.M, k->stride, W, H, k->hd.vrow,
                                                                              label);
    ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(s));
    *out = k.release();
    return JSLP_OK;
}

enum { COL_OPTIMAL = 0, COL_UNBOUNDED = 1, COL_CYCLED = 2, COL_INFEASIBLE = 3 };

// One set on the HBM path: restore the snapshot, zero its columns, simplex() with the cycle check on.
static int column_hbm(jslp_tab *t, const uint32_t *bits, int words, int32_t *status, double *eval_raw, int32_t *pivots,
                      double *rhs, int32_t *vrow) {
    cudaStream_t s = t->ctx->stream;
    int rc = jslp_restore(t);
    if (rc) return rc;
    rc = batch_scratch(t, sizeof(uint32_t) * (size_t)words);
    if (rc) return rc;
    CK(cudaMemcpyAsync(t->d_scratch, bits, sizeof(uint32_t) * (size_t)words, cudaMemcpyHostToDevice, s));
    k_zero_columns<<<std::min(t->H, t->ctx->num_sms * 4), CONE_THREADS, 0, s>>>(t->d_T, (const uint32_t *)t->d_scratch);
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    jslp_lp_status st;
    rc = run_lp(t, 0, 1, &st, false);
    if (rc) return rc;
    *status = st.cycled ? COL_CYCLED : !st.feasible ? COL_INFEASIBLE : !st.bounded ? COL_UNBOUNDED : COL_OPTIMAL;
    *eval_raw = st.evaluation_raw;
    *pivots = st.phase1_pivots + st.phase2_pivots;
    return read_column(t, 0, rhs, vrow);
}

// Sets [s0, s0 + n) in one k_node_batch<NODE_COLUMNS> launch.  Those whose log shows a cycle (per-phase histories) or
// that hit the pivot or log cap go to redo: the HBM path stops a cycle before the pivot that completes the repeat.
static int column_resident(jslp_tab *t, const uint32_t *bits, int words, int s0, int n, int32_t *status,
                           double *eval_raw, int32_t *pivots, double *rhs, int32_t *vrow, std::vector<int> &redo) {
    ResidentBufs &rb = t->rbufs;
    const int H0 = t->saved.H;
    NodeBatchDev nb;
    size_t smem = 0;
    int rc = batch_fill(t, t->saved.M, t->saved.vrow, t->saved.vcol, H0, t->saved.lastElementIndex, n, nb, &smem);
    if (rc) return rc;
    rc = batch_cuts(t, nullptr, nullptr, nullptr, n, nb);  // no cut rows
    if (rc) return rc;
    // one device block per chunk: masks, final columns, final labels
    ScratchLayout L;
    const size_t b_keep = L.take(sizeof(uint32_t) * (size_t)n * words), b_rhs = L.take(sizeof(double) * (size_t)n * H0);
    const size_t b_vrow = L.take(sizeof(int) * (size_t)n * H0);
    rc = batch_scratch(t, L.bytes);
    if (rc) return rc;
    char *base = (char *)t->d_scratch;
    CK(cudaMemcpyAsync(base + b_keep, bits + (size_t)s0 * words, sizeof(uint32_t) * (size_t)n * words,
                       cudaMemcpyHostToDevice, t->ctx->stream));
    nb.keep = (const uint32_t *)(base + b_keep); nb.keep_words = words;
    nb.out_rhs = (double *)(base + b_rhs); nb.out_vrow = (int *)(base + b_vrow);
    rc = batch_launch<NODE_COLUMNS>(t, nb, n, smem, rhs + (size_t)s0 * H0, vrow + (size_t)s0 * H0);
    if (rc) return rc;
    std::vector<int> hit;
    rc = batch_screen(t, n, [&](int i) { return !rb.h_out[i].r.overflow; }, hit);
    if (rc) return rc;
    for (int i = 0; i < n; i++) {
        const NodeResult &r = rb.h_out[i].r;
        if (r.overflow || hit[i] >= 0) { redo.push_back(s0 + i); continue; }
        status[s0 + i] = r.status == ST_OPTIMAL ? COL_OPTIMAL : r.status == ST_UNBOUNDED ? COL_UNBOUNDED : COL_INFEASIBLE;
        eval_raw[s0 + i] = r.eval_raw;
        pivots[s0 + i] = r.p1 + r.p2;
    }
    return JSLP_OK;
}

extern "C" int jslp_column_batch(jslp_tab *t, const uint8_t *keep_cols, int n_sets, int32_t *status, double *eval_raw,
                                 int32_t *pivots, double *rhs, int32_t *vrow) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    if (n_sets < 0 || (n_sets > 0 && (!keep_cols || !status || !eval_raw || !pivots || !rhs || !vrow)))
        return fail(JSLP_E_INVALID, "column_batch: bad keep / output arguments");
    if (!t->saved.valid) return fail(JSLP_E_INVALID, "column_batch needs a snapshot (jslp_save)");
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, "column_batch: optional objectives are not supported");
    if (n_sets == 0) return JSLP_OK;
    CK(cudaSetDevice(t->ctx->device));
    const int W = t->W, H0 = t->saved.H;
    // keep masks, bit-packed over the columns (column 0 always kept)
    const int words = (W + 31) / 32;
    std::vector<uint32_t> bits = pack_bits(keep_cols, W, nullptr, n_sets, words);
    for (int i = 0; i < n_sets; i++) bits[(size_t)i * words] |= 1u;
    const CallerState caller(t);
    // every set has the snapshot's height, so either all of them are resident or none, and a launch's are consecutive
    int rc = batch_route(
        t, n_sets, [&](int) { return H0; }, true,
        [&](const int *idx, int m, std::vector<int> &redo) {
            return column_resident(t, bits.data(), words, idx[0], m, status, eval_raw, pivots, rhs, vrow, redo);
        },
        [&](int i) {
            return column_hbm(t, bits.data() + (size_t)i * words, words, status + i, eval_raw + i, pivots + i,
                              rhs + (size_t)i * H0, vrow + (size_t)i * H0);
        });
    const int rc2 = jslp_restore(t);
    if (rc == JSLP_OK) rc = rc2;
    CK(cudaStreamSynchronize(t->ctx->stream));
    caller.restore(t);
    return rc;
}

extern "C" int jslp_column(jslp_tab *t, int col, double *out) {
    if (!t || !out) return fail(JSLP_E_INVALID, "NULL argument");
    if (col < 0 || col >= t->W) return fail(JSLP_E_INVALID, "column: index out of range");
    CK(cudaSetDevice(t->ctx->device));
    return read_column(t, col, out, nullptr);
}
