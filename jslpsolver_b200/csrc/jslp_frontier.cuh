// jslpsolver_b200/csrc/jslp_frontier.cuh -- the Pareto frontier of a two-objective LP from the optimal tableau of its
// first objective (included by jslp_api.cu after jslp_parametric.cuh; no reference counterpart).  DESIGN.md section 2g
// is the contract; in short, with C2 the second objective's row-0 entries by label (sigma2 * c2_j, 0 for slacks):
//
//   pricing   R2[c] = delta(c) + sum over blocks of FR_ROWS rows of 1..H-1 (in block order) of the block partial
//             +0 - C2[vrow[r]] * M[r,c] - ... (ascending rows, rows with C2 == 0 skipped), delta(0) = 0,
//             delta(c) = C2[vcol[c]];  E = R2 - M[0,:].  One kernel, k_price_objective.
//   path      the cost-parametric step of section 2d (k_param_select kind 2) from theta = 0 to 1 with E as the
//             direction, E registered as the tableau's one optional objective so that the step carries it through
//             every pivot as simplex.ts:393-412 carries an optional objective.
//
// The caller's tableau, labels, staged pivot, record and descriptor are restored before jslp_frontier returns.
#pragma once

namespace jslp {

static constexpr int FR_ROWS = 64;   // rows per block of the pricing sum (part of the contract: it fixes the order)
static constexpr int FR_COLS = 128;  // columns per CTA of k_price_objective, one per thread

// R2 and E of section 2g.  One CTA per FR_COLS outputs walks every row block in order; two warps compact the block's
// rows with a non-zero coefficient (ascending) into shared memory, then every thread runs its column's partial over
// them.  The grid only splits columns, so any grid gives the same bits.  Output k < n_out is column c = map[k] (c = k
// without a map) and goes to r2[k] and, when e is given, e[k]; jslp_frontier prices every column (no map, n_out = W),
// jslp_lex_next writes R straight into row 0 of the next level's tableau, through the face's kept-column map.
__global__ void __launch_bounds__(FR_COLS) k_price_objective(const TabDev *Tp, const double *c2, const int *map,
                                                             int n_out, double *r2, double *e) {
    __shared__ TabDev T;
    __shared__ int s_row[FR_ROWS];
    __shared__ double s_coef[FR_ROWS];
    __shared__ unsigned int s_bal[FR_ROWS / 32];
    const int tid = threadIdx.x;
    if (tid == 0) T = *Tp;
    __syncthreads();
    const int H = T.H;
    const size_t stride = (size_t)T.stride;
    const int k_out = blockIdx.x * FR_COLS + tid;
    const bool in = k_out < n_out;
    const int c = in && map ? map[k_out] : k_out;
    double R = 0.0;
    if (in && c > 0) R = c2[T.vcol[c]];
    for (int r0 = 1; r0 < H; r0 += FR_ROWS) {
        double k = 0.0;
        unsigned int bal = 0;
        if (tid < FR_ROWS) {  // whole warps: the ballot needs every lane
            const int r = r0 + tid;
            if (r < H) k = c2[T.vrow[r]];
            bal = __ballot_sync(0xffffffffu, k != 0.0);
            if ((tid & 31) == 0) s_bal[tid >> 5] = bal;
        }
        __syncthreads();
        if (tid < FR_ROWS && k != 0.0) {
            int pos = __popc(bal & ((1u << (tid & 31)) - 1u));
            for (int w = 0; w < (tid >> 5); w++) pos += __popc(s_bal[w]);
            s_row[pos] = r0 + tid;
            s_coef[pos] = k;
        }
        __syncthreads();
        int n = 0;
#pragma unroll
        for (int w = 0; w < FR_ROWS / 32; w++) n += __popc(s_bal[w]);
        if (in) {
            double p = 0.0;
#pragma unroll 4
            for (int j = 0; j < n; j++) p = __dsub_rn(p, __dmul_rn(s_coef[j], ldg_cg(T.M + (size_t)s_row[j] * stride + c)));
            R = __dadd_rn(R, p);
        }
        __syncthreads();  // the lists are rewritten by the next block
    }
    if (in) {
        r2[k_out] = R;
        if (e) e[k_out] = __dsub_rn(R, ldg_cg(T.M + c));
    }
}

}  // namespace jslp

// Device scratch of one jslp_frontier call, carved out of t->d_front.
struct FrontierBufs {
    double *c2, *r2, *e, *optcoef, *pt_rhs;
    int *pt_vrow, *pt_at;
};

static size_t frontier_layout(const jslp_tab *t, char *base, FrontierBufs *b) {
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char *p = base ? base + off : nullptr;
        off += (bytes + 255) & ~(size_t)255;
        return (void *)p;
    };
    b->c2 = (double *)take(sizeof(double) * (size_t)t->n_index);
    b->r2 = (double *)take(sizeof(double) * (size_t)t->stride);
    b->e = (double *)take(sizeof(double) * (size_t)t->stride);
    b->optcoef = (double *)take(sizeof(double));
    b->pt_rhs = (double *)take(sizeof(double) * (size_t)PARAM_STEPS * t->rowcap);
    b->pt_vrow = (int *)take(sizeof(int) * (size_t)PARAM_STEPS * t->rowcap);
    b->pt_at = (int *)take(sizeof(int) * (size_t)PARAM_STEPS);
    return off;
}

struct FrontierDrain {
    FrontierBufs b;
    int max_points, done;
    double *pt_rhs;
    int32_t *pt_vrow, *pt_break;
};

// Copies the points the last poll appended (at most PARAM_STEPS: one per k_param_select call) out of their slots.
static int frontier_drain(jslp_tab *t, const ParamDev &cur, void *arg) {
    FrontierDrain &d = *(FrontierDrain *)arg;
    cudaStream_t s = t->ctx->stream;
    const size_t H = (size_t)t->H;
    for (int k = d.done; k < cur.npts && k < d.max_points; k++) {
        const size_t slot = (size_t)(k % PARAM_STEPS);
        CK(cudaMemcpyAsync(d.pt_rhs + (size_t)k * H, d.b.pt_rhs + slot * t->rowcap, sizeof(double) * H,
                           cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(d.pt_vrow + (size_t)k * H, d.b.pt_vrow + slot * t->rowcap, sizeof(int) * H,
                           cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(d.pt_break + k, d.b.pt_at + slot, sizeof(int), cudaMemcpyDeviceToHost, s));
    }
    CK(cudaStreamSynchronize(s));
    d.done = cur.npts;
    return JSLP_OK;
}

extern "C" int jslp_frontier(jslp_tab *t, const double *cost2_by_label, int max_breaks, int max_points, double *r2,
                             double *dir, double *theta, double *obj_raw, double *dobj, int32_t *rc_lbl, int *n_breaks,
                             int *stop, double *pt_rhs, int32_t *pt_vrow, int32_t *pt_break, int *n_points,
                             double *end_rhs, int32_t *end_vrow) {
    if (!t || !cost2_by_label || !r2 || !dir || !theta || !obj_raw || !dobj || !rc_lbl || !n_breaks || !stop ||
        !n_points || !end_rhs || !end_vrow)
        return fail(JSLP_E_INVALID, "NULL argument");
    if (max_breaks < 1) return fail(JSLP_E_INVALID, "frontier: max_breaks must be >= 1");
    if (max_points < 0 || (max_points > 0 && (!pt_rhs || !pt_vrow || !pt_break)))
        return fail(JSLP_E_INVALID, "frontier: max_points must be >= 0, with point buffers when > 0");
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, "frontier: optional objectives are not supported");
    CK(cudaSetDevice(t->ctx->device));
    cudaStream_t s = t->ctx->stream;
    int rc = ensure_step_bufs(t, step_grid(t));
    if (rc) return rc;
    if (!t->d_param) CK(cudaMalloc(&t->d_param, sizeof(ParamDev)));
    if (max_breaks > t->param_cap) {
        CK(cudaStreamSynchronize(s));
        cudaFree(t->d_plog);
        t->d_plog = nullptr;
        t->param_cap = 0;
        CK(cudaMalloc(&t->d_plog, sizeof(ParamRec) * (size_t)max_breaks));
        t->param_cap = max_breaks;
    }
    FrontierBufs b;
    const size_t bytes = frontier_layout(t, nullptr, &b);
    if (bytes > t->front_bytes) {
        CK(cudaStreamSynchronize(s));
        cudaFree(t->d_front);
        t->d_front = nullptr;
        t->front_bytes = 0;
        CK(cudaMalloc(&t->d_front, bytes));
        t->front_bytes = bytes;
    }
    frontier_layout(t, (char *)t->d_front, &b);
    rc = ensure_snapshot(t, 0);
    if (rc) return rc;
    rc = snapshot_copy(t, 0, true);
    if (rc) return rc;
    CK(cudaMemcpyAsync(b.c2, cost2_by_label, sizeof(double) * (size_t)t->n_index, cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(b.e, 0, sizeof(double) * (size_t)t->stride, s));
    k_price_objective<<<(t->W + FR_COLS - 1) / FR_COLS, FR_COLS, 0, s>>>(t->d_T, b.c2, nullptr, t->W, b.r2, b.e);
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(r2, b.r2, sizeof(double) * (size_t)t->W, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(dir, b.e, sizeof(double) * (size_t)t->W, cudaMemcpyDeviceToHost, s));
    // E becomes the tableau's one optional objective for the length of the path
    double *opt0 = t->hd.opt, *optcoef0 = t->hd.optcoef;
    t->hd.opt = b.e;
    t->hd.optcoef = b.optcoef;
    t->nOpt = 1;
    rc = push_desc(t);
    ParamDev p;
    memset(&p, 0, sizeof(p));
    p.log = (ParamRec *)t->d_plog;
    p.kind = 2;
    p.g = 1.0; p.target = 1.0; p.theta = 0.0;
    p.status = PAR_RUNNING; p.max_breaks = max_breaks;
    p.pt_rhs = b.pt_rhs; p.pt_vrow = b.pt_vrow; p.pt_at = b.pt_at;
    p.moved = 1;  // the start is the first point
    FrontierDrain d{b, max_points, 0, pt_rhs, pt_vrow, pt_break};
    int n = 0, status = 0, npts = 0;
    if (rc == JSLP_OK) rc = parametric_run(t, p, &n, &status, end_rhs, end_vrow, frontier_drain, &d);
    npts = d.done;
    std::vector<ParamRec> recs((size_t)n);
    if (rc == JSLP_OK && n > 0) {
        cudaError_t e = cudaMemcpyAsync(recs.data(), t->d_plog, sizeof(ParamRec) * (size_t)n, cudaMemcpyDeviceToHost, s);
        if (e != cudaSuccess) rc = fail(JSLP_E_CUDA, std::string("frontier log: ") + cudaGetErrorString(e));
    }
    // the caller's descriptor, tableau, labels, staged pivot and record exactly as they were
    t->hd.opt = opt0;
    t->hd.optcoef = optcoef0;
    t->nOpt = 0;
    int rc2 = push_desc(t);
    if (rc == JSLP_OK) rc = rc2;
    rc2 = snapshot_copy(t, 0, false);
    if (rc == JSLP_OK) rc = rc2;
    CK(cudaStreamSynchronize(s));
    if (rc) return rc;
    for (int k = 0; k < n; k++) {
        theta[k] = recs[k].theta; obj_raw[k] = recs[k].obj_raw; dobj[k] = recs[k].dobj;
        rc_lbl[4 * k] = recs[k].r; rc_lbl[4 * k + 1] = recs[k].c;
        rc_lbl[4 * k + 2] = recs[k].leaving; rc_lbl[4 * k + 3] = recs[k].entering;
    }
    *n_breaks = n;
    *stop = status;
    *n_points = npts;
    return JSLP_OK;
}
