// jslpsolver_b200/csrc/jslp_parametric.cuh -- parametric analysis of a solved LP: one right-hand side or one cost
// moves from its current value towards a target, and every basis change on the way is one breakpoint (included by
// jslp_api.cu; no reference counterpart).  DESIGN.md section 2d is the contract; in short, with P the precision:
//
//   rhs  (kind 0)  direction D (a column): per moved row i, sign_i * M[:,c] where its slack is non-basic in column c,
//                  sign_i at row r where it is basic in row r (two rows summed, one IEEE add).  Step bound t* = min of
//                  -M[r,0] / D[r] over restricted rows r >= 1 with D[r] < -P; shift M[r,0] += t * D[r]; the leaving
//                  row r* gets M[r*,0] = +0; entering column = dual ratio test min M[0,c] / M[r*,c] over M[r*,c] < -P.
//   cost (kind 1)  direction E (a row): -sign * M[r,:] where the variable is basic in row r, sign at column c where it
//                  is non-basic.  Step bound t* = min of -M[0,c] / E[c] over restricted columns with E[c] > P;
//                  shift M[0,c] += t * E[c]; the entering column c* gets M[0,c*] = +0; leaving row = the reference's
//                  phase-2 ratio test on c* (ratio_step).
//   frontier (kind 2)  as kind 1 with E read from the descriptor's one optional-objective row, which the step carries
//                  through every pivot (jslp_frontier.cuh, section 2g); each call first appends the current point
//                  (column 0 and the row labels) to a per-poll slot when the previous pivot changed it.
//
// sign_i = g * s_i (rhs) or g * sigma (cost), g = +1 when the target lies above the start.  The pivot itself is the
// two-kernel engine's: k_param_select stages it exactly as k_select stages Tableau.pivot(), and the in-place step
// executes it.  A CUDA graph holds k_batch_begin + PARAM_STEPS x (k_param_select, step); the host polls once per graph.
#pragma once

namespace jslp {

enum { PAR_RUNNING = 0, PAR_REACHED = 1, PAR_INFEASIBLE = 2, PAR_UNBOUNDED = 3, PAR_LIMIT = 4 };
static constexpr int PARAM_STEPS = 32;  // breakpoints per graph (per host poll)

// One piece of the path, written when the piece ends: theta there, the raw objective entry M[0,0] after the shift,
// the direction's objective entry D[0] / E[0] the piece moved along, and the basis change that ends it (-1 = none).
struct ParamRec {
    double theta, obj_raw, dobj;
    int r, c, leaving, entering;
    int pad[2];
};

struct ParamDev {
    ParamRec *log;  // max_breaks records
    int kind, n_labels;
    int label[2];
    double sign[2];
    double g, target, theta;
    int status, n, max_breaks, pad;
    // kind 2: PARAM_STEPS point slots of rowcap entries each, the record count at which each point was appended, the
    // points appended so far and whether the last staged pivot leaves a non-zero M[r*,0] (it changes the point)
    double *pt_rhs;
    int *pt_vrow, *pt_at;
    int npts, moved;
};

struct ParamSmem {
    RedSmem red;
    int row[2], col[2];
    double d0, obj, ec;
};

// Appends the record of the piece that ends here and advances theta; thread 0 only.
__device__ __forceinline__ void param_record(ParamDev *Pp, const ParamDev &P, double theta, double obj, double d0, int r,
                                             int c, int leaving, int entering, int status) {
    ParamRec e;
    e.theta = theta; e.obj_raw = obj; e.dobj = d0;
    e.r = r; e.c = c; e.leaving = leaving; e.entering = entering; e.pad[0] = e.pad[1] = 0;
    P.log[P.n] = e;
    Pp->theta = theta;
    Pp->n = P.n + 1;
    Pp->status = status;
}

// One breakpoint: locate the moved labels, build the direction on the fly, find the step bound, shift, select the
// other half of the pivot and stage it (or stop).  One CTA; does nothing once the path has stopped.  pcol (rhs) or
// prow (cost) holds the direction between the passes of one call; both are rewritten when the pivot is staged.
__global__ void __launch_bounds__(512) k_param_select(const TabDev *Tp, Rec *rec, ParamDev *Pp) {
    __shared__ TabDev T;
    __shared__ ParamDev P;
    __shared__ ParamSmem s;
    const int tid = threadIdx.x, NT = blockDim.x;
    if (tid == 0) { T = *Tp; P = *Pp; }
    if (tid < 2) { s.row[tid] = -1; s.col[tid] = -1; }
    __syncthreads();
    if (P.status != PAR_RUNNING) return;
    if (P.kind == 2 && P.moved) {  // the point the previous pivot moved to (or the start), before anything shifts
        const int slot = P.npts % PARAM_STEPS;
        const size_t off = (size_t)slot * T.rowcap;
        for (int r = tid; r < T.H; r += NT) {
            P.pt_rhs[off + r] = ldg_cg(T.M + (size_t)r * T.stride);
            P.pt_vrow[off + r] = T.vrow[r];
        }
        if (tid == 0) { P.pt_at[slot] = P.n; Pp->npts = P.npts + 1; Pp->moved = 0; }
        __syncthreads();
    }
    if (P.n >= P.max_breaks) {
        if (tid == 0) Pp->status = PAR_LIMIT;
        return;
    }
    const int W = T.W, H = T.H;
    const size_t stride = (size_t)T.stride;
    const double prec = T.prec;
    double *M = T.M;
    for (int k = 0; k < P.n_labels; k++) {
        int row, col;
        cut_lookup(T.vrow, H, T.vcol, W, P.label[k], tid, NT, row, col);
        if (row >= 0) s.row[k] = row;
        if (col >= 0) s.col[k] = col;
    }
    __syncthreads();
    const VI init = {INFINITY, INT_MAX};
    const double rho = __dmul_rn(P.g, __dsub_rn(P.target, P.theta));  // remaining distance

    if (P.kind == 0) {
        // ---- right-hand side: step bound over the rows, D kept in pcol
        const bool two = P.n_labels > 1;
        const int ca = s.col[0], cb = two ? s.col[1] : -1, ra = s.row[0], rb = two ? s.row[1] : -1;
        const double ga = P.sign[0], gb = P.sign[1];
        VI best = init;
        for (int rbase = 0; rbase < H; rbase += 8 * NT) {  // loads of a pass first, then the tests
            double rv[8], av[8], bv[8];
            int lab[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rbase + tid + k * NT;
                const bool in = r < H;
                rv[k] = in ? ldg_cg(M + r * stride) : 0.0;
                av[k] = (in && ca >= 0) ? ldg_cg(M + r * stride + ca) : 0.0;
                bv[k] = (in && cb >= 0) ? ldg_cg(M + r * stride + cb) : 0.0;
                lab[k] = (in && r > 0) ? T.vrow[r] : -1;
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rbase + tid + k * NT;
                if (r >= H) continue;
                double d = ca >= 0 ? __dmul_rn(ga, av[k]) : (r == ra ? ga : 0.0);
                if (two) d = __dadd_rn(d, cb >= 0 ? __dmul_rn(gb, bv[k]) : (r == rb ? gb : 0.0));
                T.pcol[r] = d;
                if (r == 0) s.d0 = d;
                else if (!is_unres(T, lab[k])) param_ratio(r, -rv[k], d, false, prec, best);
            }
        }
        best = block_reduce_vi<true>(best, init, s.red);
        const bool reach = best.i == INT_MAX || best.v >= rho;
        const double t = reach ? rho : best.v;
        const int rstar = reach ? -1 : best.i;
        for (int rbase = 0; rbase < H; rbase += 8 * NT) {  // the shift: M[r,0] + t * D[r], two roundings
            double rv[8], dv[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rbase + tid + k * NT;
                rv[k] = r < H ? ldg_cg(M + r * stride) : 0.0;
                dv[k] = r < H ? T.pcol[r] : 0.0;  // this thread's own store of the first pass
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rbase + tid + k * NT;
                if (r >= H) continue;
                double v = rv[k];
                if (dv[k] != 0.0) {
                    v = r == rstar ? 0.0 : __dadd_rn(v, __dmul_rn(t, dv[k]));
                    M[r * stride] = v;
                }
                if (r == 0) s.obj = v;
            }
        }
        const double theta = reach ? P.target : __dadd_rn(P.theta, __dmul_rn(P.g, t));
        if (reach) {
            if (tid == 0) param_record(Pp, P, theta, s.obj, s.d0, -1, -1, -1, -1, PAR_REACHED);
            return;
        }
        // dual ratio test on the leaving row (columns >= 1; the shift touched column 0 only)
        VI e = init;
        const double *lrow = M + rstar * stride;
        for (int c0 = 1; c0 < W; c0 += 8 * NT) {
            double cv[8], kv[8];
            int lab[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int c = c0 + tid + k * NT;
                cv[k] = c < W ? ldg_cg(M + c) : 0.0;
                kv[k] = c < W ? ldg_cg(lrow + c) : 0.0;
                lab[k] = c < W ? T.vcol[c] : -1;
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int c = c0 + tid + k * NT;
                if (c < W) param_ratio(c, cv[k], kv[k], is_unres(T, lab[k]), prec, e);
            }
        }
        e = block_reduce_vi<true>(e, init, s.red);
        if (e.i == INT_MAX) {
            if (tid == 0) param_record(Pp, P, theta, s.obj, s.d0, rstar, -1, -1, -1, PAR_INFEASIBLE);
            return;
        }
        const int cstar = e.i;
        __syncthreads();  // the shifted column 0 and every read of the direction are done before pcol is gathered
        int cnt = 0;
        for (int rbase = 0; rbase < H; rbase += 8 * NT) {  // gather the pivot column: loads, then stores
            double cv[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rbase + tid + k * NT;
                cv[k] = r < H ? ldg_cg(M + r * stride + cstar) : 0.0;
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rbase + tid + k * NT;
                if (r < H) { T.pcol[r] = cv[k]; if (nz16(cv[k])) cnt++; }
            }
        }
        cnt = block_reduce_int<1>(cnt, s.red);
        if (tid == 0) param_record(Pp, P, theta, s.obj, s.d0, rstar, cstar, T.vrow[rstar], T.vcol[cstar], PAR_RUNNING);
        cta_stage_pivot(T, rec, 2, rstar, cstar, 0, cnt);
        return;
    }

    // ---- cost: step bound over the columns, E kept in prow (kind 2: E is the carried row T.opt)
    const int rv_ = s.row[0], cv_ = s.col[0];
    const double sg = P.sign[0];
    const bool carried = P.kind == 2;
    const double *vr = carried ? T.opt : (rv_ >= 0 ? M + rv_ * stride : nullptr);
    VI best = init;
    for (int c0 = 0; c0 < W; c0 += 8 * NT) {
        double m0[8], er[8];
        int lab[8];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = c0 + tid + k * NT;
            m0[k] = c < W ? ldg_cg(M + c) : 0.0;
            er[k] = (c < W && vr != nullptr) ? ldg_cg(vr + c) : 0.0;
            lab[k] = (c < W && c > 0) ? T.vcol[c] : -1;
        }
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = c0 + tid + k * NT;
            if (c >= W) continue;
            const double e = carried ? er[k] : (vr != nullptr ? __dmul_rn(-sg, er[k]) : (c == cv_ ? sg : 0.0));
            T.prow[c] = e;
            if (c == 0) s.d0 = e;
            else param_ratio(c, m0[k], -e, is_unres(T, lab[k]), prec, best);
        }
    }
    best = block_reduce_vi<true>(best, init, s.red);
    const bool reach = best.i == INT_MAX || best.v >= rho;
    const double t = reach ? rho : best.v;
    const int cstar = reach ? -1 : best.i;
    for (int c0 = 0; c0 < W; c0 += 8 * NT) {  // the shift: M[0,c] + t * E[c], two roundings
        double m0[8], ev[8];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = c0 + tid + k * NT;
            m0[k] = c < W ? ldg_cg(M + c) : 0.0;
            ev[k] = c < W ? T.prow[c] : 0.0;  // this thread's own store of the first pass
        }
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = c0 + tid + k * NT;
            if (c >= W) continue;
            double v = m0[k];
            if (ev[k] != 0.0) {
                v = c == cstar ? 0.0 : __dadd_rn(v, __dmul_rn(t, ev[k]));
                M[c] = v;
            }
            if (c == 0) s.obj = v;
            if (c == cstar) s.ec = ev[k];
        }
    }
    const double theta = reach ? P.target : __dadd_rn(P.theta, __dmul_rn(P.g, t));
    if (reach) {
        if (tid == 0) param_record(Pp, P, theta, s.obj, s.d0, -1, -1, -1, -1, PAR_REACHED);
        return;
    }
    __syncthreads();  // the shifted cost row (M[0,c*] = +0) before the ratio test counts it
    const bool isneg = is_unres(T, T.vcol[cstar]) && s.ec < 0.0;
    VI m = init;
    int dmin = INT_MAX, cnt = 0;
    for (int rbase = 0; rbase < H; rbase += 8 * NT) {  // ratio test fused with the gather of the pivot column
        double cv[8], rv[8];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int r = rbase + tid + k * NT;
            cv[k] = r < H ? ldg_cg(M + r * stride + cstar) : 0.0;
            rv[k] = r < H ? ldg_cg(M + r * stride) : 0.0;
        }
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int r = rbase + tid + k * NT;
            if (r >= H) continue;
            T.pcol[r] = cv[k];
            ratio_step(r, cv[k], rv[k], isneg, prec, dmin, m, cnt);
        }
    }
    block_reduce_ratio(dmin, m, cnt, s.red);
    const int rstar = dmin != INT_MAX ? dmin : m.i;
    if (rstar == INT_MAX) {
        if (tid == 0) param_record(Pp, P, theta, s.obj, s.d0, -1, cstar, -1, -1, PAR_UNBOUNDED);
        return;
    }
    __syncthreads();  // every read of the direction in prow is done before the pivot row replaces it
    if (tid == 0) {
        param_record(Pp, P, theta, s.obj, s.d0, rstar, cstar, T.vrow[rstar], T.vcol[cstar], PAR_RUNNING);
        if (carried) Pp->moved = ldg_cg(M + rstar * stride) != 0.0;
    }
    cta_stage_pivot(T, rec, 2, rstar, cstar, isneg ? 1 : 0, cnt);
}

}  // namespace jslp

// The graph of one poll: k_batch_begin + PARAM_STEPS x (k_param_select, in-place step in update-only mode), captured
// on first use and kept while the step geometry stays the same.
static int param_graph(jslp_tab *t, cudaGraphExec_t *out) {
    const int grid = step_grid(t);
    const int smem = t->stride * 8;
    const int key = variant_index(t);
    if (t->param_graph && t->param_key[0] == grid && t->param_key[1] == smem && t->param_key[2] == key) {
        *out = t->param_graph;
        return JSLP_OK;
    }
    if (t->param_graph) cudaGraphExecDestroy(t->param_graph);
    t->param_graph = nullptr;
    const StepVariant &sv = step_variant(t);
    CK(cudaFuncSetAttribute(sv.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    cudaStream_t s = t->ctx->stream;
    cudaGraph_t g;
    CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    k_batch_begin<<<1, 32, 0, s>>>(t->d_rec);
    for (int i = 0; i < PARAM_STEPS; i++) {
        k_param_select<<<1, 512, 0, s>>>(t->d_T, t->d_rec, (ParamDev *)t->d_param);
        sv.fn<<<grid, sv.threads, smem, s>>>(t->d_T, t->d_rec, 0, t->hd.prow, t->stride);
    }
    cudaError_t e = cudaStreamEndCapture(s, &g);
    if (e != cudaSuccess) return fail(JSLP_E_CUDA, std::string("graph capture: ") + cudaGetErrorString(e));
    cudaGraphExec_t ge;
    e = cudaGraphInstantiate(&ge, g, 0);
    cudaGraphDestroy(g);
    if (e != cudaSuccess) return fail(JSLP_E_CUDA, std::string("graph instantiate: ") + cudaGetErrorString(e));
    t->param_graph = ge;
    t->param_key[0] = grid; t->param_key[1] = smem; t->param_key[2] = key;
    *out = ge;
    return JSLP_OK;
}

// The path on the live tableau; the caller snapshots it before and restores it after.  `drain`, when given, runs after
// every poll with the path state as the poll read it (jslp_frontier collects its point slots there).
typedef int (*param_drain_fn)(jslp_tab *t, const ParamDev &cur, void *arg);
static int parametric_run(jslp_tab *t, const ParamDev &p, int *n_out, int *status_out, double *end_rhs, int32_t *end_vrow,
                          param_drain_fn drain = nullptr, void *drain_arg = nullptr) {
    jslp_ctx *ctx = t->ctx;
    cudaStream_t s = ctx->stream;
    Rec init;
    memset(&init, 0, sizeof(init));
    init.status = ST_RUNNING; init.phase = 2; init.stop_at = -1; init.unbounded_var = -1; init.next_c = -1;
    *t->h_rec = init;
    CK(cudaMemcpyAsync(t->d_rec, t->h_rec, sizeof(Rec), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(t->d_param, &p, sizeof(ParamDev), cudaMemcpyHostToDevice, s));
    CK(cudaStreamSynchronize(s));
    cudaGraphExec_t ge;
    int rc = param_graph(t, &ge);
    if (rc) return rc;
    ParamDev cur = p;
    while (cur.status == PAR_RUNNING) {
        CK(cudaGraphLaunch(ge, s));
        ctx->launches += 1 + 2 * PARAM_STEPS;
        CK(cudaMemcpyAsync(&cur, t->d_param, sizeof(ParamDev), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        if (drain) {
            const int rc = drain(t, cur, drain_arg);
            if (rc) return rc;
        }
    }
    // the end state, before the caller restores the tableau
    CK(cudaMemcpy2DAsync(end_rhs, sizeof(double), t->hd.M, sizeof(double) * t->stride, sizeof(double), t->H,
                         cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(end_vrow, t->hd.vrow, sizeof(int) * (size_t)t->H, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    *n_out = cur.n;
    *status_out = cur.status;
    return JSLP_OK;
}

extern "C" int jslp_parametric(jslp_tab *t, int kind, const int32_t *labels, const double *signs, int n_labels,
                               double theta0, double target, int max_breaks, double *theta, double *obj_raw,
                               double *dobj, int32_t *rc_lbl, int *n_breaks, int *stop, double *end_rhs,
                               int32_t *end_vrow) {
    if (!t || !labels || !signs || !theta || !obj_raw || !dobj || !rc_lbl || !n_breaks || !stop || !end_rhs || !end_vrow)
        return fail(JSLP_E_INVALID, "NULL argument");
    if (kind != 0 && kind != 1) return fail(JSLP_E_INVALID, "parametric: kind must be 0 (rhs) or 1 (cost)");
    if (n_labels < 1 || n_labels > (kind == 0 ? 2 : 1)) return fail(JSLP_E_INVALID, "parametric: bad label count");
    if (max_breaks < 1) return fail(JSLP_E_INVALID, "parametric: max_breaks must be >= 1");
    if (!std::isfinite(theta0) || !std::isfinite(target)) return fail(JSLP_E_INVALID, "parametric: theta0 / target must be finite");
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, "parametric: optional objectives are not supported");
    for (int k = 0; k < n_labels; k++) {
        if (labels[k] < 0 || labels[k] >= t->n_index) return fail(JSLP_E_INVALID, "parametric: label out of range");
        if (signs[k] != 1.0 && signs[k] != -1.0) return fail(JSLP_E_INVALID, "parametric: signs must be +1 or -1");
    }
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
    rc = ensure_snapshot(t, 0);
    if (rc) return rc;
    rc = snapshot_copy(t, 0, true);
    if (rc) return rc;
    ParamDev p;
    memset(&p, 0, sizeof(p));
    p.log = (ParamRec *)t->d_plog;
    p.kind = kind; p.n_labels = n_labels;
    for (int k = 0; k < n_labels; k++) { p.label[k] = labels[k]; p.sign[k] = signs[k]; }
    p.g = target >= theta0 ? 1.0 : -1.0;
    p.target = target; p.theta = theta0;
    p.status = PAR_RUNNING; p.max_breaks = max_breaks;
    int n = 0, status = 0;
    rc = parametric_run(t, p, &n, &status, end_rhs, end_vrow);
    std::vector<ParamRec> recs((size_t)n);
    if (rc == JSLP_OK && n > 0) {
        cudaError_t e = cudaMemcpyAsync(recs.data(), t->d_plog, sizeof(ParamRec) * (size_t)n, cudaMemcpyDeviceToHost, s);
        if (e != cudaSuccess) rc = fail(JSLP_E_CUDA, std::string("parametric log: ") + cudaGetErrorString(e));
    }
    // the caller's tableau, labels, staged pivot and record exactly as they were
    const int rc2 = snapshot_copy(t, 0, false);
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
    return JSLP_OK;
}
