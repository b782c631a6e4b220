// jslpsolver_b200/csrc/jslp_crash.cuh -- warm start of an LP from a saved basis: crash the saved basic variables into
// the freshly uploaded tableau, one pivot each, before simplex() runs (included by jslp_api.cu; no reference
// counterpart).  DESIGN.md section 2f is the contract; in short, with P the precision, for each entering label e in
// list order:
//
//   e basic                  -> record "already basic"
//   e non-basic in column c  -> eligible rows r >= 1: leave[vrow[r]] and (M[r,c] < -P || P < M[r,c]) (crash_step);
//                               none -> record "rejected"; else the largest |M[r,c]|, lowest row on ties, is pivoted
//                               on exactly as Tableau.pivot(r, c) / jslp_pivot does it.
//
// k_crash_select takes one entry per launch, locates the label, reads the column of M and vrow in one pass (every load
// of a pass issued before any test), reduces, records the outcome and stages the pivot with cta_stage_pivot; the
// in-place step executes it.  A CUDA graph holds k_batch_begin + CRASH_STEPS x (k_crash_select, step).  Each select
// consumes exactly one entry, so the host launches ceil(n / CRASH_STEPS) graphs and reads the records back once.
#pragma once

namespace jslp {

static constexpr int CRASH_STEPS = 32;  // entries per graph
enum { CRASH_REJECTED = -1, CRASH_BASIC = -2 };  // record field 3 when no pivot is done

struct CrashDev {
    const int *enter;            // n_enter entering labels
    const unsigned char *leave;  // n_leave bytes: non-zero = the saved basis gives up the label's basic row
    int4 *out;                   // n_enter records (label, row, column, leaving label or CRASH_*)
    int n_enter, n_leave, next, n_pivots;
};

struct CrashSmem {
    RedSmem red;
    int row, col;
};

// One entry of the crash list; nothing once the list is exhausted.  pcol holds the column of the entering label
// after the pass (the pivot column when a pivot is staged; unused otherwise).
__global__ void __launch_bounds__(512) k_crash_select(const TabDev *Tp, Rec *rec, CrashDev *Cp) {
    __shared__ TabDev T;
    __shared__ CrashDev C;
    __shared__ CrashSmem s;
    const int tid = threadIdx.x, NT = blockDim.x;
    if (tid == 0) { T = *Tp; C = *Cp; s.row = -1; s.col = -1; }
    __syncthreads();
    if (C.next >= C.n_enter) return;
    const int k = C.next, label = C.enter[k];
    const int W = T.W, H = T.H;
    const size_t stride = (size_t)T.stride;
    const double prec = T.prec;
    const double *M = T.M;
    {
        int row, col;
        cut_lookup(T.vrow, H, T.vcol, W, label, tid, NT, row, col);
        if (row >= 0) s.row = row;
        if (col >= 0) s.col = col;
    }
    __syncthreads();
    const int c = s.col;
    if (s.row >= 0 || c < 0) {  // already basic, or not in the tableau at all
        if (tid == 0) {
            C.out[k] = make_int4(label, s.row, c, s.row >= 0 ? CRASH_BASIC : CRASH_REJECTED);
            Cp->next = k + 1;
        }
        return;
    }
    const VI init = {-1.0, INT_MAX};
    VI best = init;
    int cnt = 0;
    for (int rbase = 0; rbase < H; rbase += 8 * NT) {  // loads of a pass first, then the tests
        double cv[8];
        int lab[8];
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int r = rbase + tid + j * NT;
            cv[j] = r < H ? ldg_cg(M + r * stride + c) : 0.0;
            lab[j] = (r > 0 && r < H) ? T.vrow[r] : -1;
        }
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int r = rbase + tid + j * NT;
            if (r >= H) continue;
            T.pcol[r] = cv[j];  // the pivot column as jslp_pivot gathers it, row 0 included
            if (nz16(cv[j])) cnt++;
            const bool leave = lab[j] >= 0 && lab[j] < C.n_leave && C.leave[lab[j]] != 0;
            if (r > 0) crash_step(r, cv[j], leave, prec, best);
        }
    }
    best = block_reduce_vi<false>(best, init, s.red);
    cnt = block_reduce_int<1>(cnt, s.red);
    if (best.i == INT_MAX) {
        if (tid == 0) {
            C.out[k] = make_int4(label, -1, c, CRASH_REJECTED);
            Cp->next = k + 1;
        }
        return;
    }
    const int rstar = best.i;
    if (tid == 0) {  // thread 0 reads the leaving label before cta_stage_pivot swaps it, on the same thread
        C.out[k] = make_int4(label, rstar, c, T.vrow[rstar]);
        Cp->next = k + 1;
        Cp->n_pivots = C.n_pivots + 1;
    }
    cta_stage_pivot(T, rec, rec->phase, rstar, c, 0, cnt);
}

}  // namespace jslp

// The graph of CRASH_STEPS entries: k_batch_begin + CRASH_STEPS x (k_crash_select, in-place step in update-only mode),
// captured on first use and kept while the step geometry stays the same.
static int crash_graph(jslp_tab *t, cudaGraphExec_t *out) {
    const int grid = step_grid(t);
    const int smem = t->stride * 8;
    const int key = variant_index(t);
    if (t->crash_graph && t->crash_key[0] == grid && t->crash_key[1] == smem && t->crash_key[2] == key) {
        *out = t->crash_graph;
        return JSLP_OK;
    }
    if (t->crash_graph) cudaGraphExecDestroy(t->crash_graph);
    t->crash_graph = nullptr;
    const StepVariant &sv = step_variant(t);
    CK(cudaFuncSetAttribute(sv.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    cudaStream_t s = t->ctx->stream;
    cudaGraph_t g;
    CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    k_batch_begin<<<1, 32, 0, s>>>(t->d_rec);
    for (int i = 0; i < CRASH_STEPS; i++) {
        k_crash_select<<<1, 512, 0, s>>>(t->d_T, t->d_rec, (CrashDev *)t->d_crash);
        sv.fn<<<grid, sv.threads, smem, s>>>(t->d_T, t->d_rec, 0, t->hd.prow, t->stride);
    }
    cudaError_t e = cudaStreamEndCapture(s, &g);
    if (e != cudaSuccess) return fail(JSLP_E_CUDA, std::string("graph capture: ") + cudaGetErrorString(e));
    cudaGraphExec_t ge;
    e = cudaGraphInstantiate(&ge, g, 0);
    cudaGraphDestroy(g);
    if (e != cudaSuccess) return fail(JSLP_E_CUDA, std::string("graph instantiate: ") + cudaGetErrorString(e));
    t->crash_graph = ge;
    t->crash_key[0] = grid; t->crash_key[1] = smem; t->crash_key[2] = key;
    *out = ge;
    return JSLP_OK;
}

extern "C" int jslp_crash(jslp_tab *t, const int32_t *enter, int n_enter, const uint8_t *leave, int32_t *out,
                          int *n_pivots) {
    if (!t || !n_pivots || (n_enter > 0 && (!enter || !out)) || (!leave && t->n_index > 0))
        return fail(JSLP_E_INVALID, "NULL argument");
    if (n_enter < 0) return fail(JSLP_E_INVALID, "crash: n_enter must be >= 0");
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, "crash: optional objectives are not supported");
    for (int k = 0; k < n_enter; k++)
        if (enter[k] < 0 || enter[k] >= t->n_index) return fail(JSLP_E_INVALID, "crash: label out of range");
    *n_pivots = 0;
    if (n_enter == 0) return JSLP_OK;
    jslp_ctx *ctx = t->ctx;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    int rc = ensure_step_bufs(t, step_grid(t));
    if (rc) return rc;
    if (!t->d_crash) CK(cudaMalloc(&t->d_crash, sizeof(CrashDev)));
    const size_t need = sizeof(int4) * (size_t)n_enter + sizeof(int) * (size_t)n_enter + (size_t)t->n_index;
    if (need > t->crash_bytes) {
        CK(cudaStreamSynchronize(s));
        cudaFree(t->d_crash_buf);
        t->d_crash_buf = nullptr;
        t->crash_bytes = 0;
        CK(cudaMalloc(&t->d_crash_buf, need));
        t->crash_bytes = need;
    }
    char *base = (char *)t->d_crash_buf;  // records first: int4 alignment
    CrashDev c;
    memset(&c, 0, sizeof(c));
    c.out = (int4 *)base;
    c.enter = (const int *)(base + sizeof(int4) * (size_t)n_enter);
    c.leave = (const unsigned char *)(base + (sizeof(int4) + sizeof(int)) * (size_t)n_enter);
    c.n_enter = n_enter; c.n_leave = t->n_index;
    CK(cudaMemcpyAsync((void *)c.enter, enter, sizeof(int) * (size_t)n_enter, cudaMemcpyHostToDevice, s));
    if (t->n_index > 0) CK(cudaMemcpyAsync((void *)c.leave, leave, (size_t)t->n_index, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(t->d_crash, &c, sizeof(CrashDev), cudaMemcpyHostToDevice, s));
    Rec init;  // the record jslp_pivot starts from
    memset(&init, 0, sizeof(init));
    init.status = ST_RUNNING; init.phase = 2; init.stop_at = -1; init.unbounded_var = -1; init.next_c = -1;
    *t->h_rec = init;
    CK(cudaMemcpyAsync(t->d_rec, t->h_rec, sizeof(Rec), cudaMemcpyHostToDevice, s));
    cudaGraphExec_t ge;
    rc = crash_graph(t, &ge);
    if (rc) return rc;
    const int graphs = (n_enter + CRASH_STEPS - 1) / CRASH_STEPS;
    for (int i = 0; i < graphs; i++) {
        CK(cudaGraphLaunch(ge, s));
        ctx->launches += 1 + 2 * CRASH_STEPS;
    }
    CrashDev end;
    CK(cudaMemcpyAsync(&end, t->d_crash, sizeof(CrashDev), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(out, c.out, sizeof(int4) * (size_t)n_enter, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    if (end.next != n_enter) return fail(JSLP_E_CUDA, "crash: the device did not consume the whole list");
    *n_pivots = end.n_pivots;
    return JSLP_OK;
}
