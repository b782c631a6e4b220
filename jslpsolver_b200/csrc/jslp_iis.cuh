// jslpsolver_b200/csrc/jslp_iis.cuh -- phase-1 feasibility of row subsets of the saved snapshot (included by
// jslp_api.cu after jslp_bnb.cuh).  No reference counterpart: this is the test behind Solution.iis() (DESIGN.md 2c).
//
// test(S) = the reference's phase 1 (simplex.ts:25-98) on cost row 0 plus the rows of S in their original order,
// with the cycle check on.  Every slack is basic in the initial tableau, so dropping a constraint is dropping its row.
// Sets whose rows fit shared memory run one CTA each in one k_node_batch<NODE_SUBSET> launch; the others (and any set that
// hits the in-kernel pivot or log cap) run one after another on the HBM path: the kept rows are gathered into the
// tableau and the ordinary phase-1 path runs on them.
#pragma once

namespace jslp {

// row d of the current buffer = snapshot row rows[d] (whole padded rows, so the padding stays zero)
__global__ void __launch_bounds__(256) k_gather_rows(double *M, int *vrow, const double *src, const int *src_vrow,
                                                      int stride, const int *rows, int n) {
    for (int d = blockIdx.x; d < n; d += gridDim.x) {
        const int r = rows[d];
        const double *s = src + (size_t)r * stride;
        double *o = M + (size_t)d * stride;
        for (int c = threadIdx.x; c < stride; c += blockDim.x) o[c] = s[c];
        if (threadIdx.x == 0) vrow[d] = src_vrow[r];
    }
}

}  // namespace jslp

// ---- scaffolding of the analysis batches (jslp_feasibility_batch, jslp_scenario_batch, jslp_column_batch) ----------

// One grow-only device block per tab for the per-call inputs and outputs of those batches; none of them holds it
// across a call of another.
static int batch_scratch(jslp_tab *t, size_t bytes) {
    if (bytes <= t->scratch_bytes) return JSLP_OK;
    cudaFree(t->d_scratch);
    t->d_scratch = nullptr;
    t->scratch_bytes = 0;
    CK(cudaMalloc(&t->d_scratch, bytes));
    t->scratch_bytes = bytes;
    return JSLP_OK;
}

// The scalar Tableau state and the executed-pivot log describe the caller's tableau, not a batch's sets: captured on
// entry, put back by restore() once the device tableau is restored.
struct CallerState {
    int feasible, bounded, iters, unb;
    double evaluation, best;
    size_t log_size;
    explicit CallerState(const jslp_tab *t)
        : feasible(t->feasible), bounded(t->bounded), iters(t->simplexIters), unb(t->unboundedVar),
          evaluation(t->evaluation), best(t->bestPossibleEval), log_size(t->host_log.size()) {}
    void restore(jslp_tab *t) const {
        t->feasible = feasible; t->bounded = bounded; t->simplexIters = iters; t->unboundedVar = unb;
        t->evaluation = evaluation; t->bestPossibleEval = best;
        if (t->host_log.size() > log_size) t->host_log.resize(log_size);
    }
};

// The shared-memory node kernel takes a batch of H-row tableaux unless the engine is pinned to 1 or 2; every other
// set runs on the single-tableau path.
static bool batch_resident(const jslp_tab *t, int H) { return t->engine != 1 && t->engine != 2 && resident_fits(t, H); }

// Sets per launch of H-row tableaux: the per-set outputs on the device stay bounded (about 32 MB).
static int batch_chunk(int H) {
    return (int)std::max<size_t>(1, std::min<size_t>(4096, ((size_t)32 << 20) / ((size_t)12 * H)));
}

// The fields of a k_node_batch launch of n sets that do not depend on the mode: the root tableau (M, vrow, vcol; H0
// rows at t's stride, labels handed out from first_index), no room for rows beyond H0, and the records and logs of
// rbufs, sized for n.  *smem = the launch's dynamic shared memory.
static int batch_fill(jslp_tab *t, const double *M, const int *vrow, const int *vcol, int H0, int first_index, int n,
                      NodeBatchDev &nb, size_t *smem) {
    ResidentBufs &rb = t->rbufs;
    int rc = rb.ensure(n, 0, t->node_log_cap);
    if (rc) return rc;
    int Ws = 0;
    *smem = node_smem_bytes(H0, t->W, &Ws);
    memset(&nb, 0, sizeof(nb));
    nb.rootM = M; nb.root_vrow = vrow; nb.root_vcol = vcol;
    nb.out = rb.dv_out; nb.logs = rb.d_logs;
    nb.H0 = H0; nb.root_stride = t->stride; nb.first_index = first_index;
    nb.Hcap = H0; nb.Ws = Ws; nb.log_cap = t->node_log_cap; nb.max_pivots = 100000;
    return JSLP_OK;
}

// One k_node_batch<MODE> launch of n sets; with out_rhs set, the final columns and labels to rhs / vrow (n x Hcap).
template <int MODE>
static int batch_launch(jslp_tab *t, const NodeBatchDev &nb, int n, size_t smem, double *rhs, int32_t *vrow) {
    jslp_ctx *ctx = t->ctx;
    cudaStream_t s = ctx->stream;
    CK(cudaFuncSetAttribute(k_node_batch<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_node_batch<MODE><<<n, NODE_THREADS, smem, s>>>(t->d_T, nb);
    ctx->launches += 1;
    CK(cudaGetLastError());
    if (nb.out_rhs) {
        CK(cudaMemcpyAsync(rhs, nb.out_rhs, sizeof(double) * (size_t)n * nb.Hcap, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(vrow, nb.out_vrow, sizeof(int) * (size_t)n * nb.Hcap, cudaMemcpyDeviceToHost, s));
    }
    CK(cudaStreamSynchronize(s));
    return JSLP_OK;
}

// The full logs of the last launch's n sets to the host, when need says a set whose log the caller reads outgrew the
// inline head.
static int batch_fetch_logs(jslp_tab *t, int n, bool need) {
    if (!need) return JSLP_OK;
    cudaStream_t s = t->ctx->stream;
    ResidentBufs &rb = t->rbufs;
    CK(cudaMemcpyAsync(rb.h_logs, rb.d_logs, sizeof(int4) * (size_t)n * t->node_log_cap, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return JSLP_OK;
}

// Set i's pivot log: the inline head, or the full log batch_fetch_logs brought over; min(log_n, node_log_cap) entries.
static const int4 *batch_log(const jslp_tab *t, int i) {
    const NodeOut &o = t->rbufs.h_out[i];
    return o.r.log_n > NODE_LOG_HEAD ? t->rbufs.h_logs + (size_t)i * t->node_log_cap : o.log_head;
}

// The index of the first entry of a node log that closes a repeat, with one (leaving, entering) history per phase
// (simplex.ts:27,102), or -1.
static int first_cycle(const int4 *lg, int n) {
    CycleHist h[2];
    int cs, cl;
    for (int k = 0; k < n; k++)
        if (h[(lg[k].x >> 30) & 1].push_and_check(((long long)lg[k].z << 32) | (unsigned int)lg[k].w, &cs, &cl))
            return k;
    return -1;
}

// Column col of the current buffer to out and, with vrow set, the row labels (H entries each).  The host mirror's M
// is the device's current buffer between calls (run_lp adopts it after every solve).
static int read_column(jslp_tab *t, int col, double *out, int32_t *vrow) {
    cudaStream_t s = t->ctx->stream;
    CK(cudaMemcpy2DAsync(out, sizeof(double), t->hd.M + col, sizeof(double) * t->stride, sizeof(double), t->H,
                         cudaMemcpyDeviceToHost, s));
    if (vrow) CK(cudaMemcpyAsync(vrow, t->hd.vrow, sizeof(int) * (size_t)t->H, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return JSLP_OK;
}

// One set on the HBM path: gather its rows, run phase 1 with the cycle check on.  The caller restores the snapshot.
static int feasibility_hbm(jslp_tab *t, const uint8_t *keep, int32_t *verdict, int32_t *pivots) {
    const int H0 = t->saved.H;
    std::vector<int> rows;
    for (int r = 0; r < H0; r++)
        if (r == 0 || keep[r]) rows.push_back(r);
    const int n = (int)rows.size();
    if (n == 1) { *verdict = 0; *pivots = 0; return JSLP_OK; }  // no row: phase 1 finds no leaving row
    cudaStream_t s = t->ctx->stream;
    int rc = batch_scratch(t, sizeof(int) * (size_t)n);
    if (rc) return rc;
    int *d_rows = (int *)t->d_scratch;
    CK(cudaMemcpyAsync(d_rows, rows.data(), sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, s));
    k_gather_rows<<<std::min(n, t->ctx->num_sms * 4), 256, 0, s>>>(t->hd.M, t->hd.vrow, t->saved.M, t->saved.vrow,
                                                                   t->stride, d_rows, n);
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(t->hd.vcol, t->saved.vcol, sizeof(int) * (size_t)t->W, cudaMemcpyDeviceToDevice, s));
    t->H = n;
    rc = push_desc(t);
    if (rc) return rc;
    jslp_lp_status st;
    rc = run_lp(t, 1, 1, &st, false);
    if (rc) return rc;
    *verdict = st.cycled ? 2 : (st.feasible ? 0 : 1);
    *pivots = st.phase1_pivots;
    return JSLP_OK;
}

// All sets in one k_node_batch<NODE_SUBSET> launch.  Sets whose log shows a cycle are undecided, stopped before the pivot
// that completes the repeat, as the reference's phase 1 stops; sets that hit the pivot or log cap first go to redo.
static int feasibility_resident(jslp_tab *t, const uint8_t *keep, int n_sets, int32_t *verdict, int32_t *pivots,
                                std::vector<int> &redo) {
    ResidentBufs &rb = t->rbufs;
    const int H0 = t->saved.H;
    NodeBatchDev nb;
    size_t smem = 0;
    int rc = batch_fill(t, t->saved.M, t->saved.vrow, t->saved.vcol, H0, t->saved.lastElementIndex, n_sets, nb, &smem);
    if (rc) return rc;
    for (int i = 0; i <= n_sets; i++) rb.h_off[i] = 0;  // no cut rows
    nb.cuts = rb.dv_cuts; nb.cut_off = rb.dv_off;
    // keep masks, bit-packed, in device memory: one copy per launch
    const int words = (H0 + 31) / 32;
    std::vector<uint32_t> bits((size_t)n_sets * words, 0u);
    for (int i = 0; i < n_sets; i++)
        for (int r = 0; r < H0; r++)
            if (keep[(size_t)i * H0 + r]) bits[(size_t)i * words + (r >> 5)] |= 1u << (r & 31);
    rc = batch_scratch(t, sizeof(uint32_t) * bits.size());
    if (rc) return rc;
    CK(cudaMemcpyAsync(t->d_scratch, bits.data(), sizeof(uint32_t) * bits.size(), cudaMemcpyHostToDevice,
                       t->ctx->stream));
    nb.keep = (const uint32_t *)t->d_scratch; nb.keep_words = words; nb.phase1_only = 1;
    if (n_sets <= NODE_INLINE_OFF) nb.n_inline = n_sets;  // cut_off_inline: all zero
    rc = batch_launch<NODE_SUBSET>(t, nb, n_sets, smem, nullptr, nullptr);
    if (rc) return rc;
    bool need_full = false;
    for (int i = 0; i < n_sets; i++) need_full |= rb.h_out[i].r.log_n > NODE_LOG_HEAD;
    rc = batch_fetch_logs(t, n_sets, need_full);
    if (rc) return rc;
    for (int i = 0; i < n_sets; i++) {
        const NodeResult &r = rb.h_out[i].r;
        // phase 1 keeps its own history (simplex.ts:27): every entry of this log is a phase-1 entry
        const int hit_at = first_cycle(batch_log(t, i), std::min(r.log_n, t->node_log_cap));
        if (hit_at >= 0) { verdict[i] = 2; if (pivots) pivots[i] = hit_at; continue; }
        if (r.overflow) { redo.push_back(i); continue; }
        verdict[i] = r.status == ST_P1_DONE ? 0 : 1;
        if (pivots) pivots[i] = r.p1;
    }
    return JSLP_OK;
}

extern "C" int jslp_feasibility_batch(jslp_tab *t, const uint8_t *keep, int n_sets, int32_t *verdict, int32_t *pivots) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    if (n_sets < 0 || (n_sets > 0 && (!keep || !verdict))) return fail(JSLP_E_INVALID, "bad keep / verdict arguments");
    if (!t->saved.valid) return fail(JSLP_E_INVALID, "feasibility_batch needs a snapshot (jslp_save)");
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, "feasibility_batch: optional objectives are not supported");
    if (n_sets == 0) return JSLP_OK;
    CK(cudaSetDevice(t->ctx->device));
    const int H0 = t->saved.H;
    const CallerState caller(t);
    std::vector<int> redo;
    int rc = JSLP_OK;
    if (batch_resident(t, H0)) {
        rc = feasibility_resident(t, keep, n_sets, verdict, pivots, redo);
    } else {
        for (int i = 0; i < n_sets; i++) redo.push_back(i);
    }
    for (size_t k = 0; k < redo.size() && rc == JSLP_OK; k++) {
        const int i = redo[k];
        int32_t p = 0;
        rc = feasibility_hbm(t, keep + (size_t)i * H0, verdict + i, &p);
        if (pivots) pivots[i] = p;
    }
    const int rc2 = jslp_restore(t);
    if (rc == JSLP_OK) rc = rc2;
    caller.restore(t);
    return rc;
}
