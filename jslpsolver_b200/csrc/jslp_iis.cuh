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

static int iis_scratch(jslp_tab *t, size_t bytes) {
    if (bytes <= t->iis_bytes) return JSLP_OK;
    cudaFree(t->d_iis);
    t->d_iis = nullptr;
    t->iis_bytes = 0;
    CK(cudaMalloc(&t->d_iis, bytes));
    t->iis_bytes = bytes;
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
    int rc = iis_scratch(t, sizeof(int) * (size_t)n);
    if (rc) return rc;
    int *d_rows = (int *)t->d_iis;
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
    jslp_ctx *ctx = t->ctx;
    cudaStream_t s = ctx->stream;
    ResidentBufs &rb = t->rbufs;
    const int H0 = t->saved.H;
    int Ws = 0;
    const size_t smem = node_smem_bytes(H0, t->W, &Ws);
    const int log_cap = t->node_log_cap;
    int rc = rb.ensure(n_sets, 0, log_cap);
    if (rc) return rc;
    for (int i = 0; i <= n_sets; i++) rb.h_off[i] = 0;  // no cut rows
    // keep masks, bit-packed, in device memory: one copy per launch
    const int words = (H0 + 31) / 32;
    std::vector<uint32_t> bits((size_t)n_sets * words, 0u);
    for (int i = 0; i < n_sets; i++)
        for (int r = 0; r < H0; r++)
            if (keep[(size_t)i * H0 + r]) bits[(size_t)i * words + (r >> 5)] |= 1u << (r & 31);
    rc = iis_scratch(t, sizeof(uint32_t) * bits.size());
    if (rc) return rc;
    CK(cudaMemcpyAsync(t->d_iis, bits.data(), sizeof(uint32_t) * bits.size(), cudaMemcpyHostToDevice, s));
    NodeBatchDev nb;
    memset(&nb, 0, sizeof(nb));
    nb.rootM = t->saved.M; nb.root_vrow = t->saved.vrow; nb.root_vcol = t->saved.vcol;
    nb.cuts = rb.dv_cuts; nb.cut_off = rb.dv_off; nb.out = rb.dv_out; nb.logs = rb.d_logs;
    nb.H0 = H0; nb.root_stride = t->stride; nb.first_index = t->saved.lastElementIndex;
    nb.Hcap = H0; nb.Ws = Ws; nb.log_cap = log_cap; nb.max_pivots = 100000;
    nb.keep = (const uint32_t *)t->d_iis; nb.keep_words = words; nb.phase1_only = 1;
    if (n_sets <= NODE_INLINE_OFF) nb.n_inline = n_sets;  // cut_off_inline: all zero
    CK(cudaFuncSetAttribute(k_node_batch<NODE_SUBSET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_node_batch<NODE_SUBSET><<<n_sets, NODE_THREADS, smem, s>>>(t->d_T, nb);
    ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(s));
    bool need_full = false;
    for (int i = 0; i < n_sets; i++) need_full |= rb.h_out[i].r.log_n > NODE_LOG_HEAD;
    if (need_full) {
        CK(cudaMemcpyAsync(rb.h_logs, rb.d_logs, sizeof(int4) * (size_t)n_sets * log_cap, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
    }
    for (int i = 0; i < n_sets; i++) {
        const NodeResult &r = rb.h_out[i].r;
        // phase 1 keeps its own history (simplex.ts:27): every entry of this log is a phase-1 entry
        const int4 *lg = r.log_n > NODE_LOG_HEAD ? rb.h_logs + (size_t)i * log_cap : rb.h_out[i].log_head;
        CycleHist h;
        int cs, cl, hit_at = -1;
        for (int k = 0; k < r.log_n && k < log_cap; k++)
            if (h.push_and_check(((long long)lg[k].z << 32) | (unsigned int)lg[k].w, &cs, &cl)) { hit_at = k; break; }
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
    // the scalar Tableau state and the executed-pivot log describe the tableau, not these tests
    const int feasible = t->feasible, bounded = t->bounded, iters = t->simplexIters, unb = t->unboundedVar;
    const double evaluation = t->evaluation, best = t->bestPossibleEval;
    const size_t log_size = t->host_log.size();
    std::vector<int> redo;
    int rc = JSLP_OK;
    if (t->engine != 1 && t->engine != 2 && resident_fits(t, H0)) {
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
    t->feasible = feasible; t->bounded = bounded; t->simplexIters = iters; t->unboundedVar = unb;
    t->evaluation = evaluation; t->bestPossibleEval = best;
    if (t->host_log.size() > log_size) t->host_log.resize(log_size);
    return rc;
}
