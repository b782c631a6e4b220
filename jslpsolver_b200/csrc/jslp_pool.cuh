// jslpsolver_b200/csrc/jslp_pool.cuh -- the region LPs of a MIP solution-pool search (included by jslp_api.cu after
// jslp_cone.cuh; no reference counterpart).  DESIGN.md section 2m is the contract; in short, with M the saved snapshot
// (the model's initial tableau, every structural column non-basic), region i is
//
//   M with the fixings of i applied in list order -- M[r,0] = M[r,0] - v * M[r,j], then M[r,j] = +0, for every row r,
//   row 0 included -- followed by the cut rows of i as addCutConstraints builds them, then simplex() with the cycle
//   check as asked, then the isIntegral / getMostFractionalVar scan.
//
// Regions whose rows fit shared memory run one CTA each in k_node_batch<NODE_POOL> (the fixings ride the scenario edit
// loop as EDIT_FIX_COL edits); the others, and any region whose log shows a cycle or that hits the in-kernel pivot or
// log cap, run one after another on the single-tableau path: jslp_restore, k_row_edits, jslp_add_cuts, run_lp,
// mip_scan.  Both apply the fixings with the same arithmetic in the same order.  jslp_target_batch (section 2o) adds
// cost edits and jslp_box_batch (section 2s) right-hand-side edits to the same node LP.
#pragma once

namespace jslp {

// The row pass of one node on the current buffer (the single-tableau path of jslp_pool_batch, jslp_target_batch and
// jslp_box_batch): one thread per row, the EDIT_RHS_COL, EDIT_RHS_ROW and EDIT_FIX_COL edits in list order, the
// arithmetic of k_node_batch<NODE_POOL>'s row pass.  Other kinds are skipped: they belong to the column pass.
__global__ void __launch_bounds__(256) k_row_edits(const TabDev *Tp, const EditDev *edits, int n) {
    const TabDev &T = *Tp;
    const int r = blockIdx.x * 256 + threadIdx.x;
    if (r >= T.H) return;
    double *row = T.M + (size_t)r * T.stride;
    double x = row[0];
    for (int k = 0; k < n; k++) {
        const EditDev e = edits[k];
        if (e.kind == EDIT_RHS_COL) x = edit_axpy_sub(x, e.d, row[e.pos]);
        else if (e.kind == EDIT_RHS_ROW && e.pos == r) x = edit_sub(x, e.d);
        else if (e.kind == EDIT_FIX_COL) { x = edit_axpy_sub(x, e.d, row[e.pos]); row[e.pos] = 0.0; }
    }
    row[0] = x;
}

}  // namespace jslp

enum { POOL_OPTIMAL = 0, POOL_INFEASIBLE = 1, POOL_UNBOUNDED = 2, POOL_CYCLED = 3 };

// What jslp_pool_batch hands back per region, and where.
struct PoolOut {
    int32_t *status, *is_integral, *branch_var, *pivots;
    double *evaluation, *branch_value, *rhs;
    int32_t *vrow;
    int row_stride;
    // the verdict of region i; column 0 and the labels (H entries) are copied by the caller when it is integral
    void set(int i, int st, double eval_raw, double precision, int integral, int bvar, double bval, int piv) {
        status[i] = st;
        evaluation[i] = st == POOL_OPTIMAL ? jslp_round_evaluation(eval_raw, precision) : st == POOL_UNBOUNDED ? -INFINITY : 0.0;
        is_integral[i] = st == POOL_OPTIMAL ? integral : 0;
        branch_var[i] = st == POOL_OPTIMAL && !integral ? bvar : -1;
        branch_value[i] = st == POOL_OPTIMAL && !integral ? bval : 0.0;
        pivots[i] = piv;
    }
};

// One node on the single-tableau path: the right-hand-side edits and fixings by k_row_edits, then the cost edits in
// list order with jslp_update_cost's kernels (the arithmetic of k_node_batch<NODE_POOL>'s column pass), then the cut
// rows.  The caller restores the snapshot.
static int pool_hbm(jslp_tab *t, const EditDev *edits, int n_edits, const jslp_cut *cuts, int n_cuts, int check_cycles,
                    int i, PoolOut &o) {
    cudaStream_t s = t->ctx->stream;
    int rc = jslp_restore(t);
    if (rc) return rc;
    std::vector<EditDev> rows;
    for (int k = 0; k < n_edits; k++)
        if (edits[k].kind == EDIT_RHS_COL || edits[k].kind == EDIT_RHS_ROW || edits[k].kind == EDIT_FIX_COL)
            rows.push_back(edits[k]);
    if (!rows.empty()) {
        rc = batch_scratch(t, sizeof(EditDev) * rows.size());
        if (rc) return rc;
        CK(cudaMemcpyAsync(t->d_scratch, rows.data(), sizeof(EditDev) * rows.size(), cudaMemcpyHostToDevice, s));
        k_row_edits<<<(t->H + 255) / 256, 256, 0, s>>>(t->d_T, (const EditDev *)t->d_scratch, (int)rows.size());
        t->ctx->launches += 1;
        CK(cudaGetLastError());
    }
    for (int k = 0; k < n_edits; k++) {
        const EditDev &e = edits[k];
        if (e.kind == EDIT_COST_ROW)
            k_row_axpy<<<std::max(1, (t->W + 255) / 256), 256, 0, s>>>(t->hd.M, t->hd.M + (size_t)e.pos * t->stride, e.d,
                                                                      t->W, 1);
        else if (e.kind == EDIT_COST_COL)
            k_entry_sub<<<1, 1, 0, s>>>(t->hd.M + e.pos, e.d);
        else
            continue;
        t->ctx->launches += 1;
        CK(cudaGetLastError());
    }
    rc = jslp_add_cuts(t, cuts, n_cuts);
    if (rc) return rc;
    jslp_lp_status st;
    rc = run_lp(t, 0, check_cycles, &st, false);
    if (rc) return rc;
    const int status = st.cycled ? POOL_CYCLED : !st.feasible ? POOL_INFEASIBLE : !st.bounded ? POOL_UNBOUNDED : POOL_OPTIMAL;
    MipOut mo{};
    mo.var_index = -1;
    if (status == POOL_OPTIMAL) {
        rc = mip_scan(t, &mo);
        if (rc) return rc;
    }
    o.set(i, status, st.evaluation_raw, t->precision, mo.is_integral, mo.var_index, mo.value,
          st.phase1_pivots + st.phase2_pivots);
    if (o.is_integral[i]) return read_column(t, 0, o.rhs + (size_t)i * o.row_stride, o.vrow + (size_t)i * o.row_stride);
    return JSLP_OK;
}

// Nodes idx[0..n) in one k_node_batch<NODE_POOL> launch.  Those whose log shows a cycle (per-phase histories, with
// check_cycles) or that hit the pivot or log cap go to redo.
static int pool_resident(jslp_tab *t, const std::vector<EditDev> &edits, const int32_t *edit_off, const jslp_cut *cuts,
                         const int32_t *cut_off, const int *idx, int n, int check_cycles, PoolOut &o,
                         std::vector<int> &redo) {
    ResidentBufs &rb = t->rbufs;
    const int H0 = t->saved.H;
    int maxc = 0, tote = 0;
    for (int k = 0; k < n; k++) {
        maxc = std::max(maxc, cut_off[idx[k] + 1] - cut_off[idx[k]]);
        tote += edit_off[idx[k] + 1] - edit_off[idx[k]];
    }
    NodeBatchDev nb;
    size_t smem = 0;
    int rc = batch_fill(t, t->saved.M, t->saved.vrow, t->saved.vcol, H0, t->saved.lastElementIndex, n, nb, &smem);
    if (rc) return rc;
    rc = batch_cuts(t, cuts, cut_off, idx, n, nb);
    if (rc) return rc;
    nb.Hcap = H0 + maxc;
    smem = node_smem_bytes(nb.Hcap, t->W, nullptr);
    std::vector<int> eoff((size_t)n + 1);
    std::vector<EditDev> ed((size_t)std::max(1, tote));
    int f = 0;
    for (int k = 0; k < n; k++) {
        eoff[k] = f;
        for (int h = edit_off[idx[k]]; h < edit_off[idx[k] + 1]; h++) {
            nb.cost_edits |= edits[h].kind == EDIT_COST_ROW || edits[h].kind == EDIT_COST_COL;
            ed[f++] = edits[h];
        }
    }
    eoff[n] = f;
    // one device block per chunk: edit offsets, edits, final columns, final labels
    const size_t n_out = (size_t)n * nb.Hcap;
    ScratchLayout L;
    const size_t b_off = L.take(sizeof(int) * (size_t)(n + 1)), b_ed = L.take(sizeof(EditDev) * (size_t)tote);
    const size_t b_rhs = L.take(sizeof(double) * n_out), b_vrow = L.take(sizeof(int) * n_out);
    rc = batch_scratch(t, L.bytes);
    if (rc) return rc;
    char *base = (char *)t->d_scratch;
    cudaStream_t s = t->ctx->stream;
    CK(cudaMemcpyAsync(base + b_off, eoff.data(), sizeof(int) * (size_t)(n + 1), cudaMemcpyHostToDevice, s));
    if (tote > 0) CK(cudaMemcpyAsync(base + b_ed, ed.data(), sizeof(EditDev) * (size_t)tote, cudaMemcpyHostToDevice, s));
    nb.edit_off = (const int *)(base + b_off);
    nb.edits = (const EditDev *)(base + b_ed);
    nb.out_rhs = (double *)(base + b_rhs); nb.out_vrow = (int *)(base + b_vrow);
    std::vector<double> rhs(n_out);
    std::vector<int32_t> vrow(n_out);
    rc = batch_launch<NODE_POOL>(t, nb, n, smem, rhs.data(), vrow.data());
    if (rc) return rc;
    std::vector<int> hit;
    rc = batch_screen(t, n, [&](int k) { return check_cycles && !rb.h_out[k].r.overflow; }, hit);
    if (rc) return rc;
    for (int k = 0; k < n; k++) {
        const NodeResult &r = rb.h_out[k].r;
        const int i = idx[k];
        if (r.overflow || hit[k] >= 0) { redo.push_back(i); continue; }
        const int st = r.status == ST_OPTIMAL ? POOL_OPTIMAL : r.status == ST_UNBOUNDED ? POOL_UNBOUNDED : POOL_INFEASIBLE;
        o.set(i, st, r.eval_raw, t->precision, r.is_integral, r.branch_var, r.branch_value, r.p1 + r.p2);
        if (o.is_integral[i]) {
            const int Hn = H0 + cut_off[i + 1] - cut_off[i];
            memcpy(o.rhs + (size_t)i * o.row_stride, rhs.data() + (size_t)k * nb.Hcap, sizeof(double) * (size_t)Hn);
            memcpy(o.vrow + (size_t)i * o.row_stride, vrow.data() + (size_t)k * nb.Hcap, sizeof(int32_t) * (size_t)Hn);
        }
    }
    return JSLP_OK;
}

// The node LPs of jslp_pool_batch and jslp_target_batch: node i is the snapshot with edits[edit_off[i] ..
// edit_off[i+1]) and the cut rows cuts[cut_off[i] .. cut_off[i+1]), routed by batch_route on its height (snapshot rows
// plus cuts); the tableau ends equal to the snapshot, with the caller's scalar state.
static int pool_run(jslp_tab *t, const std::vector<EditDev> &edits, const int32_t *edit_off, const jslp_cut *cuts,
                    const int32_t *cut_off, int n_nodes, int check_cycles, PoolOut &o) {
    CK(cudaSetDevice(t->ctx->device));
    const CallerState caller(t);
    int rc = batch_route(
        t, n_nodes, [&](int i) { return t->saved.H + cut_off[i + 1] - cut_off[i]; }, true,
        [&](const int *idx, int m, std::vector<int> &redo) {
            return pool_resident(t, edits, edit_off, cuts, cut_off, idx, m, check_cycles, o, redo);
        },
        [&](int i) {
            return pool_hbm(t, edits.data() + edit_off[i], edit_off[i + 1] - edit_off[i], cuts + cut_off[i],
                            cut_off[i + 1] - cut_off[i], check_cycles, i, o);
        });
    const int rc2 = jslp_restore(t);
    if (rc == JSLP_OK) rc = rc2;
    CK(cudaStreamSynchronize(t->ctx->stream));
    caller.restore(t);
    return rc;
}

// The checks jslp_pool_batch and jslp_target_batch share, with `what` naming the entry point and `node` its nodes in
// the messages.
static int pool_check(jslp_tab *t, const int32_t *edit_offsets, const jslp_cut *cuts, const int32_t *cut_offsets,
                      int n_nodes, int row_stride, bool outputs, const std::string &what, const char *node) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    if (n_nodes < 0 || (n_nodes > 0 && (!edit_offsets || !cut_offsets || !outputs)))
        return fail(JSLP_E_INVALID, what + ": bad offsets / output arguments");
    if (!t->saved.valid) return fail(JSLP_E_INVALID, what + " needs a snapshot (jslp_save)");
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, what + ": optional objectives are not supported");
    if (n_nodes == 0) return JSLP_OK;
    const int rc = batch_check_offsets({edit_offsets, cut_offsets}, n_nodes, what);
    if (rc) return rc;
    for (int i = 0; i < n_nodes; i++)
        if (t->saved.H + cut_offsets[i + 1] - cut_offsets[i] > row_stride)
            return fail(JSLP_E_INVALID, what + ": row_stride is below a " + node + "'s height (rows plus cuts)");
    return JSLP_OK;
}

// Every cut row of a batch is a min or max bound on a label of the snapshot.
static int pool_check_cuts(const jslp_tab *t, const jslp_cut *cuts, int n_cuts, const std::string &what) {
    for (int k = 0; k < n_cuts; k++)
        if ((cuts[k].type != 0 && cuts[k].type != 1) || cuts[k].var_index < 0 || cuts[k].var_index >= t->saved.nVars)
            return fail(JSLP_E_INVALID, what + ": cut type must be 0 (min) or 1 (max), on a label of the snapshot");
    return JSLP_OK;
}

extern "C" int jslp_pool_batch(jslp_tab *t, const jslp_fix *fixes, const int32_t *fix_offsets, const jslp_cut *cuts,
                               const int32_t *cut_offsets, int n_nodes, int check_cycles, int row_stride,
                               int32_t *status, double *evaluation, int32_t *is_integral, int32_t *branch_var,
                               double *branch_value, int32_t *pivots, double *rhs, int32_t *vrow) {
    int rc = pool_check(t, fix_offsets, cuts, cut_offsets, n_nodes, row_stride,
                        status && evaluation && is_integral && branch_var && branch_value && pivots && rhs && vrow,
                        "pool_batch", "region");
    if (rc || n_nodes == 0) return rc;
    const int n_fixes = fix_offsets[n_nodes], n_cuts = cut_offsets[n_nodes];
    if ((n_fixes > 0 && !fixes) || (n_cuts > 0 && !cuts)) return fail(JSLP_E_INVALID, "pool_batch: fixes / cuts is NULL");
    std::vector<EditDev> fx((size_t)n_fixes);
    for (int k = 0; k < n_fixes; k++) {
        if (fixes[k].column < 1 || fixes[k].column >= t->W) return fail(JSLP_E_INVALID, "pool_batch: fixed column out of range");
        fx[k] = EditDev{EDIT_FIX_COL, fixes[k].column, fixes[k].value};
    }
    rc = pool_check_cuts(t, cuts, n_cuts, "pool_batch");
    if (rc) return rc;
    PoolOut o{status, is_integral, branch_var, pivots, evaluation, branch_value, rhs, vrow, row_stride};
    return pool_run(t, fx, fix_offsets, cuts, cut_offsets, n_nodes, check_cycles, o);
}

// The edits of jslp_target_batch and jslp_box_batch resolved once against the snapshot's labels, as
// jslp_scenario_batch resolves them: kind 1 (updateCost) always, kind 0 (updateRightHandSide) when `rhs` is set, and
// then only before the node's cost edits, so that the row pass and the column pass apply them in list order.
static int node_edits(jslp_tab *t, const jslp_scenario_edit *edits, const int32_t *edit_offsets, int n_nodes, bool rhs,
                      const std::string &what, std::vector<EditDev> &ed) {
    CK(cudaSetDevice(t->ctx->device));
    HostMaps m;
    m.vrow.resize((size_t)t->saved.H);
    m.vcol.resize((size_t)t->W);
    cudaStream_t s = t->ctx->stream;
    CK(cudaMemcpyAsync(m.vrow.data(), t->saved.vrow, sizeof(int) * m.vrow.size(), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(m.vcol.data(), t->saved.vcol, sizeof(int) * m.vcol.size(), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    ed.resize((size_t)edit_offsets[n_nodes]);
    for (int i = 0; i < n_nodes; i++)
        for (int k = edit_offsets[i]; k < edit_offsets[i + 1]; k++) {
            const int kind = edits[k].kind;
            if (!rhs && kind != 1) return fail(JSLP_E_INVALID, what + ": edit kind must be 1 (cost)");
            if (rhs && kind != 0 && kind != 1) return fail(JSLP_E_INVALID, what + ": edit kind must be 0 (rhs) or 1 (cost)");
            if (kind == 0 && k > edit_offsets[i] && edits[k - 1].kind == 1)
                return fail(JSLP_E_INVALID, what + ": a node's right-hand-side edits come before its cost edits");
            if (!resolve_edit(m, edits[k], &ed[k]))
                return fail(JSLP_E_INVALID, what + (rhs ? ": unknown constraint or variable index" : ": unknown variable index"));
        }
    return JSLP_OK;
}

// jslp_target_batch and jslp_box_batch: the checks, the edits resolved, the node LPs.
static int edit_batch(jslp_tab *t, const jslp_scenario_edit *edits, const int32_t *edit_offsets, const jslp_cut *cuts,
                      const int32_t *cut_offsets, int n_nodes, int check_cycles, int row_stride, int32_t *status,
                      double *evaluation, int32_t *is_integral, int32_t *branch_var, double *branch_value,
                      int32_t *pivots, double *rhs, int32_t *vrow, bool rhs_edits, const std::string &what) {
    int rc = pool_check(t, edit_offsets, cuts, cut_offsets, n_nodes, row_stride,
                        status && evaluation && is_integral && branch_var && branch_value && pivots && rhs && vrow,
                        what, "node");
    if (rc || n_nodes == 0) return rc;
    const int n_edits = edit_offsets[n_nodes], n_cuts = cut_offsets[n_nodes];
    if ((n_edits > 0 && !edits) || (n_cuts > 0 && !cuts)) return fail(JSLP_E_INVALID, what + ": edits / cuts is NULL");
    std::vector<EditDev> ed;
    rc = node_edits(t, edits, edit_offsets, n_nodes, rhs_edits, what, ed);
    if (rc) return rc;
    rc = pool_check_cuts(t, cuts, n_cuts, what);
    if (rc) return rc;
    PoolOut o{status, is_integral, branch_var, pivots, evaluation, branch_value, rhs, vrow, row_stride};
    return pool_run(t, ed, edit_offsets, cuts, cut_offsets, n_nodes, check_cycles, o);
}

extern "C" int jslp_target_batch(jslp_tab *t, const jslp_scenario_edit *edits, const int32_t *edit_offsets,
                                 const jslp_cut *cuts, const int32_t *cut_offsets, int n_nodes, int check_cycles,
                                 int row_stride, int32_t *status, double *evaluation, int32_t *is_integral,
                                 int32_t *branch_var, double *branch_value, int32_t *pivots, double *rhs, int32_t *vrow) {
    return edit_batch(t, edits, edit_offsets, cuts, cut_offsets, n_nodes, check_cycles, row_stride, status, evaluation,
                      is_integral, branch_var, branch_value, pivots, rhs, vrow, false, "target_batch");
}

extern "C" int jslp_box_batch(jslp_tab *t, const jslp_scenario_edit *edits, const int32_t *edit_offsets,
                              const jslp_cut *cuts, const int32_t *cut_offsets, int n_nodes, int check_cycles,
                              int row_stride, int32_t *status, double *evaluation, int32_t *is_integral,
                              int32_t *branch_var, double *branch_value, int32_t *pivots, double *rhs, int32_t *vrow) {
    return edit_batch(t, edits, edit_offsets, cuts, cut_offsets, n_nodes, check_cycles, row_stride, status, evaluation,
                      is_integral, branch_var, branch_value, pivots, rhs, vrow, true, "box_batch");
}
