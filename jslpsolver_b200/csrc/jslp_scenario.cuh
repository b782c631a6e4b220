// jslpsolver_b200/csrc/jslp_scenario.cuh -- what-if scenarios on a solved tableau (included by jslp_api.cu after
// jslp_parametric.cuh).  The reference re-optimises one edit at a time (Constraint.setRightHandSide / Model.setCost,
// then simplex(); model.ts:247-273, dynamic-modification.ts:78-160); this runs a whole list of such edit sets, each
// from the same tableau (DESIGN.md 2e).
//
// Every edit in scope writes column 0 or row 0 only, so one scenario is the restored tableau plus two passes.
// Scenarios whose tableau fits shared memory run one CTA each in k_node_batch<NODE_SCENARIO>; the others, and any
// scenario whose log shows a cycle or that hits the in-kernel pivot or log cap, run one after another on the
// single-tableau path: restore, jslp_update_rhs / jslp_update_cost, run_lp -- the sequential definition itself.
// The source of both is a private snapshot (snaps[2]): not the user's jslp_save snapshot, and not snaps[0..1], which
// run_lp uses for its cycle replays.
#pragma once

enum { SCEN_OPTIMAL = 0, SCEN_INFEASIBLE = 1, SCEN_UNBOUNDED = 2, SCEN_CYCLED = 3 };

// Edit e (kind 0 or 1) resolved against the labels m: a right-hand-side or cost edit of the row its label is basic in,
// or of the column it is non-basic in.  False when the label is in neither.
static bool resolve_edit(const HostMaps &m, const jslp_scenario_edit &e, EditDev *out) {
    const int row = m.row_of(e.index), col = row < 0 ? m.col_of(e.index) : -1;
    if (row < 0 && col < 0) return false;
    if (e.kind == 0) *out = row < 0 ? EditDev{EDIT_RHS_COL, col, e.difference} : EditDev{EDIT_RHS_ROW, row, e.difference};
    else *out = row < 0 ? EditDev{EDIT_COST_COL, col, e.difference} : EditDev{EDIT_COST_ROW, row, e.difference};
    return true;
}

// The certificate outputs of jslp_recourse_batch (DESIGN.md 2u): the multipliers of n_rows row labels per scenario,
// to d_u + s * n_rows (device), at the position pos[label] (host; d_pos on the device) of each label.
struct RecourseCert {
    std::vector<int> pos;
    const int *d_pos;
    double *d_u;
    int n_rows;
};

// The certificate row of a scenario that ended with `status` and final column 0 `rhs` (H entries): row 0 at an
// optimum; when infeasible, the row phase 1 stopped at -- the first most negative entry below -precision, which is the
// row its last selection took (simplex.ts:38-54) and which no pivot has touched since; -1 otherwise.
static int cert_row(const jslp_tab *t, int status, const double *rhs) {
    if (status == SCEN_OPTIMAL) return 0;
    if (status != SCEN_INFEASIBLE) return -1;
    int r0 = -1;
    double v = -t->precision;
    for (int r = 1; r < t->H; r++)
        if (rhs[r] < v) { v = rhs[r]; r0 = r; }
    return r0;
}

// The certificate multipliers of scenario s on the single-tableau path, whose final state is the current tableau: its
// certificate row in one contiguous copy (the tableau is row-major), gathered through the final labels as
// k_node_batch<NODE_SCENARIO> gathers them, to d_u + s * n_rows.
static int cert_sequential(jslp_tab *t, const RecourseCert &c, int s, int status, const double *rhs,
                           const int32_t *vrow) {
    std::vector<double> u((size_t)c.n_rows, 0.0);
    const int cr = cert_row(t, status, rhs);
    cudaStream_t st = t->ctx->stream;
    if (cr >= 0) {
        std::vector<double> row((size_t)t->W);
        std::vector<int> vcol((size_t)t->W);
        CK(cudaMemcpyAsync(row.data(), t->hd.M + (size_t)cr * t->stride, sizeof(double) * (size_t)t->W,
                           cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(vcol.data(), t->hd.vcol, sizeof(int) * (size_t)t->W, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        const int nl = (int)c.pos.size();
        for (int k = 1; k < t->W; k++)
            if (vcol[k] >= 0 && vcol[k] < nl && c.pos[vcol[k]] >= 0) u[c.pos[vcol[k]]] = row[k];
        for (int r = 1; r < t->H; r++)
            if (vrow[r] >= 0 && vrow[r] < nl && c.pos[vrow[r]] >= 0) u[c.pos[vrow[r]]] = r == cr ? 1.0 : 0.0;
    }
    if (c.n_rows > 0)
        CK(cudaMemcpyAsync(c.d_u + (size_t)s * c.n_rows, u.data(), sizeof(double) * (size_t)c.n_rows,
                           cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));
    return JSLP_OK;
}

// One scenario on the single-tableau path, from the private snapshot.
static int scenario_sequential(jslp_tab *t, const jslp_scenario_edit *e, int n, int check_cycles, int32_t *status,
                               double *eval_raw, int32_t *p1, int32_t *p2, double *rhs, int32_t *vrow) {
    int rc = snapshot_copy(t, 2, false);
    for (int k = 0; k < n && rc == JSLP_OK; k++)
        rc = e[k].kind == 0 ? jslp_update_rhs(t, e[k].index, e[k].difference)
                            : jslp_update_cost(t, e[k].index, -1, e[k].difference);
    if (rc) return rc;
    jslp_lp_status st;
    rc = run_lp(t, 0, check_cycles, &st, false);
    if (rc) return rc;
    *status = st.cycled ? SCEN_CYCLED : !st.feasible ? SCEN_INFEASIBLE : !st.bounded ? SCEN_UNBOUNDED : SCEN_OPTIMAL;
    *eval_raw = st.evaluation_raw;
    *p1 = st.phase1_pivots;
    *p2 = st.phase2_pivots;
    return read_column(t, 0, rhs, vrow);
}

// Scenarios [s0, s0 + n) in one k_node_batch<NODE_SCENARIO> launch.  Those whose log shows a cycle (per-phase
// histories, as eval_nodes_resident) or that hit the pivot or log cap go to redo.
static int scenario_resident(jslp_tab *t, const std::vector<EditDev> &res, const int32_t *offsets, int s0, int n,
                             int check_cycles, int32_t *status, double *eval_raw, int32_t *p1, int32_t *p2,
                             double *rhs, int32_t *vrow, const RecourseCert *cert, std::vector<int> &redo) {
    ResidentBufs &rb = t->rbufs;
    const int H0 = t->H;
    const Snapshot &src = t->snaps[2];
    NodeBatchDev nb;
    size_t smem = 0;
    int rc = batch_fill(t, src.M, src.vrow, src.vcol, H0, t->lastElementIndex, n, nb, &smem);
    if (rc) return rc;
    // one device block per chunk: offsets, edits, final columns, final labels
    const int e0 = offsets[s0], ne = offsets[s0 + n] - e0;
    ScratchLayout L;
    const size_t b_off = L.take(sizeof(int) * (size_t)(n + 1)), b_ed = L.take(sizeof(EditDev) * (size_t)ne);
    const size_t b_rhs = L.take(sizeof(double) * (size_t)n * H0), b_vrow = L.take(sizeof(int) * (size_t)n * H0);
    rc = batch_scratch(t, L.bytes);
    if (rc) return rc;
    char *base = (char *)t->d_scratch;
    std::vector<int> off((size_t)n + 1);
    for (int i = 0; i <= n; i++) off[i] = offsets[s0 + i] - e0;
    cudaStream_t s = t->ctx->stream;
    CK(cudaMemcpyAsync(base + b_off, off.data(), sizeof(int) * (size_t)(n + 1), cudaMemcpyHostToDevice, s));
    if (ne > 0) CK(cudaMemcpyAsync(base + b_ed, res.data() + e0, sizeof(EditDev) * (size_t)ne, cudaMemcpyHostToDevice, s));
    nb.cut_off = (const int *)(base + b_off);
    nb.edits = (const EditDev *)(base + b_ed);
    nb.out_rhs = (double *)(base + b_rhs); nb.out_vrow = (int *)(base + b_vrow);
    if (cert) {
        nb.cert_u = cert->d_u + (size_t)s0 * cert->n_rows;
        nb.cert_pos = cert->d_pos;
        nb.cert_n = cert->n_rows;
        nb.cert_labels = (int)cert->pos.size();
    }
    if (n <= NODE_INLINE_OFF) {
        nb.n_inline = n;
        for (int i = 0; i <= n; i++) nb.cut_off_inline[i] = off[i];
    }
    rc = batch_launch<NODE_SCENARIO>(t, nb, n, smem, rhs + (size_t)s0 * H0, vrow + (size_t)s0 * H0);
    if (rc) return rc;
    std::vector<int> hit;
    rc = batch_screen(t, n, [&](int i) { return check_cycles && !rb.h_out[i].r.overflow; }, hit);
    if (rc) return rc;
    for (int i = 0; i < n; i++) {
        const NodeResult &r = rb.h_out[i].r;
        if (r.overflow || hit[i] >= 0) { redo.push_back(s0 + i); continue; }
        status[s0 + i] = r.status == ST_OPTIMAL ? SCEN_OPTIMAL : r.status == ST_UNBOUNDED ? SCEN_UNBOUNDED : SCEN_INFEASIBLE;
        eval_raw[s0 + i] = r.eval_raw;
        p1[s0 + i] = r.p1;
        p2[s0 + i] = r.p2;
    }
    return JSLP_OK;
}

// The argument checks of jslp_scenario_batch and jslp_recourse_batch (`what` names the caller in the messages).
static int scenario_check(jslp_tab *t, const jslp_scenario_edit *edits, const int32_t *offsets, int n_scenarios,
                          int32_t *status, double *eval_raw, int32_t *p1, int32_t *p2, double *rhs, int32_t *vrow,
                          const char *what) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    const std::string w(what);
    if (n_scenarios < 0 || (n_scenarios > 0 && (!offsets || !status || !eval_raw || !p1 || !p2 || !rhs || !vrow)))
        return fail(JSLP_E_INVALID, w + ": bad offsets / output arguments");
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, w + ": optional objectives are not supported");
    if (n_scenarios == 0) return JSLP_OK;
    int rc = batch_check_offsets({offsets}, n_scenarios, w);
    if (rc) return rc;
    if (offsets[n_scenarios] > 0 && !edits) return fail(JSLP_E_INVALID, w + ": edits is NULL");
    return JSLP_OK;
}

// jslp_scenario_batch once the arguments are checked (n_scenarios > 0) and the labels loaded into m; with cert set,
// every scenario's certificate multipliers go to cert->d_u as well.
static int scenario_run(jslp_tab *t, const HostMaps &m, const jslp_scenario_edit *edits, const int32_t *offsets,
                        int n_scenarios, int check_cycles, int32_t *status, double *eval_raw, int32_t *p1, int32_t *p2,
                        double *rhs, int32_t *vrow, const RecourseCert *cert) {
    const int n_edits = offsets[n_scenarios];
    // updateRightHandSide / updateCost resolved once against the labels: no edit pivots, so the positions are the
    // same for every scenario and every edit of it
    std::vector<EditDev> res((size_t)n_edits);
    for (int i = 0; i < n_scenarios; i++)
        for (int k = offsets[i]; k < offsets[i + 1]; k++) {
            const jslp_scenario_edit &e = edits[k];
            if (e.kind != 0 && e.kind != 1) return fail(JSLP_E_INVALID, "scenario_batch: edit kind must be 0 (rhs) or 1 (cost)");
            if (e.kind == 0 && k > offsets[i] && edits[k - 1].kind == 1)
                return fail(JSLP_E_INVALID, "scenario_batch: a scenario's right-hand-side edits come before its cost edits");
            if (!resolve_edit(m, e, &res[k])) return fail(JSLP_E_INVALID, "scenario_batch: unknown constraint or variable index");
        }
    const CallerState caller(t);
    int rc = ensure_snapshot(t, 2);
    if (rc) return rc;
    rc = snapshot_copy(t, 2, true);
    if (rc) return rc;
    // every scenario has the tab's height, so either all of them are resident or none, and a launch's are consecutive
    const int H = t->H;
    rc = batch_route(
        t, n_scenarios, [&](int) { return H; }, true,
        [&](const int *idx, int m, std::vector<int> &redo) {
            return scenario_resident(t, res, offsets, idx[0], m, check_cycles, status, eval_raw, p1, p2, rhs, vrow,
                                     cert, redo);
        },
        [&](int i) {
            const int rc1 = scenario_sequential(t, edits + offsets[i], offsets[i + 1] - offsets[i], check_cycles,
                                                status + i, eval_raw + i, p1 + i, p2 + i, rhs + (size_t)i * H,
                                                vrow + (size_t)i * H);
            if (rc1 || !cert) return rc1;
            return cert_sequential(t, *cert, i, status[i], rhs + (size_t)i * H, vrow + (size_t)i * H);
        });
    // the caller's tableau, labels, staged pivot and record exactly as they were
    const int rc2 = snapshot_copy(t, 2, false);
    if (rc == JSLP_OK) rc = rc2;
    CK(cudaStreamSynchronize(t->ctx->stream));
    caller.restore(t);
    return rc;
}

extern "C" int jslp_scenario_batch(jslp_tab *t, const jslp_scenario_edit *edits, const int32_t *offsets, int n_scenarios,
                                   int check_cycles, int32_t *status, double *eval_raw, int32_t *p1, int32_t *p2,
                                   double *rhs, int32_t *vrow) {
    int rc = scenario_check(t, edits, offsets, n_scenarios, status, eval_raw, p1, p2, rhs, vrow, "scenario_batch");
    if (rc || n_scenarios == 0) return rc;
    CK(cudaSetDevice(t->ctx->device));
    HostMaps m;
    rc = load_maps(t, m);
    if (rc) return rc;
    return scenario_run(t, m, edits, offsets, n_scenarios, check_cycles, status, eval_raw, p1, p2, rhs, vrow, nullptr);
}
