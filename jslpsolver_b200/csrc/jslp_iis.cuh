// jslpsolver_b200/csrc/jslp_iis.cuh -- the row-subset batch behind jslp_feasibility_batch and jslp_conflict_batch
// (included by jslp_api.cu after jslp_bnb.cuh; its launch helpers are jslp_batch.cuh's).  No reference
// counterpart: the feasibility test is the one behind Solution.iis() (DESIGN.md 2c), the conflict nodes the ones behind
// Conflict() (DESIGN.md 2n).
//
// A row-subset node is cost row 0 plus the snapshot rows it keeps, in their original order, then its cut rows as
// addCutConstraints builds them (labels from the snapshot's lastElementIndex), then the reference's phase 1
// (simplex.ts:25-98) with the cycle check on, then, with an integer mask, the isIntegral / getMostFractionalVar scan
// restricted to it.  Every slack is basic in the initial tableau, so dropping a constraint is dropping its row.  Nodes
// whose kept rows plus cuts fit shared memory run one CTA each in k_node_batch<NODE_CONFLICT>; the others (and any node
// that hits the in-kernel pivot or log cap) run one after another on the single-tableau path: k_gather_rows,
// jslp_add_cuts, run_lp (phase 1), k_mip_scan_masked, read_column.
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

// The masked isIntegral / getMostFractionalVar scan of the current tableau (the single-tableau path).
__global__ void __launch_bounds__(256) k_mip_scan_masked(const TabDev *Tp, MipOut *out, const uint32_t *imask) {
    __shared__ RedSmem red;
    __shared__ TabDev T;
    if (threadIdx.x == 0) T = *Tp;
    __syncthreads();
    cta_mip_scan<true>(T, out, red, imask);
}

}  // namespace jslp

// ---- row-subset batches (jslp_feasibility_batch, jslp_conflict_batch) ------------------------------------------------

enum { SUBSET_FEASIBLE = 0, SUBSET_INFEASIBLE = 1, SUBSET_CYCLED = 2 };

// Cost row 0 plus the snapshot rows a keep mask of H0 bytes keeps (row 0 always).
static int kept_height(const uint8_t *keep, int H0) {
    int h = 1;
    for (int r = 1; r < H0; r++) h += keep[r] != 0;
    return h;
}

// A batch of row-subset nodes of the snapshot, and where their results go.  Node i keeps the rows of keep[i * H0 ..];
// with cuts set, cuts[cut_off[i] .. cut_off[i + 1]) follow them; height[i] counts both and the cost row.  With int_keep
// set (n_int bytes per node) the scan runs over the node's integer mask.  status and pivots are per node (pivots may be
// null); with is_integral set, is_integral / branch_var / branch_value too; with rhs set, column 0 and the row labels of
// every node that did not cycle go to rhs / vrow + i * row_stride.
struct SubsetBatch {
    const uint8_t *keep = nullptr, *int_keep = nullptr;
    const jslp_cut *cuts = nullptr;
    const int32_t *cut_off = nullptr;
    const int *height = nullptr;
    int32_t *status = nullptr, *pivots = nullptr, *is_integral = nullptr, *branch_var = nullptr;
    double *branch_value = nullptr, *rhs = nullptr;
    int32_t *vrow = nullptr;
    int row_stride = 0;
    int cuts_of(int i) const { return cuts ? cut_off[i + 1] - cut_off[i] : 0; }
    void set(int i, int st, int integral, int bvar, double bval, int piv) const {
        status[i] = st;
        if (pivots) pivots[i] = piv;
        if (!is_integral) return;
        is_integral[i] = st == SUBSET_FEASIBLE ? integral : 0;
        branch_var[i] = st == SUBSET_FEASIBLE && !integral ? bvar : -1;
        branch_value[i] = st == SUBSET_FEASIBLE && !integral ? bval : 0.0;
    }
};

// Node i on the single-tableau path: its rows gathered from the snapshot over the current buffer (every row phase 1
// reads is written), the snapshot's column labels, height and label counters, then its cuts, phase 1, the scan and the
// column as the batch asks.  No snapshot copy per node: the caller restores the snapshot at the end of the batch.
static int subset_hbm(jslp_tab *t, const SubsetBatch &b, int i) {
    const int H0 = t->saved.H, nc = b.cuts_of(i);
    if (b.height[i] == 1 && !b.int_keep && !b.rhs) {  // no row: phase 1 finds no leaving row
        b.set(i, SUBSET_FEASIBLE, 1, -1, 0.0, 0);
        return JSLP_OK;
    }
    std::vector<int> rows;
    for (int r = 0; r < H0; r++)
        if (r == 0 || b.keep[(size_t)i * H0 + r]) rows.push_back(r);
    const int n = (int)rows.size();
    const std::vector<uint32_t> imask =
        b.int_keep ? pack_bits(b.int_keep, t->n_int, &i, 1, (t->n_int + 31) / 32) : std::vector<uint32_t>();
    ScratchLayout L;
    const size_t b_rows = L.take(sizeof(int) * (size_t)n), b_mask = L.take(sizeof(uint32_t) * imask.size());
    int rc = batch_scratch(t, L.bytes);
    if (rc) return rc;
    cudaStream_t s = t->ctx->stream;
    int *d_rows = (int *)((char *)t->d_scratch + b_rows);
    uint32_t *d_mask = (uint32_t *)((char *)t->d_scratch + b_mask);
    CK(cudaMemcpyAsync(d_rows, rows.data(), sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, s));
    if (!imask.empty())
        CK(cudaMemcpyAsync(d_mask, imask.data(), sizeof(uint32_t) * imask.size(), cudaMemcpyHostToDevice, s));
    k_gather_rows<<<std::min(n, t->ctx->num_sms * 4), 256, 0, s>>>(t->hd.M, t->hd.vrow, t->saved.M, t->saved.vrow,
                                                                   t->stride, d_rows, n);
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(t->hd.vcol, t->saved.vcol, sizeof(int) * (size_t)t->W, cudaMemcpyDeviceToDevice, s));
    t->H = n; t->nVars = t->saved.nVars; t->lastElementIndex = t->saved.lastElementIndex;  // the cut labels start there
    rc = push_desc(t);
    if (rc) return rc;
    if (nc > 0) {
        rc = jslp_add_cuts(t, b.cuts + b.cut_off[i], nc);
        if (rc) return rc;
    }
    int status = SUBSET_FEASIBLE, piv = 0;
    if (t->H > 1) {  // with no row besides the cost row, phase 1 finds no leaving row
        jslp_lp_status st;
        rc = run_lp(t, 1, 1, &st, false);
        if (rc) return rc;
        status = st.cycled ? SUBSET_CYCLED : st.feasible ? SUBSET_FEASIBLE : SUBSET_INFEASIBLE;
        piv = st.phase1_pivots;
    }
    MipOut mo{};
    mo.is_integral = 1;
    mo.var_index = -1;
    if (status == SUBSET_FEASIBLE && b.int_keep && t->hd.intpos != nullptr && t->n_int > 0) {
        k_mip_scan_masked<<<1, 256, 0, s>>>(t->d_T, t->d_mip, d_mask);
        t->ctx->launches += 1;
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(t->h_mip, t->d_mip, sizeof(MipOut), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        mo = *t->h_mip;
    }
    b.set(i, status, mo.is_integral, mo.var_index, mo.value, piv);
    if (status == SUBSET_CYCLED || !b.rhs) return JSLP_OK;
    return read_column(t, 0, b.rhs + (size_t)i * b.row_stride, b.vrow + (size_t)i * b.row_stride);
}

// Nodes idx[0..n) in one k_node_batch<NODE_CONFLICT> launch.  A node whose log shows a cycle is cycled, stopped before
// the pivot that completes the repeat, as the reference's phase 1 stops; a node that hits the pivot or log cap first
// goes to redo.
static int subset_resident(jslp_tab *t, const SubsetBatch &b, const int *idx, int n, std::vector<int> &redo) {
    ResidentBufs &rb = t->rbufs;
    const int H0 = t->saved.H;
    int Hcap = 1;
    for (int k = 0; k < n; k++) Hcap = std::max(Hcap, b.height[idx[k]]);
    NodeBatchDev nb;
    size_t smem = 0;
    int rc = batch_fill(t, t->saved.M, t->saved.vrow, t->saved.vcol, H0, t->saved.lastElementIndex, n, nb, &smem);
    if (rc) return rc;
    rc = batch_cuts(t, b.cuts, b.cut_off, idx, n, nb);
    if (rc) return rc;
    nb.Hcap = Hcap;  // kept rows plus cuts: the kernel compacts the kept rows
    smem = node_smem_bytes(Hcap, t->W, nullptr);
    // one device block per launch: keep masks, integer masks, final columns, final labels (the last three as asked)
    const int kw = (H0 + 31) / 32, iw = std::max(1, (t->n_int + 31) / 32);
    const std::vector<uint32_t> kbits = pack_bits(b.keep, H0, idx, n, kw);
    const std::vector<uint32_t> ibits = b.int_keep ? pack_bits(b.int_keep, t->n_int, idx, n, iw) : std::vector<uint32_t>();
    const size_t n_out = b.rhs ? (size_t)n * Hcap : 0;
    ScratchLayout L;
    const size_t b_keep = L.take(sizeof(uint32_t) * kbits.size()), b_int = L.take(sizeof(uint32_t) * ibits.size());
    const size_t b_rhs = L.take(sizeof(double) * n_out), b_vrow = L.take(sizeof(int) * n_out);
    rc = batch_scratch(t, L.bytes);
    if (rc) return rc;
    char *base = (char *)t->d_scratch;
    cudaStream_t s = t->ctx->stream;
    CK(cudaMemcpyAsync(base + b_keep, kbits.data(), sizeof(uint32_t) * kbits.size(), cudaMemcpyHostToDevice, s));
    nb.keep = (const uint32_t *)(base + b_keep); nb.keep_words = kw;
    if (b.int_keep) {
        CK(cudaMemcpyAsync(base + b_int, ibits.data(), sizeof(uint32_t) * ibits.size(), cudaMemcpyHostToDevice, s));
        nb.int_keep = (const uint32_t *)(base + b_int); nb.int_words = iw;
    }
    if (b.rhs) { nb.out_rhs = (double *)(base + b_rhs); nb.out_vrow = (int *)(base + b_vrow); }
    std::vector<double> rhs(n_out);
    std::vector<int32_t> vrow(n_out);
    rc = batch_launch<NODE_CONFLICT>(t, nb, n, smem, rhs.data(), vrow.data());
    if (rc) return rc;
    // phase 1 keeps its own history (simplex.ts:27): every entry of these logs is a phase-1 entry
    std::vector<int> hit;
    rc = batch_screen(t, n, [](int) { return true; }, hit);
    if (rc) return rc;
    for (int k = 0; k < n; k++) {
        const NodeResult &r = rb.h_out[k].r;
        const int i = idx[k];
        if (hit[k] >= 0) { b.set(i, SUBSET_CYCLED, 0, -1, 0.0, hit[k]); continue; }
        if (r.overflow) { redo.push_back(i); continue; }
        const int st = r.status == ST_P1_DONE ? SUBSET_FEASIBLE : SUBSET_INFEASIBLE;
        b.set(i, st, r.is_integral, r.branch_var, r.branch_value, r.p1);
        if (!b.rhs) continue;
        memcpy(b.rhs + (size_t)i * b.row_stride, rhs.data() + (size_t)k * Hcap, sizeof(double) * (size_t)b.height[i]);
        memcpy(b.vrow + (size_t)i * b.row_stride, vrow.data() + (size_t)k * Hcap, sizeof(int32_t) * (size_t)b.height[i]);
    }
    return JSLP_OK;
}

// Every node of b, routed by batch_route on its height.  Only the column outputs bound a launch: without them every
// resident node runs in one.  The snapshot and the caller's scalar state are restored at the end.
static int subset_batch(jslp_tab *t, int n_nodes, const SubsetBatch &b) {
    CK(cudaSetDevice(t->ctx->device));
    const CallerState caller(t);
    int rc = batch_route(
        t, n_nodes, [&](int i) { return b.height[i]; }, b.rhs != nullptr,
        [&](const int *idx, int m, std::vector<int> &redo) { return subset_resident(t, b, idx, m, redo); },
        [&](int i) { return subset_hbm(t, b, i); });
    const int rc2 = jslp_restore(t);  // device-to-device copies, ordered before every later read on the tab's stream
    if (rc == JSLP_OK) rc = rc2;
    caller.restore(t);
    return rc;
}

// test(S) of DESIGN.md 2c: a row-subset node without cuts, integer mask or column outputs; the verdict is its status.
extern "C" int jslp_feasibility_batch(jslp_tab *t, const uint8_t *keep, int n_sets, int32_t *verdict, int32_t *pivots) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    if (n_sets < 0 || (n_sets > 0 && (!keep || !verdict))) return fail(JSLP_E_INVALID, "bad keep / verdict arguments");
    if (!t->saved.valid) return fail(JSLP_E_INVALID, "feasibility_batch needs a snapshot (jslp_save)");
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, "feasibility_batch: optional objectives are not supported");
    if (n_sets == 0) return JSLP_OK;
    const int H0 = t->saved.H;
    std::vector<int> height((size_t)n_sets);
    for (int i = 0; i < n_sets; i++) height[i] = kept_height(keep + (size_t)i * H0, H0);
    SubsetBatch b;
    b.keep = keep; b.height = height.data();
    b.status = verdict; b.pivots = pivots;
    return subset_batch(t, n_sets, b);
}
