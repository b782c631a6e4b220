// jslpsolver_b200/csrc/jslp_conflict.cuh -- the node LPs of the feasibility searches behind a MIP conflict (included
// by jslp_api.cu after jslp_pool.cuh; no reference counterpart).  DESIGN.md section 2n is the contract; in short, with
// M the saved snapshot (the model's initial tableau), node i is
//
//   cost row 0 plus the rows of M kept by node i, in their original order, followed by the cut rows of i as
//   addCutConstraints builds them (labels from the snapshot's lastElementIndex), then the reference's phase 1 with the
//   cycle check on, then the isIntegral / getMostFractionalVar scan restricted to the integer positions in i's mask.
//
// Nodes whose kept rows plus cuts fit shared memory run one CTA each in k_node_batch<NODE_CONFLICT>; the others, and
// any node that hits the in-kernel pivot or log cap, run one after another on the single-tableau path: k_gather_rows,
// jslp_add_cuts, run_lp (phase 1), k_mip_scan_masked, read_column.
#pragma once

namespace jslp {

// The masked isIntegral / getMostFractionalVar scan of the current tableau (the single-tableau path).
__global__ void __launch_bounds__(256) k_mip_scan_masked(const TabDev *Tp, MipOut *out, const uint32_t *imask) {
    __shared__ RedSmem red;
    __shared__ TabDev T;
    if (threadIdx.x == 0) T = *Tp;
    __syncthreads();
    cta_mip_scan<true>(T, out, red, imask);
}

}  // namespace jslp

enum { CONFLICT_FEASIBLE = 0, CONFLICT_INFEASIBLE = 1, CONFLICT_CYCLED = 2 };

// What jslp_conflict_batch hands back per node, and where.
struct ConflictOut {
    int32_t *status, *is_integral, *branch_var, *pivots;
    double *branch_value, *rhs;
    int32_t *vrow;
    int row_stride;
    void set(int i, int st, int integral, int bvar, double bval, int piv) {
        status[i] = st;
        is_integral[i] = st == CONFLICT_FEASIBLE ? integral : 0;
        branch_var[i] = st == CONFLICT_FEASIBLE && !integral ? bvar : -1;
        branch_value[i] = st == CONFLICT_FEASIBLE && !integral ? bval : 0.0;
        pivots[i] = piv;
    }
};

// The bit-packed masks of n nodes: bits[k * words + (j >> 5)] bit (j & 31) = bytes[idx[k] * len + j] != 0.
static std::vector<uint32_t> conflict_bits(const uint8_t *bytes, int len, const int *idx, int n, int words) {
    std::vector<uint32_t> bits((size_t)std::max(1, n * words), 0u);
    for (int k = 0; k < n; k++)
        for (int j = 0; j < len; j++)
            if (bytes[(size_t)idx[k] * len + j]) bits[(size_t)k * words + (j >> 5)] |= 1u << (j & 31);
    return bits;
}

// One node on the single-tableau path.  The caller restores the snapshot at the end of the batch.
static int conflict_hbm(jslp_tab *t, const uint8_t *keep, const uint8_t *int_keep, const jslp_cut *cuts, int n_cuts,
                        int i, ConflictOut &o) {
    int rc = jslp_restore(t);  // the snapshot's height, labels and lastElementIndex (the cut labels start there)
    if (rc) return rc;
    const int H0 = t->saved.H;
    std::vector<int> rows;
    for (int r = 0; r < H0; r++)
        if (r == 0 || keep[r]) rows.push_back(r);
    const int n = (int)rows.size(), iw = (t->n_int + 31) / 32;
    const int idx0 = 0;
    const std::vector<uint32_t> imask = conflict_bits(int_keep, t->n_int, &idx0, 1, iw);
    const size_t b_mask = (sizeof(int) * (size_t)n + 15) & ~(size_t)15;
    rc = batch_scratch(t, b_mask + sizeof(uint32_t) * imask.size());
    if (rc) return rc;
    cudaStream_t s = t->ctx->stream;
    int *d_rows = (int *)t->d_scratch;
    uint32_t *d_mask = (uint32_t *)((char *)t->d_scratch + b_mask);
    CK(cudaMemcpyAsync(d_rows, rows.data(), sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_mask, imask.data(), sizeof(uint32_t) * imask.size(), cudaMemcpyHostToDevice, s));
    k_gather_rows<<<std::min(n, t->ctx->num_sms * 4), 256, 0, s>>>(t->hd.M, t->hd.vrow, t->saved.M, t->saved.vrow,
                                                                   t->stride, d_rows, n);
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    t->H = n;
    rc = push_desc(t);
    if (rc) return rc;
    rc = jslp_add_cuts(t, cuts, n_cuts);
    if (rc) return rc;
    int status = CONFLICT_FEASIBLE, piv = 0;
    if (t->H > 1) {  // with no row besides the cost row, phase 1 finds no leaving row
        jslp_lp_status st;
        rc = run_lp(t, 1, 1, &st, false);
        if (rc) return rc;
        status = st.cycled ? CONFLICT_CYCLED : st.feasible ? CONFLICT_FEASIBLE : CONFLICT_INFEASIBLE;
        piv = st.phase1_pivots;
    }
    MipOut mo{};
    mo.is_integral = 1;
    mo.var_index = -1;
    if (status == CONFLICT_FEASIBLE && t->hd.intpos != nullptr && t->n_int > 0) {
        k_mip_scan_masked<<<1, 256, 0, s>>>(t->d_T, t->d_mip, d_mask);
        t->ctx->launches += 1;
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(t->h_mip, t->d_mip, sizeof(MipOut), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        mo = *t->h_mip;
    }
    o.set(i, status, mo.is_integral, mo.var_index, mo.value, piv);
    if (status == CONFLICT_CYCLED) return JSLP_OK;
    return read_column(t, 0, o.rhs + (size_t)i * o.row_stride, o.vrow + (size_t)i * o.row_stride);
}

// Nodes idx[0..n) in one k_node_batch<NODE_CONFLICT> launch.  A node whose log shows a cycle is cycled, stopped before
// the pivot that completes the repeat, as the reference's phase 1 stops; a node that hits the pivot or log cap first
// goes to redo.
static int conflict_resident(jslp_tab *t, const uint8_t *keep, const uint8_t *int_keep, const jslp_cut *cuts,
                             const int32_t *cut_off, const int *idx, const int *height, int n, ConflictOut &o,
                             std::vector<int> &redo) {
    ResidentBufs &rb = t->rbufs;
    const int H0 = t->saved.H;
    int Hcap = 1, totc = 0;
    for (int k = 0; k < n; k++) {
        Hcap = std::max(Hcap, height[idx[k]]);
        totc += cut_off[idx[k] + 1] - cut_off[idx[k]];
    }
    int rc = rb.ensure(n, totc, t->node_log_cap);
    if (rc) return rc;
    NodeBatchDev nb;
    size_t smem = 0;
    rc = batch_fill(t, t->saved.M, t->saved.vrow, t->saved.vcol, H0, t->saved.lastElementIndex, n, nb, &smem);
    if (rc) return rc;
    nb.Hcap = Hcap;  // kept rows plus cuts: the kernel compacts the kept rows
    smem = node_smem_bytes(Hcap, t->W, nullptr);
    // cut rows: mapped host memory, as branch-and-cut's node launches read them
    int c = 0;
    for (int k = 0; k < n; k++) {
        rb.h_off[k] = c;
        for (int h = cut_off[idx[k]]; h < cut_off[idx[k] + 1]; h++, c++) {
            rb.h_cuts[c].type = cuts[h].type; rb.h_cuts[c].var_index = cuts[h].var_index; rb.h_cuts[c].value = cuts[h].value;
        }
    }
    rb.h_off[n] = c;
    nb.cuts = rb.dv_cuts; nb.cut_off = rb.dv_off;
    if (n <= NODE_INLINE_OFF) {
        nb.n_inline = n;
        for (int k = 0; k <= n; k++) nb.cut_off_inline[k] = rb.h_off[k];
    }
    // one device block per chunk: keep masks, integer masks, final columns, final labels
    const int kw = (H0 + 31) / 32, iw = std::max(1, (t->n_int + 31) / 32);
    const std::vector<uint32_t> kbits = conflict_bits(keep, H0, idx, n, kw);
    const std::vector<uint32_t> ibits = conflict_bits(int_keep, t->n_int, idx, n, iw);
    const size_t b_int = (sizeof(uint32_t) * kbits.size() + 15) & ~(size_t)15;
    const size_t b_rhs = b_int + ((sizeof(uint32_t) * ibits.size() + 15) & ~(size_t)15);
    const size_t b_vrow = b_rhs + sizeof(double) * (size_t)n * Hcap;
    rc = batch_scratch(t, b_vrow + sizeof(int) * (size_t)n * Hcap);
    if (rc) return rc;
    char *base = (char *)t->d_scratch;
    cudaStream_t s = t->ctx->stream;
    CK(cudaMemcpyAsync(base, kbits.data(), sizeof(uint32_t) * kbits.size(), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(base + b_int, ibits.data(), sizeof(uint32_t) * ibits.size(), cudaMemcpyHostToDevice, s));
    nb.keep = (const uint32_t *)base; nb.keep_words = kw;
    nb.int_keep = (const uint32_t *)(base + b_int); nb.int_words = iw;
    nb.out_rhs = (double *)(base + b_rhs); nb.out_vrow = (int *)(base + b_vrow);
    std::vector<double> rhs((size_t)n * Hcap);
    std::vector<int32_t> vrow((size_t)n * Hcap);
    rc = batch_launch<NODE_CONFLICT>(t, nb, n, smem, rhs.data(), vrow.data());
    if (rc) return rc;
    bool need_full = false;
    for (int k = 0; k < n; k++) need_full |= rb.h_out[k].r.log_n > NODE_LOG_HEAD;
    rc = batch_fetch_logs(t, n, need_full);
    if (rc) return rc;
    for (int k = 0; k < n; k++) {
        const NodeResult &r = rb.h_out[k].r;
        const int i = idx[k];
        // phase 1 keeps its own history (simplex.ts:27): every entry of this log is a phase-1 entry
        const int hit_at = first_cycle(batch_log(t, k), std::min(r.log_n, t->node_log_cap));
        if (hit_at >= 0) { o.set(i, CONFLICT_CYCLED, 0, -1, 0.0, hit_at); continue; }
        if (r.overflow) { redo.push_back(i); continue; }
        const int st = r.status == ST_P1_DONE ? CONFLICT_FEASIBLE : CONFLICT_INFEASIBLE;
        o.set(i, st, r.is_integral, r.branch_var, r.branch_value, r.p1);
        memcpy(o.rhs + (size_t)i * o.row_stride, rhs.data() + (size_t)k * Hcap, sizeof(double) * (size_t)height[i]);
        memcpy(o.vrow + (size_t)i * o.row_stride, vrow.data() + (size_t)k * Hcap, sizeof(int32_t) * (size_t)height[i]);
    }
    return JSLP_OK;
}

extern "C" int jslp_conflict_batch(jslp_tab *t, const uint8_t *keep, const uint8_t *int_keep, const jslp_cut *cuts,
                                   const int32_t *cut_offsets, int n_nodes, int row_stride, int32_t *status,
                                   int32_t *is_integral, int32_t *branch_var, double *branch_value, int32_t *pivots,
                                   double *rhs, int32_t *vrow) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    if (n_nodes < 0 || (n_nodes > 0 && (!keep || (!int_keep && t->n_int > 0) || !cut_offsets || !status ||
                                        !is_integral || !branch_var || !branch_value || !pivots || !rhs || !vrow)))
        return fail(JSLP_E_INVALID, "conflict_batch: bad keep / offsets / output arguments");
    if (!t->saved.valid) return fail(JSLP_E_INVALID, "conflict_batch needs a snapshot (jslp_save)");
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, "conflict_batch: optional objectives are not supported");
    if (n_nodes == 0) return JSLP_OK;
    if (cut_offsets[0] != 0) return fail(JSLP_E_INVALID, "conflict_batch: cut_offsets[0] must be 0");
    const int H0 = t->saved.H;
    std::vector<int> height((size_t)n_nodes);  // cost row, kept rows and cut rows of each node
    for (int i = 0; i < n_nodes; i++) {
        if (cut_offsets[i + 1] < cut_offsets[i]) return fail(JSLP_E_INVALID, "conflict_batch: offsets must not decrease");
        int h = 1;
        for (int r = 1; r < H0; r++) h += keep[(size_t)i * H0 + r] != 0;
        height[i] = h + cut_offsets[i + 1] - cut_offsets[i];
        if (height[i] > row_stride)
            return fail(JSLP_E_INVALID, "conflict_batch: row_stride is below a node's height (kept rows plus cuts)");
    }
    const int n_cuts = cut_offsets[n_nodes];
    if (n_cuts > 0 && !cuts) return fail(JSLP_E_INVALID, "conflict_batch: cuts is NULL");
    for (int k = 0; k < n_cuts; k++)
        if ((cuts[k].type != 0 && cuts[k].type != 1) || cuts[k].var_index < 0 || cuts[k].var_index >= t->saved.nVars)
            return fail(JSLP_E_INVALID, "conflict_batch: cut type must be 0 (min) or 1 (max), on a label of the snapshot");
    CK(cudaSetDevice(t->ctx->device));
    ConflictOut o{status, is_integral, branch_var, pivots, branch_value, rhs, vrow, row_stride};
    const CallerState caller(t);
    std::vector<int> res, redo;
    int hmax = 1;
    for (int i = 0; i < n_nodes; i++) {
        if (batch_resident(t, height[i])) { res.push_back(i); hmax = std::max(hmax, height[i]); }
        else redo.push_back(i);
    }
    int rc = JSLP_OK;
    const int chunk = batch_chunk(hmax);
    for (size_t k0 = 0; k0 < res.size() && rc == JSLP_OK; k0 += chunk)
        rc = conflict_resident(t, keep, int_keep, cuts, cut_offsets, res.data() + k0, height.data(),
                               (int)std::min<size_t>(chunk, res.size() - k0), o, redo);
    for (size_t k = 0; k < redo.size() && rc == JSLP_OK; k++) {
        const int i = redo[k];
        rc = conflict_hbm(t, keep + (size_t)i * H0, int_keep + (size_t)i * t->n_int, cuts + cut_offsets[i],
                          cut_offsets[i + 1] - cut_offsets[i], i, o);
    }
    const int rc2 = jslp_restore(t);
    if (rc == JSLP_OK) rc = rc2;
    CK(cudaStreamSynchronize(t->ctx->stream));
    caller.restore(t);
    return rc;
}
