// jslpsolver_b200/csrc/jslp_conflict.cuh -- the node LPs of the feasibility searches behind a MIP conflict (included
// by jslp_api.cu after jslp_pool.cuh; no reference counterpart).  DESIGN.md section 2n is the contract; in short, with
// M the saved snapshot (the model's initial tableau), node i is
//
//   cost row 0 plus the rows of M kept by node i, in their original order, followed by the cut rows of i as
//   addCutConstraints builds them (labels from the snapshot's lastElementIndex), then the reference's phase 1 with the
//   cycle check on, then the isIntegral / getMostFractionalVar scan restricted to the integer positions in i's mask.
//
// That is a row-subset node with every part asked for: subset_batch (jslp_iis.cuh) runs the batch.
#pragma once

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
    int rc = batch_check_offsets({cut_offsets}, n_nodes, "conflict_batch", "cut_offsets[0]");
    if (rc) return rc;
    const int H0 = t->saved.H;
    std::vector<int> height((size_t)n_nodes);  // cost row, kept rows and cut rows of each node
    for (int i = 0; i < n_nodes; i++) {
        height[i] = kept_height(keep + (size_t)i * H0, H0) + cut_offsets[i + 1] - cut_offsets[i];
        if (height[i] > row_stride)
            return fail(JSLP_E_INVALID, "conflict_batch: row_stride is below a node's height (kept rows plus cuts)");
    }
    const int n_cuts = cut_offsets[n_nodes];
    if (n_cuts > 0 && !cuts) return fail(JSLP_E_INVALID, "conflict_batch: cuts is NULL");
    rc = pool_check_cuts(t, cuts, n_cuts, "conflict_batch");
    if (rc) return rc;
    SubsetBatch b;
    b.keep = keep; b.int_keep = int_keep; b.cuts = cuts; b.cut_off = cut_offsets; b.height = height.data();
    b.status = status; b.pivots = pivots; b.is_integral = is_integral; b.branch_var = branch_var;
    b.branch_value = branch_value; b.rhs = rhs; b.vrow = vrow; b.row_stride = row_stride;
    return subset_batch(t, n_nodes, b);
}
