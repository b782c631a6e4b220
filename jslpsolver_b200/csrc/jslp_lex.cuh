// jslpsolver_b200/csrc/jslp_lex.cuh -- one step of a lexicographic (hierarchical) objective chain: the optimum of level
// k turned into the starting tableau of level k+1 (included by jslp_api.cu after jslp_bound.cuh; no reference
// counterpart).  DESIGN.md section 2j is the contract; in short, with M the optimal tableau of level k, C the next
// objective by label and t >= 0 the allowance level k may give up:
//
//   t == 0   the section 2h face of M (k_face_plan / k_face_gather), with row 0 = R at the kept columns
//   t > 0    the section 2i bound tableau of M (contiguous copy + k_bound_rows), with row 0 = R at every column
//   R        section 2g's pricing of C against M (k_price_objective, E not written), padding +0
//
// Column 0 is the parent's (plus t in the bound row), so the new tableau starts primal feasible and level k+1 is a
// phase 2 from the previous optimum.  Row 0 is written on the device; only W' and the kept columns leave it.
#pragma once

extern "C" int jslp_lex_next(jslp_tab *t, const double *cost_by_label, double allowance, jslp_tab **next,
                             int32_t *n_keep, int32_t *kept_cols) {
    if (!t || !cost_by_label || !next || !n_keep) return fail(JSLP_E_INVALID, "NULL argument");
    *next = nullptr;
    if (!(allowance >= 0.0) || std::isinf(allowance))
        return fail(JSLP_E_INVALID, "lex_next: the allowance must be finite and >= 0");
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, "lex_next: optional objectives are not supported");
    CK(cudaSetDevice(t->ctx->device));
    cudaStream_t s = t->ctx->stream;
    double *d_cost = nullptr;
    CK(cudaMalloc(&d_cost, sizeof(double) * (size_t)std::max(1, t->n_index)));
    int rc = JSLP_OK;
    cudaError_t e = cudaMemcpyAsync(d_cost, cost_by_label, sizeof(double) * (size_t)t->n_index, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) rc = fail(JSLP_E_CUDA, std::string("lex_next: ") + cudaGetErrorString(e));
    if (rc == JSLP_OK && allowance == 0.0) {
        rc = face_build(t, d_cost, next, n_keep, kept_cols);
    } else if (rc == JSLP_OK) {
        rc = bound_build(t, allowance, d_cost, next);
        if (rc == JSLP_OK) {  // the bound row bans no column
            *n_keep = t->W;
            if (kept_cols)
                for (int c = 0; c < t->W; c++) kept_cols[c] = c;
        }
    }
    cudaFree(d_cost);  // cudaFree waits for the kernels that read it
    return rc;
}
