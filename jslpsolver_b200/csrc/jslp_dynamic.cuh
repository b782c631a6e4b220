// jslpsolver_b200/csrc/jslp_dynamic.cuh -- the dynamic-modification API on a device-resident tableau
// (included by jslp_api.cu).
//
// Replaces src/tableau/dynamic-modification.ts:16-55,78-316: after a solve the model may be edited (right-hand
// sides, costs, coefficients, rows and columns added or removed) and re-solved WITHOUT rebuilding and re-uploading
// the tableau.  Every edit is a row or column operation on the tableau as it stands in HBM, done by a small kernel
// with the reference's operand order (difference * entry, then add / subtract: two roundings); the index maps the
// reference keeps on the host (rowByVarIndex / colByVarIndex) are derived from the device's varIndexByRow /
// varIndexByCol when an edit needs them.  None of this is hot: one launch per edit.
#pragma once

namespace jslp {

// dst[c] += alpha * src[c] (add != 0) or dst[c] -= alpha * src[c], c in [0, W)
__global__ void __launch_bounds__(256) k_row_axpy(double *dst, const double *src, double alpha, int W, int add) {
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < W; c += gridDim.x * blockDim.x)
        dst[c] = add ? edit_axpy_add(dst[c], alpha, src[c]) : edit_axpy_sub(dst[c], alpha, src[c]);
}
// M[r][dcol] -= alpha * M[r][scol] for r in [0, H) and for every optional-objective row
__global__ void __launch_bounds__(256) k_col_axpy(const TabDev *Tp, int dcol, int scol, double alpha) {
    const TabDev &T = *Tp;
    const int n = T.H + T.nOpt;
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
        double *row = r < T.H ? T.M + (size_t)r * T.stride : T.opt + (size_t)(r - T.H) * T.stride;
        row[dcol] = edit_axpy_sub(row[dcol], alpha, row[scol]);
    }
}
__global__ void k_entry_sub(double *p, double v) { *p = edit_sub(*p, v); }
__global__ void k_entry_set(double *p, double v) { *p = v; }

// addConstraint (dynamic-modification.ts:162-220): the new row, term by term in the caller's order.
// term_row[k] >= 0: the term's variable is basic in that row; else term_col[k] is its column.
__global__ void __launch_bounds__(256) k_add_constraint(const TabDev *Tp, int row, double sign, double rhs, const int *term_row,
                                                        const int *term_col, const double *term_coef, int n_terms, int slack_index) {
    const TabDev &T = *Tp;
    double *dst = T.M + (size_t)row * T.stride;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < T.stride; c += gridDim.x * blockDim.x) {
        double v = 0.0;
        if (c < T.W) {
            if (c == 0) v = __dmul_rn(sign, rhs);
            for (int k = 0; k < n_terms; k++) {
                const double sc = __dmul_rn(sign, term_coef[k]);
                if (term_row[k] < 0) {
                    if (term_col[k] == c) v = __dadd_rn(v, sc);
                } else {
                    v = __dsub_rn(v, __dmul_rn(sc, T.M[(size_t)term_row[k] * T.stride + c]));
                }
            }
        }
        dst[c] = v;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) T.vrow[row] = slack_index;
}
// removeConstraint (:231-243): swap rows r and last, relabel
__global__ void __launch_bounds__(256) k_swap_rows(const TabDev *Tp, int r, int last) {
    const TabDev &T = *Tp;
    double *a = T.M + (size_t)r * T.stride, *b = T.M + (size_t)last * T.stride;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < T.stride; c += gridDim.x * blockDim.x) {
        const double tmp = b[c];
        b[c] = a[c];
        a[c] = tmp;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) { T.vrow[r] = T.vrow[last]; T.vrow[last] = -1; }
}
// column scol -> column dcol in every row (removeVariable :310-313), or a zero / given first entry (addVariable)
__global__ void __launch_bounds__(256) k_copy_col(const TabDev *Tp, int dcol, int scol, int zero_src) {
    const TabDev &T = *Tp;
    const int n = T.H + T.nOpt;
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
        double *row = r < T.H ? T.M + (size_t)r * T.stride : T.opt + (size_t)(r - T.H) * T.stride;
        if (scol >= 0 && r < T.H) row[dcol] = row[scol];
        else if (scol < 0) row[dcol] = 0.0;
        if (zero_src && scol >= 0) row[scol] = 0.0;   // keeps the padding beyond the logical width zero
    }
    if (blockIdx.x == 0 && threadIdx.x == 0 && scol >= 0) T.vcol[dcol] = T.vcol[scol];
}
__global__ void k_set_vcol(const TabDev *Tp, int col, int label) { Tp->vcol[col] = label; }

}  // namespace jslp

// == the scalar bookkeeping of Tableau the host mirrors: width, height, nVars, lastElementIndex, stride, row capacity
extern "C" int jslp_tab_info(jslp_tab *t, int32_t *out6) {
    if (!t || !out6) return fail(JSLP_E_INVALID, "NULL argument");
    out6[0] = t->W; out6[1] = t->H; out6[2] = t->nVars; out6[3] = t->lastElementIndex; out6[4] = t->stride; out6[5] = t->rowcap;
    return JSLP_OK;
}

// unrestrictedVars / integer position by var index cover indices [0, n): grown when an edit introduces a new index
static int ensure_index_arrays(jslp_tab *t, int n) {
    if (n <= t->n_index) return JSLP_OK;
    cudaStream_t s = t->ctx->stream;
    CK(cudaStreamSynchronize(s));
    if (t->hd.unres) {
        unsigned char *u = nullptr;
        CK(cudaMalloc(&u, (size_t)n));
        CK(cudaMemsetAsync(u, 0, (size_t)n, s));
        CK(cudaMemcpyAsync(u, t->hd.unres, (size_t)t->n_index, cudaMemcpyDeviceToDevice, s));
        CK(cudaStreamSynchronize(s));
        cudaFree(t->hd.unres);
        t->hd.unres = u;
    }
    if (t->hd.intpos) {
        int *p = nullptr;
        CK(cudaMalloc(&p, sizeof(int) * (size_t)n));
        CK(cudaMemsetAsync(p, 0xff, sizeof(int) * (size_t)n, s));
        CK(cudaMemcpyAsync(p, t->hd.intpos, sizeof(int) * (size_t)t->n_index, cudaMemcpyDeviceToDevice, s));
        CK(cudaStreamSynchronize(s));
        cudaFree(t->hd.intpos);
        t->hd.intpos = p;
        t->h_intpos.resize((size_t)n, -1);
    }
    t->n_index = n;
    t->slots.release();  // slot descriptors copy these pointers
    return JSLP_OK;
}

// rowByVarIndex / colByVarIndex of the current tableau (host copies, rebuilt per edit)
struct HostMaps {
    std::vector<int> vrow, vcol;
    int row_of(int v) const { for (size_t r = 1; r < vrow.size(); r++) if (vrow[r] == v) return (int)r; return -1; }
    int col_of(int v) const { for (size_t c = 1; c < vcol.size(); c++) if (vcol[c] == v) return (int)c; return -1; }
};
static int load_maps(jslp_tab *t, HostMaps &m) {
    m.vrow.resize((size_t)t->H);
    m.vcol.resize((size_t)t->W);
    return jslp_download(t, nullptr, nullptr, nullptr, m.vrow.data(), m.vcol.data(), nullptr, nullptr, nullptr);
}

// == Tableau.putInBase (dynamic-modification.ts:16-34)
extern "C" int jslp_put_in_base(jslp_tab *t, int var_index, int *row) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    HostMaps m;
    int rc = load_maps(t, m);
    if (rc) return rc;
    int r = m.row_of(var_index);
    if (r == -1) {
        const int c = m.col_of(var_index);
        if (c < 0) return fail(JSLP_E_INVALID, "putInBase: variable is neither basic nor non-basic");
        std::vector<double> col((size_t)t->H);
        CK(cudaMemcpy2DAsync(col.data(), sizeof(double), t->hd.M + c, sizeof(double) * t->stride, sizeof(double), t->H,
                             cudaMemcpyDeviceToHost, t->ctx->stream));
        CK(cudaStreamSynchronize(t->ctx->stream));
        for (int r1 = 1; r1 < t->H; r1++)
            if (col[r1] < -t->precision || t->precision < col[r1]) { r = r1; break; }
        if (r == -1) return fail(JSLP_E_INVALID, "putInBase: the variable's column has no pivot element");
        rc = jslp_pivot(t, r, c);
        if (rc) return rc;
    }
    if (row) *row = r;
    return JSLP_OK;
}

// == Tableau.takeOutOfBase (:36-55).  The reference bounds its scan by the HEIGHT and indexes the flat matrix, so
// with height > width it reads on into the following rows; restated over the logical (stride == width) layout.
extern "C" int jslp_take_out_of_base(jslp_tab *t, int var_index, int *col) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    HostMaps m;
    int rc = load_maps(t, m);
    if (rc) return rc;
    int c = m.col_of(var_index);
    if (c == -1) {
        const int r = m.row_of(var_index);
        if (r < 0) return fail(JSLP_E_INVALID, "takeOutOfBase: variable is neither basic nor non-basic");
        const int rows = std::min(t->H - r, (t->H - 1) / t->W + 2);
        std::vector<double> flat((size_t)rows * t->W);
        CK(cudaMemcpy2DAsync(flat.data(), sizeof(double) * t->W, t->hd.M + (size_t)r * t->stride, sizeof(double) * t->stride,
                             sizeof(double) * t->W, rows, cudaMemcpyDeviceToHost, t->ctx->stream));
        CK(cudaStreamSynchronize(t->ctx->stream));
        for (int c1 = 1; c1 < t->H && (size_t)c1 < flat.size(); c1++)
            if (flat[c1] < -t->precision || t->precision < flat[c1]) { c = c1; break; }
        if (c == -1 || c >= t->W) return fail(JSLP_E_INVALID, "takeOutOfBase: the variable's row has no pivot element");
        rc = jslp_pivot(t, r, c);
        if (rc) return rc;
    }
    if (col) *col = c;
    return JSLP_OK;
}

// == Tableau.updateRightHandSide (:78-106)
extern "C" int jslp_update_rhs(jslp_tab *t, int constraint_index, double difference) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    HostMaps m;
    int rc = load_maps(t, m);
    if (rc) return rc;
    cudaStream_t s = t->ctx->stream;
    const int row = m.row_of(constraint_index);
    if (row == -1) {
        const int col = m.col_of(constraint_index);
        if (col < 0) return fail(JSLP_E_INVALID, "updateRightHandSide: unknown constraint index");
        k_col_axpy<<<std::max(1, (t->H + t->nOpt + 255) / 256), 256, 0, s>>>(t->d_T, 0, col, difference);
    } else {
        k_entry_sub<<<1, 1, 0, s>>>(t->hd.M + (size_t)row * t->stride, difference);
    }
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    return JSLP_OK;
}

// == Tableau.updateConstraintCoefficient (:108-135)
extern "C" int jslp_update_coefficient(jslp_tab *t, int constraint_index, int var_index, double difference) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    if (constraint_index == var_index)
        return fail(JSLP_E_INVALID, "[Tableau.updateConstraintCoefficient] constraint index should not be equal to variable index !");
    int r = -1;
    int rc = jslp_put_in_base(t, constraint_index, &r);
    if (rc) return rc;
    HostMaps m;
    rc = load_maps(t, m);
    if (rc) return rc;
    cudaStream_t s = t->ctx->stream;
    double *row = t->hd.M + (size_t)r * t->stride;
    const int colVar = m.col_of(var_index);
    if (colVar == -1) {
        const int rowVar = m.row_of(var_index);
        if (rowVar < 0) return fail(JSLP_E_INVALID, "updateConstraintCoefficient: unknown variable index");
        k_row_axpy<<<std::max(1, (t->W + 255) / 256), 256, 0, s>>>(row, t->hd.M + (size_t)rowVar * t->stride, difference, t->W, 1);
    } else {
        k_entry_sub<<<1, 1, 0, s>>>(row + colVar, difference);
    }
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    return JSLP_OK;
}

// == Tableau.updateCost (:137-160); opt_slot = -1 for a priority-0 variable (cost row), else the position of
// objectivesByPriority[variable.priority] in the uploaded optional objectives
extern "C" int jslp_update_cost(jslp_tab *t, int var_index, int opt_slot, double difference) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    if (opt_slot >= t->nOpt) return fail(JSLP_E_INVALID, "updateCost: optional objective out of range");
    HostMaps m;
    int rc = load_maps(t, m);
    if (rc) return rc;
    cudaStream_t s = t->ctx->stream;
    const int col = m.col_of(var_index);
    if (col == -1) {
        const int row = m.row_of(var_index);
        if (row < 0) return fail(JSLP_E_INVALID, "updateCost: unknown variable index");
        double *dst = opt_slot < 0 ? t->hd.M : t->hd.opt + (size_t)opt_slot * t->stride;
        k_row_axpy<<<std::max(1, (t->W + 255) / 256), 256, 0, s>>>(dst, t->hd.M + (size_t)row * t->stride, difference, t->W, 1);
    } else {
        k_entry_sub<<<1, 1, 0, s>>>(t->hd.M + col, difference);  // row 0 (dynamic-modification.ts:158), whatever the priority
    }
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    return JSLP_OK;
}

// == Tableau.addConstraint (:162-220)
extern "C" int jslp_add_constraint(jslp_tab *t, int is_upper_bound, double rhs, int slack_index, const int32_t *term_var,
                                   const double *term_coef, int n_terms) {
    if (!t || n_terms < 0 || (n_terms > 0 && (!term_var || !term_coef))) return fail(JSLP_E_INVALID, "bad argument");
    HostMaps m;
    int rc = load_maps(t, m);
    if (rc) return rc;
    std::vector<int> trow((size_t)std::max(1, n_terms)), tcol((size_t)std::max(1, n_terms));
    for (int k = 0; k < n_terms; k++) {
        trow[k] = m.row_of(term_var[k]);
        tcol[k] = trow[k] < 0 ? m.col_of(term_var[k]) : -1;
        if (trow[k] < 0 && tcol[k] < 0) return fail(JSLP_E_INVALID, "addConstraint: a term's variable is not in the tableau");
    }
    cudaStream_t s = t->ctx->stream;
    const int grid_before = step_grid(t);
    rc = grow_rows(t, t->H + 1);
    if (rc) return rc;
    int *d_i = nullptr;
    double *d_c = nullptr;
    CK(cudaMalloc(&d_i, sizeof(int) * 2 * (size_t)std::max(1, n_terms)));
    CK(cudaMalloc(&d_c, sizeof(double) * (size_t)std::max(1, n_terms)));
    if (n_terms > 0) {
        CK(cudaMemcpyAsync(d_i, trow.data(), sizeof(int) * n_terms, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_i + n_terms, tcol.data(), sizeof(int) * n_terms, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_c, term_coef, sizeof(double) * n_terms, cudaMemcpyHostToDevice, s));
    }
    const int row = t->H;
    t->H += 1;
    t->lastElementIndex = std::max(t->lastElementIndex, slack_index + 1);  // Tableau.getNewElementIndex handed it out
    rc = push_desc(t);
    if (rc) return rc;
    k_add_constraint<<<std::max(1, (t->stride + 255) / 256), 256, 0, s>>>(t->d_T, row, is_upper_bound ? 1.0 : -1.0, rhs, d_i, d_i + n_terms,
                                                                        d_c, n_terms, slack_index);
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(s));
    cudaFree(d_i); cudaFree(d_c);
    if (step_grid(t) != grid_before) drop_graphs(t);
    return JSLP_OK;
}

// == Tableau.removeConstraint (:222-251); availableIndexes / constraint.slack.index are host bookkeeping of the caller
extern "C" int jslp_remove_constraint(jslp_tab *t, int slack_index) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    int r = -1;
    int rc = jslp_put_in_base(t, slack_index, &r);
    if (rc) return rc;
    const int grid_before = step_grid(t);
    k_swap_rows<<<std::max(1, (t->stride + 255) / 256), 256, 0, t->ctx->stream>>>(t->d_T, r, t->H - 1);
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    t->H -= 1;
    rc = push_desc(t);
    if (rc) return rc;
    if (step_grid(t) != grid_before) drop_graphs(t);
    return JSLP_OK;
}

// Re-lays the tableau out with a wider row stride (addVariable past the padded width).
static int restride(jslp_tab *t, int new_stride) {
    cudaStream_t s = t->ctx->stream;
    CK(cudaStreamSynchronize(s));
    const int old = t->stride;
    auto widen2d = [&](double **p, int rows) -> int {
        if (!*p) return JSLP_OK;
        double *n = nullptr;
        CK(cudaMalloc(&n, sizeof(double) * (size_t)rows * new_stride));
        CK(cudaMemsetAsync(n, 0, sizeof(double) * (size_t)rows * new_stride, s));
        CK(cudaMemcpy2DAsync(n, sizeof(double) * new_stride, *p, sizeof(double) * old, sizeof(double) * old, rows, cudaMemcpyDeviceToDevice, s));
        CK(cudaStreamSynchronize(s));
        cudaFree(*p);
        *p = n;
        return JSLP_OK;
    };
    int rc;
    if ((rc = widen2d(&t->hd.M, t->rowcap)) || (rc = widen2d(&t->hd.M2, t->rowcap)) || (rc = widen2d(&t->hd.prow, 1)) ||
        (rc = widen2d(&t->hd.opt, t->nOpt)))
        return rc;
    int *vc = nullptr;
    CK(cudaMalloc(&vc, sizeof(int) * (size_t)new_stride));
    CK(cudaMemsetAsync(vc, 0xff, sizeof(int) * (size_t)new_stride, s));
    CK(cudaMemcpyAsync(vc, t->hd.vcol, sizeof(int) * (size_t)t->W, cudaMemcpyDeviceToDevice, s));
    CK(cudaStreamSynchronize(s));
    cudaFree(t->hd.vcol);
    t->hd.vcol = vc;
    cudaFree(t->hd.optflag);
    CK(cudaMalloc(&t->hd.optflag, (size_t)new_stride));
    t->stride = new_stride;
    free_saved(t->saved);      // snapshots of the old layout are void
    free_snap(t->snaps[0]);
    free_snap(t->snaps[1]);
    free_snap(t->snaps[2]);
    t->slots.release();
    drop_graphs(t);
    t->g_batch = 0;            // graphs bake the stride in: force a rebuild
    return JSLP_OK;
}

// == Tableau.addVariable (:253-302); cost_entry = model.isMinimization ? -variable.cost : variable.cost;
// opt_slot = -1 for priority 0, else the optional objective that receives the cost (setOptionalObjective)
extern "C" int jslp_add_variable(jslp_tab *t, int var_index, double cost_entry, int opt_slot, int is_integer, int is_unrestricted) {
    if (!t || var_index < 0) return fail(JSLP_E_INVALID, "bad argument");
    if (opt_slot >= t->nOpt) return fail(JSLP_E_INVALID, "addVariable: optional objective out of range (new priorities need a re-upload)");
    if ((size_t)(t->W + 1) * 8 > 200 * 1024) return fail(JSLP_E_CAPACITY, "width exceeds the shared-memory pivot-row staging limit");
    int rc;
    if (t->W + 1 > t->stride) {
        rc = restride(t, t->stride + 16);
        if (rc) return rc;
    }
    cudaStream_t s = t->ctx->stream;
    if (is_integer || is_unrestricted) {  // Model.addVariable pushes onto integerVariables / unrestrictedVariables
        if (is_unrestricted && !t->hd.unres) {
            CK(cudaMalloc(&t->hd.unres, (size_t)t->n_index));
            CK(cudaMemsetAsync(t->hd.unres, 0, (size_t)t->n_index, s));
        }
        if (is_integer && !t->hd.intpos) {
            CK(cudaMalloc(&t->hd.intpos, sizeof(int) * (size_t)t->n_index));
            CK(cudaMemsetAsync(t->hd.intpos, 0xff, sizeof(int) * (size_t)t->n_index, s));
            t->h_intpos.assign((size_t)t->n_index, -1);
        }
        rc = ensure_index_arrays(t, var_index + 1);
        if (rc) return rc;
        if (is_unrestricted) {
            const unsigned char one = 1;
            CK(cudaMemcpyAsync(t->hd.unres + var_index, &one, 1, cudaMemcpyHostToDevice, s));
        }
        if (is_integer) {
            const int pos = t->n_int;
            CK(cudaMemcpyAsync(t->hd.intpos + var_index, &pos, sizeof(int), cudaMemcpyHostToDevice, s));
            t->h_intpos[(size_t)var_index] = pos;
            t->n_int += 1;
        }
        CK(cudaStreamSynchronize(s));
    }
    t->lastElementIndex = std::max(t->lastElementIndex, var_index + 1);
    const int col = t->W;
    t->W += 1;
    set_pricing_params(t);
    rc = push_desc(t);
    if (rc) return rc;
    k_copy_col<<<std::max(1, (t->H + t->nOpt + 255) / 256), 256, 0, s>>>(t->d_T, col, -1, 0);  // new column = 0
    if (opt_slot < 0) k_entry_set<<<1, 1, 0, s>>>(t->hd.M + col, cost_entry);
    else k_entry_set<<<1, 1, 0, s>>>(t->hd.opt + (size_t)opt_slot * t->stride + col, cost_entry);
    k_set_vcol<<<1, 1, 0, s>>>(t->d_T, col, var_index);
    t->ctx->launches += 3;
    CK(cudaGetLastError());
    drop_graphs(t);  // pricing parameters changed
    t->g_batch = 0;
    t->slots.release();  // node slots are laid out for one width
    t->saved.valid = false;  // ... and so is a saved snapshot (backup.ts restores `width` with the matrix)
    return JSLP_OK;
}

// == Tableau.removeVariable (:304-316) as the reference intends it: the variable leaves the basis, its column is
// overwritten by the last column, the width shrinks by one.  (The reference only decrements `width` and goes on
// indexing the un-compacted Float64Array with the new width; the device layout keeps its row stride, so rows stay
// where they are.  DESIGN.md lists this as a deliberate difference.)
extern "C" int jslp_remove_variable(jslp_tab *t, int var_index) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    if (t->W <= 2) return fail(JSLP_E_INVALID, "removeVariable: the tableau has one structural column left");
    int c = -1;
    int rc = jslp_take_out_of_base(t, var_index, &c);
    if (rc) return rc;
    cudaStream_t s = t->ctx->stream;
    const int last = t->W - 1;
    k_copy_col<<<std::max(1, (t->H + t->nOpt + 255) / 256), 256, 0, s>>>(t->d_T, c, last, c != last);
    if (c == last) k_copy_col<<<std::max(1, (t->H + t->nOpt + 255) / 256), 256, 0, s>>>(t->d_T, last, -1, 0);
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    t->W -= 1;
    set_pricing_params(t);
    rc = push_desc(t);
    if (rc) return rc;
    drop_graphs(t);
    t->g_batch = 0;
    t->slots.release();
    t->saved.valid = false;
    return JSLP_OK;
}
