// jslpsolver_b200/csrc/jslp_bound.cuh -- the optimum of a solved LP with its objective turned into one bound row, as a
// tableau of its own (included by jslp_api.cu after jslp_face.cuh; no reference counterpart).  DESIGN.md section 2i is
// the contract; in short, with M the final tableau (H x W), t >= 0 the allowance and l* = max(n_index,
// lastElementIndex), the first label neither the label tables nor the cut rows have handed out:
//
//   B ((H+1) x W): rows 1..H-1 = M's rows bit for bit, column 0 included; row 0 = +0 everywhere, padding included;
//   B[H,0] = t, B[H,c] = -M[0,c] for c >= 1 (a sign flip: +0 becomes -0, a NaN stays a NaN), padding +0
//   vrow' = (vrow..., l*), vcol' = vcol; l* restricted and not integer
//
// At the optimum, result(x) = z + sigma * sum_c M[0,c] x_N(c), so D = sum_c (-M[0,c]) x_N(c) is what a point loses
// against the optimum in either sense, and row H is the dictionary row of the slack of D <= t.  Every feasible point
// of B is a plan at most t worse than the optimum, and any objective set on B with jslp_update_cost /
// jslp_scenario_batch is optimised over those plans (Solution.variability(gap=...)).  Rows 1..H-1 are one
// device-to-device copy; k_bound_rows writes rows 0 and H and the new label.  Nothing leaves the device.
#pragma once

namespace jslp {

static constexpr int BOUND_THREADS = 256;  // columns of B's stride per CTA of k_bound_rows

// Rows 0 and H of B and vrow'[H] from row 0 of whichever ping-pong buffer of the parent is current.  Grid: the stride
// of B in tiles of 256 columns, one thread per column, so every element of both rows, the padding included, is
// written exactly once.
__global__ void __launch_bounds__(BOUND_THREADS) k_bound_rows(const TabDev *Tp, double allowance, double *B,
                                                              int bstride, int *vrow_out, int label) {
    const TabDev &T = *Tp;
    const int W = T.W, H = T.H;
    const int c = blockIdx.x * BOUND_THREADS + threadIdx.x;
    if (c >= bstride) return;
    double v = 0.0;
    if (c == 0)
        v = allowance;
    else if (c < W)  // the IEEE sign flip itself, so no NaN is quietened or rewritten on the way
        v = __longlong_as_double(__double_as_longlong(ldg_cg(T.M + c)) ^ (long long)(1ull << 63));
    B[c] = 0.0;
    B[(size_t)H * bstride + c] = v;
    if (c == 0) vrow_out[H] = label;
}

}  // namespace jslp

// Rows [r0, H) of t's current buffer into the same rows of its sibling c, and t's row and column labels.  The
// ping-pong step swaps TabDev.M / M2 on the device, so the source is the device's view of "current".
static int sibling_copy_rows(const jslp_tab *t, jslp_tab *c, int r0) {
    cudaStream_t s = t->ctx->stream;
    const int W = t->W, H = t->H;
    TabDev cur;
    CK(cudaMemcpyAsync(&cur, t->d_T, sizeof(TabDev), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    if (H > r0) {
        if (c->stride == t->stride)
            CK(cudaMemcpyAsync(c->hd.M + (size_t)r0 * c->stride, cur.M + (size_t)r0 * t->stride,
                               sizeof(double) * (size_t)(H - r0) * t->stride, cudaMemcpyDeviceToDevice, s));
        else  // a parent that removeVariable left wider than ceil16(W): its logical width, row by row
            CK(cudaMemcpy2DAsync(c->hd.M + (size_t)r0 * c->stride, sizeof(double) * c->stride,
                                 cur.M + (size_t)r0 * t->stride, sizeof(double) * t->stride, sizeof(double) * W, H - r0,
                                 cudaMemcpyDeviceToDevice, s));
    }
    CK(cudaMemcpyAsync(c->hd.vrow, t->hd.vrow, sizeof(int) * (size_t)H, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(c->hd.vcol, t->hd.vcol, sizeof(int) * (size_t)W, cudaMemcpyDeviceToDevice, s));
    return JSLP_OK;
}

// The bound tableau of t into *out.  With d_cost (a device array of C by label) row 0 is the next objective priced
// against t at every column (k_price_objective, section 2j) instead of +0.
static int bound_build(jslp_tab *t, double allowance, const double *d_cost, jslp_tab **out) {
    jslp_ctx *ctx = t->ctx;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const int W = t->W, H = t->H;
    const int label = first_free_label(t);
    TabOwner b;
    int rc = sibling_create(t, W, H + 1, 1, b);
    if (rc) return rc;
    rc = sibling_copy_rows(t, b.get(), 1);
    if (rc) return rc;
    k_bound_rows<<<(b->stride + BOUND_THREADS - 1) / BOUND_THREADS, BOUND_THREADS, 0, s>>>(t->d_T, allowance, b->hd.M,
                                                                                          b->stride, b->hd.vrow, label);
    ctx->launches += 1;
    CK(cudaGetLastError());
    if (d_cost) {  // over the +0 k_bound_rows wrote at columns 0..W-1; the padding stays +0
        k_price_objective<<<(W + FR_COLS - 1) / FR_COLS, FR_COLS, 0, s>>>(t->d_T, d_cost, nullptr, W, b->hd.M,
                                                                          nullptr);
        ctx->launches += 1;
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(s));
    *out = b.release();
    return JSLP_OK;
}

extern "C" int jslp_bound_create(jslp_tab *t, double allowance, jslp_tab **out) {
    if (!t || !out) return fail(JSLP_E_INVALID, "NULL argument");
    *out = nullptr;
    if (!(allowance >= 0.0) || std::isinf(allowance))
        return fail(JSLP_E_INVALID, "bound_create: the allowance must be finite and >= 0");
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, "bound_create: optional objectives are not supported");
    return bound_build(t, allowance, nullptr, out);
}
