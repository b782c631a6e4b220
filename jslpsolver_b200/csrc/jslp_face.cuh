// jslpsolver_b200/csrc/jslp_face.cuh -- the optimal face of a solved LP as a tableau of its own (included by
// jslp_api.cu; no reference counterpart).  DESIGN.md section 2h is the contract; in short, with M the final tableau
// (H x W) and P its precision:
//
//   column 0 is kept; column c >= 1 is kept iff M[0,c] >= -P && M[0,c] <= P (a NaN entry bans the column)
//   map[k] = the k-th kept column, W' = their number
//   F (H x W'): F[r,k] = M[r,map[k]] bit for bit for r >= 1, row 0 = +0 everywhere, stride ceil16(W'), padding +0
//   vrow' = vrow, vcol'[k] = vcol[map[k]]
//
// With every reduced cost of the right sign, a feasible point is optimal exactly when the banned columns stay at 0, so
// every vertex of F is an optimum of the LP and any objective can be optimised over them (Solution.variability()).
// k_face_plan compacts the kept columns in one CTA; the host reads W' back, creates the sibling tab, and
// k_face_gather fills it.  Nothing but W' (and map[], when the caller asks for it) leaves the device.
#pragma once

namespace jslp {

static constexpr int FACE_PLAN_THREADS = 512;
static constexpr int FACE_PLAN_TILES = 4;   // tiles of 512 columns per pass: their loads are issued together
static constexpr int FACE_TILE = 16;        // gather CTA: 16 columns (one 128-byte line of F) x 16 rows per step
static constexpr int FACE_ROWS = 64;        // rows per gather CTA

// map[k], vcol_out[k] for k < W' and *n_keep = W', in column order.  One CTA: a warp ballot ranks the kept columns of
// a warp, the warp totals are summed in warp order, and the count so far is carried from tile to tile.
__global__ void __launch_bounds__(FACE_PLAN_THREADS) k_face_plan(const TabDev *Tp, int *map, int *vcol_out,
                                                                 int *n_keep) {
    __shared__ TabDev T;
    __shared__ int warp_total[FACE_PLAN_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) T = *Tp;
    __syncthreads();
    const int W = T.W;
    const double prec = T.prec;
    const double *cost = T.M;  // row 0 of whichever ping-pong buffer is current
    int carry = 0;
    for (int c0 = 0; c0 < W; c0 += FACE_PLAN_TILES * FACE_PLAN_THREADS) {
        double v[FACE_PLAN_TILES];
        int lab[FACE_PLAN_TILES];
#pragma unroll
        for (int j = 0; j < FACE_PLAN_TILES; j++) {  // loads of a pass first, then the tests
            const int c = c0 + j * FACE_PLAN_THREADS + tid;
            v[j] = c < W ? ldg_cg(cost + c) : 0.0;
            lab[j] = c < W ? T.vcol[c] : -1;
        }
#pragma unroll
        for (int j = 0; j < FACE_PLAN_TILES; j++) {
            const int c = c0 + j * FACE_PLAN_THREADS + tid;
            const bool keep = c < W && (c == 0 || (v[j] >= -prec && v[j] <= prec));
            const unsigned int votes = __ballot_sync(0xffffffffu, keep);
            if (lane == 0) warp_total[warp] = __popc(votes);
            __syncthreads();
            int before = carry, all = 0;
#pragma unroll
            for (int w = 0; w < FACE_PLAN_THREADS / 32; w++) {
                const int n = warp_total[w];
                if (w < warp) before += n;
                all += n;
            }
            if (keep) {
                const int k = before + __popc(votes & ((1u << lane) - 1u));
                map[k] = c;
                vcol_out[k] = lab[j];
            }
            carry += all;
            __syncthreads();
        }
    }
    if (tid == 0) *n_keep = carry;
}

// F and vrow' from M, vrow and map.  Grid (tiles of 16 columns of F's stride, blocks of FACE_ROWS rows): every element
// of F, row 0 and the stride padding included, is written by exactly one thread from values only, so no grid changes
// the result.  The CTAs of the first column tile copy the row labels.
__global__ void __launch_bounds__(FACE_TILE * FACE_TILE) k_face_gather(const TabDev *Tp, const int *map, int n_keep,
                                                                       double *F, int fstride, int *vrow_out) {
    const TabDev &T = *Tp;
    const int H = T.H;
    const size_t stride = (size_t)T.stride;
    const double *M = T.M;
    const int tx = threadIdx.x % FACE_TILE, ty = threadIdx.x / FACE_TILE;
    const int k = blockIdx.x * FACE_TILE + tx;
    const int r0 = blockIdx.y * FACE_ROWS;
    const int c = k < n_keep ? map[k] : -1;
    double v[FACE_ROWS / FACE_TILE];
#pragma unroll
    for (int j = 0; j < FACE_ROWS / FACE_TILE; j++) {  // the gathers of this thread first, then the stores
        const int r = r0 + j * FACE_TILE + ty;
        v[j] = (c >= 0 && r > 0 && r < H) ? ldg_cg(M + r * stride + c) : 0.0;
    }
#pragma unroll
    for (int j = 0; j < FACE_ROWS / FACE_TILE; j++) {
        const int r = r0 + j * FACE_TILE + ty;
        if (r < H) F[(size_t)r * fstride + k] = v[j];
    }
    if (blockIdx.x == 0 && threadIdx.x < FACE_ROWS && r0 + threadIdx.x < H)
        vrow_out[r0 + threadIdx.x] = T.vrow[r0 + threadIdx.x];
}

}  // namespace jslp

// Owners for what a builder allocates: CK returns early, and a half-built sibling must not outlive the call.
struct TabDestroy { void operator()(jslp_tab *t) const { jslp_tab_destroy(t); } };
struct DevFree { void operator()(void *p) const { cudaFree(p); } };
using TabOwner = std::unique_ptr<jslp_tab, TabDestroy>;

// l* = max(n_index, lastElementIndex): the first label neither the label tables nor the cut rows have handed out.
static int first_free_label(const jslp_tab *t) { return std::max(t->n_index, t->lastElementIndex); }

// A sibling tab of t (jslp_face_create, jslp_bound_create, jslp_elastic_create, jslp_cone_create), W x H in the same
// context, with row capacity max(t's, H).  With new_labels == 0 it has t's labels (nVars, lastElementIndex, n_index);
// otherwise new_labels more, l*..l*+new_labels-1: nVars + new_labels and lastElementIndex = n_index = l* + new_labels,
// so cut rows would take labels after them.  It takes over the unrestricted / integer tables over labels [0, n_index)
// (the new labels restricted and not integer) and every jslp_tab_set_option value, and its descriptor is on the
// device.  The element indices stay the parent's, so a label means the same in both tabs.
static int sibling_create(const jslp_tab *t, int W, int H, int new_labels, TabOwner &child) {
    jslp_tab *f = nullptr;
    int rc = jslp_tab_create(t->ctx, W, H, std::max(t->rowcap, H), t->precision, &f);
    if (rc) return rc;
    child.reset(f);
    if (new_labels == 0) {
        f->nVars = t->nVars; f->lastElementIndex = t->lastElementIndex; f->n_index = t->n_index;
    } else {
        const int label = first_free_label(t);
        f->nVars = t->nVars + new_labels; f->lastElementIndex = label + new_labels; f->n_index = label + new_labels;
    }
    cudaStream_t s = t->ctx->stream;
    const size_t n0 = (size_t)t->n_index, n1 = (size_t)f->n_index;
    if (t->hd.unres) {
        CK(cudaMalloc(&f->hd.unres, n1));
        if (n1 > n0) CK(cudaMemsetAsync(f->hd.unres + n0, 0, n1 - n0, s));
        CK(cudaMemcpyAsync(f->hd.unres, t->hd.unres, n0, cudaMemcpyDeviceToDevice, s));
    }
    if (t->hd.intpos) {
        CK(cudaMalloc(&f->hd.intpos, sizeof(int) * n1));
        if (n1 > n0) CK(cudaMemsetAsync(f->hd.intpos + n0, 0xff, sizeof(int) * (n1 - n0), s));
        CK(cudaMemcpyAsync(f->hd.intpos, t->hd.intpos, sizeof(int) * n0, cudaMemcpyDeviceToDevice, s));
    }
    f->h_intpos = t->h_intpos; f->n_int = t->n_int;
    if (!f->h_intpos.empty() && f->h_intpos.size() < n1) f->h_intpos.resize(n1, -1);
    f->engine = t->engine; f->batch = t->batch; f->host_log_cap = t->host_log_cap;
    f->variant = t->variant; f->grid_per_sm = t->grid_per_sm; f->lookahead = t->lookahead;
    f->timeline_cap = t->timeline_cap; f->pdl = t->pdl; f->pingpong = t->pingpong;
    f->node_slots = t->node_slots; f->node_log_cap = t->node_log_cap; f->slot_steps = t->slot_steps;
    f->slot_variant = t->slot_variant; f->use_mir = t->use_mir;
    return push_desc(f);
}

// The face of t into *face (nullptr when only column 0 is kept).  With d_cost (a device array of C by label) row 0 is
// the next objective priced against t at the kept columns (k_price_objective through map[], section 2j) instead of +0.
static int face_build(jslp_tab *t, const double *d_cost, jslp_tab **face, int32_t *n_keep, int32_t *kept_cols) {
    jslp_ctx *ctx = t->ctx;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const int W = t->W, H = t->H;
    int *d_plan = nullptr;  // map[W], vcol'[W], W'
    CK(cudaMalloc(&d_plan, sizeof(int) * (2 * (size_t)W + 1)));
    const std::unique_ptr<int, DevFree> plan(d_plan);
    int *d_map = d_plan, *d_vcol = d_plan + W, *d_n = d_plan + 2 * (size_t)W;
    int Wk = 0;
    k_face_plan<<<1, FACE_PLAN_THREADS, 0, s>>>(t->d_T, d_map, d_vcol, d_n);
    ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(&Wk, d_n, sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    if (Wk < 1 || Wk > W) return fail(JSLP_E_CUDA, "face_create: the plan kernel returned a bad column count");
    *n_keep = Wk;
    if (kept_cols) {
        CK(cudaMemcpyAsync(kept_cols, d_map, sizeof(int) * (size_t)Wk, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
    }
    if (Wk == 1) return JSLP_OK;  // nothing but column 0: the optimum is the only point of the face
    TabOwner f;
    const int rc = sibling_create(t, Wk, H, 0, f);
    if (rc) return rc;
    CK(cudaMemcpyAsync(f->hd.vcol, d_vcol, sizeof(int) * (size_t)Wk, cudaMemcpyDeviceToDevice, s));
    const dim3 grid((unsigned)(f->stride / FACE_TILE), (unsigned)((H + FACE_ROWS - 1) / FACE_ROWS));
    k_face_gather<<<grid, FACE_TILE * FACE_TILE, 0, s>>>(t->d_T, d_map, Wk, f->hd.M, f->stride, f->hd.vrow);
    ctx->launches += 1;
    CK(cudaGetLastError());
    if (d_cost) {  // over the +0 the gather wrote at the kept columns; the padding stays +0
        k_price_objective<<<(Wk + FR_COLS - 1) / FR_COLS, FR_COLS, 0, s>>>(t->d_T, d_cost, d_map, Wk, f->hd.M,
                                                                           nullptr);
        ctx->launches += 1;
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(s));
    *face = f.release();
    return JSLP_OK;
}

extern "C" int jslp_face_create(jslp_tab *t, jslp_tab **face, int32_t *n_keep, int32_t *kept_cols) {
    if (!t || !face || !n_keep) return fail(JSLP_E_INVALID, "NULL argument");
    *face = nullptr;
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, "face_create: optional objectives are not supported");
    return face_build(t, nullptr, face, n_keep, kept_cols);
}
