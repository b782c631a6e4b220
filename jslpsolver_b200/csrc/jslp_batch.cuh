// jslpsolver_b200/csrc/jslp_batch.cuh -- the host side of k_node_batch launches, shared by branch and cut
// (jslp_bnb.cuh, jslp_forest.cuh) and the analysis batches (jslp_feasibility_batch, jslp_conflict_batch,
// jslp_scenario_batch, jslp_column_batch, jslp_pool_batch, jslp_target_batch).  Included by jslp_api.cu just before
// jslp_bnb.cuh.  Each caller keeps its own flow, its own single-tableau path and its own verdicts; what is here is the
// shared-memory budget of a node, the argument checks and scratch layout of a batch, the route-and-redo order of its
// sets, the staging of a launch's inputs, the launch itself and the cycle screen of its logs.
#pragma once

#include <map>
#include <mutex>

static size_t node_smem_bytes(int Hcap, int W, int *Ws_out) {
    const int Ws = (W + 1) & ~1;  // even row stride: 16-byte aligned rows (TMA restore)
    if (Ws_out) *Ws_out = Ws;
    return sizeof(double) * ((size_t)Hcap * Ws + 2 * (size_t)Ws + Hcap + 1) + sizeof(CutDev) * (size_t)Hcap +
           sizeof(int) * (2 * (size_t)Hcap + W) + 16;
}

static bool resident_fits(const jslp_tab *t, int Hcap) {
    return t->nOpt == 0 && node_smem_bytes(Hcap, t->W, nullptr) <= (size_t)t->ctx->max_smem_optin - 4096;
}

// One grow-only device block per tab for the per-call inputs and outputs of the analysis batches; none of them holds it
// across a call of another.
static int batch_scratch(jslp_tab *t, size_t bytes) {
    if (bytes <= t->scratch_bytes) return JSLP_OK;
    cudaFree(t->d_scratch);
    t->d_scratch = nullptr;
    t->scratch_bytes = 0;
    CK(cudaMalloc(&t->d_scratch, bytes));
    t->scratch_bytes = bytes;
    return JSLP_OK;
}

// The parts of one call's scratch block, each at a 16-byte-aligned offset: take() returns the next part's offset, and
// bytes is what batch_scratch must hold once every part is taken.
struct ScratchLayout {
    size_t bytes = 0;
    size_t take(size_t n) {
        const size_t at = bytes;
        bytes += (n + 15) & ~(size_t)15;
        return at;
    }
};

// The scalar Tableau state and the executed-pivot log describe the caller's tableau, not a batch's sets: captured on
// entry, put back by restore() once the device tableau is restored.
struct CallerState {
    int feasible, bounded, iters, unb;
    double evaluation, best;
    size_t log_size;
    explicit CallerState(const jslp_tab *t)
        : feasible(t->feasible), bounded(t->bounded), iters(t->simplexIters), unb(t->unboundedVar),
          evaluation(t->evaluation), best(t->bestPossibleEval), log_size(t->host_log.size()) {}
    void restore(jslp_tab *t) const {
        t->feasible = feasible; t->bounded = bounded; t->simplexIters = iters; t->unboundedVar = unb;
        t->evaluation = evaluation; t->bestPossibleEval = best;
        if (t->host_log.size() > log_size) t->host_log.resize(log_size);
    }
};

// The offset arrays of a batch of n sets, set i's entries being [off[i], off[i + 1]) of each: every array starts at 0
// (`first` names that entry in the message) and never decreases.
static int batch_check_offsets(std::initializer_list<const int32_t *> offsets, int n, const std::string &what,
                               const char *first = "offsets[0]") {
    for (const int32_t *off : offsets)
        if (off[0] != 0) return fail(JSLP_E_INVALID, what + ": " + first + " must be 0");
    for (int i = 0; i < n; i++)
        for (const int32_t *off : offsets)
            if (off[i + 1] < off[i]) return fail(JSLP_E_INVALID, what + ": offsets must not decrease");
    return JSLP_OK;
}

// The shared-memory node kernel takes a batch of H-row tableaux unless the engine is pinned to 1 or 2; every other
// set runs on the single-tableau path.
static bool batch_resident(const jslp_tab *t, int H) { return t->engine != 1 && t->engine != 2 && resident_fits(t, H); }

// Sets per launch of H-row tableaux: the per-set outputs on the device stay bounded (about 32 MB).
static int batch_chunk(int H) {
    return (int)std::max<size_t>(1, std::min<size_t>(4096, ((size_t)32 << 20) / ((size_t)12 * H)));
}

// The path of each of n sets and the order they run in: set i goes to the node kernel when batch_resident(t,
// height_of(i)), in launches resident(idx, m, redo) of at most batch_chunk(tallest resident height) sets, or of every
// resident set at once when !chunked; single(i) then runs the others one after another, the too-tall sets in index
// order, then the ones the launches put in redo, in launch order.
template <typename HeightOf, typename Resident, typename Single>
static int batch_route(const jslp_tab *t, int n, HeightOf height_of, bool chunked, Resident resident, Single single) {
    std::vector<int> res, redo;
    int hmax = 1;
    for (int i = 0; i < n; i++) {
        const int h = height_of(i);
        if (batch_resident(t, h)) { res.push_back(i); hmax = std::max(hmax, h); }
        else redo.push_back(i);
    }
    const size_t chunk = chunked ? (size_t)batch_chunk(hmax) : std::max<size_t>(1, res.size());
    for (size_t k0 = 0; k0 < res.size(); k0 += chunk) {
        const int rc = resident(res.data() + k0, (int)std::min(chunk, res.size() - k0), redo);
        if (rc) return rc;
    }
    for (const int i : redo) {
        const int rc = single(i);
        if (rc) return rc;
    }
    return JSLP_OK;
}

// The fields of a k_node_batch launch of n sets that do not depend on the mode: the root tableau (M, vrow, vcol; H0
// rows at t's stride, labels handed out from first_index), no room for rows beyond H0, and the records and logs of
// rbufs, sized for n.  *smem = the launch's dynamic shared memory.
static int batch_fill(jslp_tab *t, const double *M, const int *vrow, const int *vcol, int H0, int first_index, int n,
                      NodeBatchDev &nb, size_t *smem) {
    ResidentBufs &rb = t->rbufs;
    int rc = rb.ensure(n, 0, t->node_log_cap);
    if (rc) return rc;
    int Ws = 0;
    *smem = node_smem_bytes(H0, t->W, &Ws);
    memset(&nb, 0, sizeof(nb));
    nb.rootM = M; nb.root_vrow = vrow; nb.root_vcol = vcol;
    nb.out = rb.dv_out; nb.logs = rb.d_logs;
    nb.H0 = H0; nb.root_stride = t->stride; nb.first_index = first_index;
    nb.Hcap = H0; nb.Ws = Ws; nb.log_cap = t->node_log_cap; nb.max_pivots = 100000;
    return JSLP_OK;
}

// The cut rows of n sets to rbufs, where nb reads them: set k's are the cuts_of(k).second rows from cuts_of(k).first,
// in mapped host memory, so that the kernel reads them itself, with the offsets inline in nb as well when they fit.
template <typename CutsOf>
static int stage_cuts(jslp_tab *t, int n, CutsOf cuts_of, NodeBatchDev &nb) {
    ResidentBufs &rb = t->rbufs;
    int totc = 0;
    for (int k = 0; k < n; k++) totc += cuts_of(k).second;
    int rc = rb.ensure(n, totc, t->node_log_cap);
    if (rc) return rc;
    int c = 0;
    for (int k = 0; k < n; k++) {
        rb.h_off[k] = c;
        const std::pair<const jslp_cut *, int> cl = cuts_of(k);
        for (int h = 0; h < cl.second; h++, c++) {
            rb.h_cuts[c].type = cl.first[h].type; rb.h_cuts[c].var_index = cl.first[h].var_index;
            rb.h_cuts[c].value = cl.first[h].value;
        }
    }
    rb.h_off[n] = c;
    nb.cuts = rb.dv_cuts; nb.cut_off = rb.dv_off;
    if (n <= NODE_INLINE_OFF) {
        nb.n_inline = n;
        for (int k = 0; k <= n; k++) nb.cut_off_inline[k] = rb.h_off[k];
    }
    return JSLP_OK;
}

// stage_cuts of sets idx[0..n): set k's are cuts[cut_off[idx[k]] .. cut_off[idx[k] + 1]) (none when cuts is null).
static int batch_cuts(jslp_tab *t, const jslp_cut *cuts, const int32_t *cut_off, const int *idx, int n,
                      NodeBatchDev &nb) {
    return stage_cuts(t, n, [&](int k) {
        return cuts ? std::make_pair(cuts + cut_off[idx[k]], (int)(cut_off[idx[k] + 1] - cut_off[idx[k]]))
                    : std::make_pair(cuts, 0);
    }, nb);
}

// stage_cuts of n branch-and-cut nodes: node k's are branch(k)->cuts.
template <typename BranchOf>
static int branch_cuts(jslp_tab *t, int n, BranchOf branch, NodeBatchDev &nb) {
    return stage_cuts(t, n, [&](int k) {
        const std::vector<jslp_cut> &c = branch(k)->cuts;
        return std::make_pair(c.data(), (int)c.size());
    }, nb);
}

// The bit-packed masks of n sets: bits[k * words + (j >> 5)] bit (j & 31) = bytes[i * len + j] != 0, with i = idx[k]
// (i = k when idx is null).
static std::vector<uint32_t> pack_bits(const uint8_t *bytes, int len, const int *idx, int n, int words) {
    std::vector<uint32_t> bits((size_t)std::max(1, n * words), 0u);
    for (int k = 0; k < n; k++) {
        const uint8_t *b = bytes + (size_t)(idx ? idx[k] : k) * len;
        for (int j = 0; j < len; j++)
            if (b[j]) bits[(size_t)k * words + (j >> 5)] |= 1u << (j & 31);
    }
    return bits;
}

// One k_node_batch<MODE> launch of n sets, waited for; with nb.out_rhs set, the final columns and labels to rhs / vrow
// (n x Hcap).  The dynamic shared-memory limit is an attribute of the kernel on the device, which every tab, context
// and rank thread on it shares: it is kept per (device, mode), only ever raised, and checked and set under one lock.
template <int MODE>
static int batch_launch(jslp_tab *t, const NodeBatchDev &nb, int n, size_t smem, double *rhs, int32_t *vrow) {
    jslp_ctx *ctx = t->ctx;
    cudaStream_t s = ctx->stream;
    {
        static std::mutex mu;
        static std::map<int, size_t> limit;  // device -> the attribute's value
        std::lock_guard<std::mutex> lock(mu);
        size_t &cur = limit[ctx->device];
        if (smem > cur) {
            CK(cudaFuncSetAttribute(k_node_batch<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            cur = smem;
        }
    }
    k_node_batch<MODE><<<n, NODE_THREADS, smem, s>>>(t->d_T, nb);
    ctx->launches += 1;
    CK(cudaGetLastError());
    if (nb.out_rhs) {
        CK(cudaMemcpyAsync(rhs, nb.out_rhs, sizeof(double) * (size_t)n * nb.Hcap, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(vrow, nb.out_vrow, sizeof(int) * (size_t)n * nb.Hcap, cudaMemcpyDeviceToHost, s));
    }
    CK(cudaStreamSynchronize(s));
    return JSLP_OK;
}

// Set i's pivot log: the inline head, or the full log batch_screen brought over; min(log_n, node_log_cap) entries.
static const int4 *batch_log(const jslp_tab *t, int i) {
    const NodeOut &o = t->rbufs.h_out[i];
    return o.r.log_n > NODE_LOG_HEAD ? t->rbufs.h_logs + (size_t)i * t->node_log_cap : o.log_head;
}

// The cycle screen of the last launch's n sets: hit[k] = first_cycle of set k's log (per-phase histories) when
// screened(k), else -1.  The full logs come to the host only when a screened set's log outgrew the inline head.
template <typename Screened>
static int batch_screen(jslp_tab *t, int n, Screened screened, std::vector<int> &hit) {
    const ResidentBufs &rb = t->rbufs;
    bool need_full = false;
    for (int k = 0; k < n; k++) need_full |= screened(k) && rb.h_out[k].r.log_n > NODE_LOG_HEAD;
    if (need_full) {  // rare: a set with a long pivot sequence
        CK(cudaMemcpyAsync(rb.h_logs, rb.d_logs, sizeof(int4) * (size_t)n * t->node_log_cap, cudaMemcpyDeviceToHost,
                           t->ctx->stream));
        CK(cudaStreamSynchronize(t->ctx->stream));
    }
    hit.assign((size_t)n, -1);
    for (int k = 0; k < n; k++)
        if (screened(k)) hit[k] = first_cycle(batch_log(t, k), std::min(rb.h_out[k].r.log_n, t->node_log_cap));
    return JSLP_OK;
}

// Column col of the current buffer to out and, with vrow set, the row labels (H entries each).  The host mirror's M
// is the device's current buffer between calls (run_lp adopts it after every solve).
static int read_column(jslp_tab *t, int col, double *out, int32_t *vrow) {
    cudaStream_t s = t->ctx->stream;
    CK(cudaMemcpy2DAsync(out, sizeof(double), t->hd.M + col, sizeof(double) * t->stride, sizeof(double), t->H,
                         cudaMemcpyDeviceToHost, s));
    if (vrow) CK(cudaMemcpyAsync(vrow, t->hd.vrow, sizeof(int) * (size_t)t->H, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return JSLP_OK;
}
