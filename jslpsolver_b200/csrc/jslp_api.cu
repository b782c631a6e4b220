// jslpsolver_b200/csrc/jslp_api.cu -- C ABI (include/jslp_b200.h) over the sm_90a kernels.
//
// Host-side responsibilities (everything else is on the device):
//   * tableau storage management (padded rows, growth on addCutConstraints)
//   * enqueueing batches of pivot steps as CUDA graphs and polling the pivot record
//   * checkForCycles (simplex.ts:415-440) over the drained pivot log, with snapshot + replay so
//     the final state is the one the reference stops in (it stops BEFORE the repeating pivot)
//   * setEvaluation rounding (tableau.ts:420-430) and the Tableau flag contract
//   * the branch-and-cut frontier (branch-and-cut.ts:54-199, min-heap.ts) -- see jslp_bnb.cuh
#include "../../include/jslp_b200.h"
#include "jslp_kernels.cuh"
#include "jslp_node_kernel.cuh"
#include "jslp_slots.cuh"
#include "jslp_hostmath.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

using namespace jslp;

static thread_local std::string g_err = "";
static int fail(int code, const std::string &msg) {
    g_err = msg;
    return code;
}
#define CK(call)                                                                                 \
    do {                                                                                         \
        cudaError_t e_ = (call);                                                                 \
        if (e_ != cudaSuccess)                                                                   \
            return fail(JSLP_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));        \
    } while (0)

struct jslp_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool owns_stream = false;
    int num_sms = 132;                // H100 SXM; replaced by the device's own properties in jslp_ctx_create
    int max_smem_optin = 48 * 1024;
    int64_t l2_bytes = 50 << 20;
    int64_t launches = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
};

struct Saved {
    bool valid = false;
    int H = 0, nVars = 0, lastElementIndex = 0;
    double *M = nullptr;
    int *vrow = nullptr, *vcol = nullptr;
    double *opt = nullptr;
    int rowcap = 0;
};

struct Snapshot {  // per-batch restart point for cycle rewind
    double *M = nullptr, *opt = nullptr, *prow = nullptr, *pcol = nullptr, *optcoef = nullptr;
    int *vrow = nullptr, *vcol = nullptr;
    Rec *rec = nullptr;
    int rowcap = 0;
};

#include "jslp_frontier.h"
using jslp_bnb::NodeLogEntry;

// Host/device staging for batches of shared-memory-resident node LPs (k_node_batch).
// Buffers of the shared-memory-resident node path.  Inputs (cut lists) and outputs (NodeOut records)
// live in MAPPED pinned host memory: the kernel reads/writes them across PCIe itself, so a round is
// one launch + one stream sync with no copy operations on the stream.
struct ResidentBufs {
    CutDev *h_cuts = nullptr, *dv_cuts = nullptr;   // host pointer / device alias
    int *h_off = nullptr, *dv_off = nullptr;
    NodeOut *h_out = nullptr, *dv_out = nullptr;
    int4 *d_logs = nullptr, *h_logs = nullptr;      // full logs: device memory, fetched only when needed
    int cap_nodes = 0, cap_cuts = 0;
    size_t cap_log_entries = 0;
    void release() {
        cudaFree(d_logs);
        cudaFreeHost(h_cuts); cudaFreeHost(h_off); cudaFreeHost(h_out); cudaFreeHost(h_logs);
        h_cuts = dv_cuts = nullptr; h_off = dv_off = nullptr; h_out = dv_out = nullptr; d_logs = h_logs = nullptr;
        cap_nodes = cap_cuts = 0; cap_log_entries = 0;
    }
    template <typename T>
    static int mapped(T **h, T **d, size_t bytes) {
        CK(cudaHostAlloc((void **)h, bytes, cudaHostAllocMapped));
        CK(cudaHostGetDevicePointer((void **)d, (void *)*h, 0));
        return JSLP_OK;
    }
    int ensure(int n, int totc, int lc) {
        int rc;
        if (n > cap_nodes) {
            const int cn = std::max(64, n * 2);
            cudaFreeHost(h_off); cudaFreeHost(h_out);
            h_off = nullptr; h_out = nullptr;
            if ((rc = mapped(&h_off, &dv_off, sizeof(int) * (size_t)(cn + 1)))) return rc;
            if ((rc = mapped(&h_out, &dv_out, sizeof(NodeOut) * (size_t)cn))) return rc;
            cap_nodes = cn;
        }
        if ((size_t)n * lc > cap_log_entries) {
            const size_t ce = std::max((size_t)64 * 512, (size_t)n * lc * 2);
            cudaFree(d_logs); cudaFreeHost(h_logs);
            d_logs = nullptr; h_logs = nullptr;
            CK(cudaMalloc(&d_logs, sizeof(int4) * ce));
            CK(cudaMallocHost(&h_logs, sizeof(int4) * ce));
            cap_log_entries = ce;
        }
        if (totc > cap_cuts || !h_cuts) {
            const int cc = std::max(1024, totc * 2);
            cudaFreeHost(h_cuts);
            h_cuts = nullptr;
            if ((rc = mapped(&h_cuts, &dv_cuts, sizeof(CutDev) * (size_t)cc))) return rc;
            cap_cuts = cc;
        }
        return JSLP_OK;
    }
};

struct jslp_tab {
    jslp_ctx *ctx = nullptr;
    TabDev hd{};            // host mirror of the device descriptor
    TabDev *d_T = nullptr;
    Rec *d_rec = nullptr;
    Rec *h_rec = nullptr;   // pinned
    int4 *h_log = nullptr;  // pinned, plog_cap entries
    MipOut *d_mip = nullptr, *h_mip = nullptr;
    CutDev *d_cuts = nullptr;
    CutDev *h_cuts = nullptr;
    int cuts_cap = 0;
    int W = 0, H = 0, rowcap = 0, stride = 0, nOpt = 0, n_index = 0, n_int = 0;
    double precision = 1e-8;
    // Tableau scalar state (tableau.ts:59-92)
    int feasible = 1, bounded = 1, simplexIters = 0, unboundedVar = -1;
    int nVars = 0, lastElementIndex = 0;
    double evaluation = 0, bestPossibleEval = 0;
    int isIntegralFlag = 0, bncIterations = 0;
    // options
    int engine = 0, batch = 256;
    int variant = -1 /* auto */, grid_per_sm = 0, lookahead = 1, timeline_cap = 0, part_cap = 0, g_variant = -1, pdl = 0, pingpong = 1;
    int64_t host_log_cap = 0;
    std::vector<int4> host_log;
    // graphs
    // [0 = fused, 1 = two-kernel][kind]: kinds 0..N_KINDS-2 are the geometrically growing first
    // batches of a solve (24, 48, 96, 192 steps), the last kind is the steady-state batch; built lazily
    cudaGraphExec_t graphs[2][5] = {{nullptr, nullptr, nullptr, nullptr, nullptr}, {nullptr, nullptr, nullptr, nullptr, nullptr}};
    int g_batch = 0, g_grid = 0, g_smem = 0;
    cudaEvent_t ev_slot[2] = {nullptr, nullptr};
    Saved saved;
    Snapshot snaps[3];  // one restart point per in-flight batch; [2] = jslp_scenario_batch's source tableau
    std::vector<NodeLogEntry> node_log;
    struct StoredSolution { double evaluation; std::vector<int> vrow; std::vector<double> rhs; };
    std::vector<StoredSolution> solutions;  // keep_solutions (branch-and-cut.ts:143-153)
    int64_t slot_pivots = 0;
    double slot_ms = 0, slot_bytes = 0;
    int64_t cycle_redos_kernel = 0, cycle_redos_slots = 0, cycle_redos_pruned = 0;  // jslp_bnb_status
    ResidentBufs rbufs;
    NodeSlots slots;        // K3: HBM-resident node batch (jslp_slots.cuh)
    int use_mir = 0;        // model.useMIRCuts (JSLP_OPT_USE_MIR_CUTS)
    std::vector<int> h_intpos;  // host copy of TabDev.intpos (computeFractionalVolume runs on the host)
    std::vector<int> h_vrow_upload;  // the row labels of the last jslp_tab_upload (jslp_elastic_create checks them)
    int *d_count = nullptr, *h_count = nullptr;
    int node_slots = -1;    // JSLP_OPT_NODE_SLOTS: -1 = auto, 0 = off (one node at a time), n = at most n slots
    int node_log_cap = 512; // pivot-log entries per node of the shared-memory node kernel (overflow -> HBM path)
    int slot_steps = 32;    // pivots per slot per host poll
    int slot_variant = 12;  // kernel instantiation of the slot batch: flat streaming, 3 CTAs per SM (more row CTAs per slot)
    long long node_kernel_ns = 0;  // sum over rounds of the slowest node CTA (reporting)
    unsigned long long *d_sens = nullptr;  // jslp_sensitivity's key buffers: 2 x sens_cap
    size_t sens_cap = 0;
    // jslp_feasibility_batch / jslp_conflict_batch / jslp_scenario_batch / jslp_column_batch / jslp_pool_batch /
    // jslp_target_batch (batch_scratch): one launch's keep and integer masks, or the gathered row list and integer mask of one node, or
    // one chunk's offsets, resolved edits or fixings; and per-set outputs
    void *d_scratch = nullptr;
    size_t scratch_bytes = 0;
    void *d_param = nullptr, *d_plog = nullptr;  // jslp_parametric: path state and its breakpoint log
    int param_cap = 0;
    cudaGraphExec_t param_graph = nullptr;
    int param_key[3] = {0, 0, 0};  // step grid, shared memory and variant the graph was captured for
    void *d_front = nullptr;  // jslp_frontier: second objective, priced row, carried direction and point slots
    size_t front_bytes = 0;
    void *d_crash = nullptr, *d_crash_buf = nullptr;  // jslp_crash: list state; records, labels and leave mask
    size_t crash_bytes = 0;
    cudaGraphExec_t crash_graph = nullptr;
    int crash_key[3] = {0, 0, 0};
};

extern "C" const char *jslp_last_error(void) { return g_err.c_str(); }
extern "C" int jslp_abi_version(void) { return 2; }

extern "C" int jslp_ctx_create(int device, void *stream, jslp_ctx **out) {
    if (!out) return fail(JSLP_E_INVALID, "out is NULL");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0)
        return fail(JSLP_E_CUDA, std::string("no CUDA device: ") + cudaGetErrorString(e) +
                                     " (libjslp_b200 has no CPU fallback)");
    if (device < 0 || device >= n) return fail(JSLP_E_INVALID, "bad device ordinal");
    CK(cudaSetDevice(device));
    jslp_ctx *c = new jslp_ctx();
    c->device = device;
    cudaDeviceProp p;
    CK(cudaGetDeviceProperties(&p, device));
    c->num_sms = p.multiProcessorCount;
    c->max_smem_optin = (int)p.sharedMemPerBlockOptin;
    c->l2_bytes = p.l2CacheSize > 0 ? (int64_t)p.l2CacheSize : c->l2_bytes;
    if (stream) {
        c->stream = (cudaStream_t)stream;
    } else {
        CK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
        c->owns_stream = true;
    }
    CK(cudaEventCreate(&c->ev0));
    CK(cudaEventCreate(&c->ev1));
    *out = c;
    return JSLP_OK;
}

extern "C" void jslp_ctx_destroy(jslp_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->ev0) cudaEventDestroy(c->ev0);
    if (c->ev1) cudaEventDestroy(c->ev1);
    if (c->owns_stream && c->stream) cudaStreamDestroy(c->stream);
    delete c;
}
extern "C" void *jslp_ctx_stream(jslp_ctx *c) { return c ? (void *)c->stream : nullptr; }
extern "C" int64_t jslp_ctx_launches(jslp_ctx *c) { return c ? c->launches : 0; }
extern "C" int jslp_ctx_sync(jslp_ctx *c) {
    if (!c) return fail(JSLP_E_INVALID, "ctx is NULL");
    CK(cudaStreamSynchronize(c->stream));
    return JSLP_OK;
}

static const int N_KINDS = 5;
static void drop_graphs(jslp_tab *t) {
    for (int e = 0; e < 2; e++)
        for (int k = 0; k < N_KINDS; k++) {
            if (t->graphs[e][k]) cudaGraphExecDestroy(t->graphs[e][k]);
            t->graphs[e][k] = nullptr;
        }
}

static int push_desc(jslp_tab *t) {
    t->hd.W = t->W; t->hd.H = t->H; t->hd.stride = t->stride; t->hd.rowcap = t->rowcap;
    t->hd.nOpt = t->nOpt; t->hd.n_index = t->n_index; t->hd.prec = t->precision;
    CK(cudaMemcpyAsync(t->d_T, &t->hd, sizeof(TabDev), cudaMemcpyHostToDevice, t->ctx->stream));
    // the source is a pageable host struct: the runtime stages it before returning
    return JSLP_OK;
}

// phase-2 partial pricing parameters (simplex.ts:118-127), a function of the current width
static void set_pricing_params(jslp_tab *t) {
    const int nColumns = t->W - 1;
    int bs = (int)std::floor(std::sqrt((double)nColumns));
    bs = std::min(500, std::max(50, bs));
    t->hd.batch_size = bs;
    t->hd.use_partial = nColumns > bs * 2;
}

static int alloc_rows(jslp_tab *t, int rowcap) {
    // (re)allocates every buffer whose size depends on the row capacity, preserving contents
    double *M = nullptr, *M2 = nullptr, *pcol = nullptr;
    int *vrow = nullptr;
    CK(cudaMalloc(&M, sizeof(double) * (size_t)rowcap * t->stride));
    CK(cudaMalloc(&M2, sizeof(double) * (size_t)rowcap * t->stride));  // ping-pong partner
    CK(cudaMalloc(&pcol, sizeof(double) * (size_t)rowcap));
    CK(cudaMalloc(&vrow, sizeof(int) * (size_t)rowcap));
    cudaStream_t s = t->ctx->stream;
    CK(cudaMemsetAsync(M, 0, sizeof(double) * (size_t)rowcap * t->stride, s));
    CK(cudaMemsetAsync(M2, 0, sizeof(double) * (size_t)rowcap * t->stride, s));
    CK(cudaMemsetAsync(pcol, 0, sizeof(double) * (size_t)rowcap, s));
    CK(cudaMemsetAsync(vrow, 0xff, sizeof(int) * (size_t)rowcap, s));
    if (t->hd.M) {
        CK(cudaMemcpyAsync(M, t->hd.M, sizeof(double) * (size_t)t->H * t->stride, cudaMemcpyDeviceToDevice, s));
        CK(cudaMemcpyAsync(vrow, t->hd.vrow, sizeof(int) * (size_t)t->H, cudaMemcpyDeviceToDevice, s));
        CK(cudaStreamSynchronize(s));
        cudaFree(t->hd.M); cudaFree(t->hd.M2); cudaFree(t->hd.pcol); cudaFree(t->hd.vrow);
    }
    t->hd.M = M; t->hd.M2 = M2; t->hd.pcol = pcol; t->hd.vrow = vrow;
    t->rowcap = rowcap;
    return JSLP_OK;
}

extern "C" int jslp_tab_create(jslp_ctx *ctx, int width, int height, int row_capacity, double precision,
                               jslp_tab **out) {
    if (!ctx || !out) return fail(JSLP_E_INVALID, "ctx/out is NULL");
    if (width < 1 || height < 1) return fail(JSLP_E_INVALID, "width/height must be >= 1");
    if (row_capacity < height) row_capacity = height;
    CK(cudaSetDevice(ctx->device));
    jslp_tab *t = new jslp_tab();
    t->ctx = ctx;
    t->W = width; t->H = height; t->precision = precision;
    t->stride = (width + 15) & ~15;  // rows start on 128-byte lines; index math keeps the logical W
    if ((size_t)t->stride * 8 > 200 * 1024) {
        delete t;
        return fail(JSLP_E_CAPACITY, "width exceeds the shared-memory pivot-row staging limit (25600 columns)");
    }
    t->n_index = width + height - 2;
    t->nVars = t->n_index;
    t->lastElementIndex = t->n_index;
    int rc = alloc_rows(t, row_capacity);
    if (rc) { delete t; return rc; }
    CK(cudaMalloc(&t->hd.vcol, sizeof(int) * (size_t)t->stride));  // stride entries: addVariable grows W in place
    CK(cudaMalloc(&t->hd.prow, sizeof(double) * (size_t)t->stride));
    CK(cudaMalloc(&t->hd.optflag, (size_t)t->stride));
    t->hd.plog_cap = 4096;
    CK(cudaMalloc(&t->hd.plog, sizeof(int4) * (size_t)t->hd.plog_cap));
    CK(cudaMalloc(&t->d_T, sizeof(TabDev)));
    CK(cudaMalloc(&t->d_rec, sizeof(Rec)));
    CK(cudaMalloc(&t->d_mip, sizeof(MipOut)));
    CK(cudaMallocHost(&t->h_rec, sizeof(Rec) * 2));  // two read-back slots: batches are double-buffered
    CK(cudaMallocHost(&t->h_log, sizeof(int4) * 2 * (size_t)t->hd.plog_cap));
    CK(cudaEventCreateWithFlags(&t->ev_slot[0], cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&t->ev_slot[1], cudaEventDisableTiming));
    CK(cudaMallocHost(&t->h_mip, sizeof(MipOut)));
    CK(cudaMalloc(&t->d_count, sizeof(int)));
    CK(cudaMallocHost(&t->h_count, sizeof(int)));
    CK(cudaMemsetAsync(t->d_rec, 0, sizeof(Rec), ctx->stream));
    CK(cudaMemsetAsync(t->hd.prow, 0, sizeof(double) * (size_t)t->stride, ctx->stream));
    set_pricing_params(t);
    rc = push_desc(t);
    if (rc) { delete t; return rc; }
    *out = t;
    return JSLP_OK;
}

static void free_saved(Saved &s) {
    cudaFree(s.M); cudaFree(s.vrow); cudaFree(s.vcol); cudaFree(s.opt);
    s = Saved();
}
static void free_snap(Snapshot &s) {
    cudaFree(s.M); cudaFree(s.opt); cudaFree(s.prow); cudaFree(s.pcol); cudaFree(s.optcoef);
    cudaFree(s.vrow); cudaFree(s.vcol); cudaFree(s.rec);
    s = Snapshot();
}

extern "C" void jslp_tab_destroy(jslp_tab *t) {
    if (!t) return;
    cudaSetDevice(t->ctx->device);
    cudaStreamSynchronize(t->ctx->stream);
    drop_graphs(t);
    cudaFree(t->hd.M); cudaFree(t->hd.vrow); cudaFree(t->hd.vcol); cudaFree(t->hd.unres);
    cudaFree(t->hd.opt); cudaFree(t->hd.prow); cudaFree(t->hd.pcol); cudaFree(t->hd.optcoef);
    cudaFree(t->hd.plog); cudaFree(t->hd.optflag); cudaFree(t->hd.intpos);
    cudaFree(t->hd.part); cudaFree(t->hd.dbg); cudaFree(t->hd.M2);
    cudaFree(t->d_T); cudaFree(t->d_rec); cudaFree(t->d_mip); cudaFree(t->d_cuts);
    cudaFreeHost(t->h_rec); cudaFreeHost(t->h_log); cudaFreeHost(t->h_mip); cudaFreeHost(t->h_cuts);
    cudaFree(t->d_count); cudaFreeHost(t->h_count);
    cudaFree(t->d_sens); cudaFree(t->d_scratch);
    cudaFree(t->d_param); cudaFree(t->d_plog); cudaFree(t->d_front);
    if (t->param_graph) cudaGraphExecDestroy(t->param_graph);
    cudaFree(t->d_crash); cudaFree(t->d_crash_buf);
    if (t->crash_graph) cudaGraphExecDestroy(t->crash_graph);
    free_saved(t->saved);
    free_snap(t->snaps[0]);
    free_snap(t->snaps[1]);
    free_snap(t->snaps[2]);
    if (t->ev_slot[0]) cudaEventDestroy(t->ev_slot[0]);
    if (t->ev_slot[1]) cudaEventDestroy(t->ev_slot[1]);
    t->rbufs.release();
    t->slots.release();
    delete t;
}

extern "C" int jslp_tab_upload(jslp_tab *t, const double *matrix, const int32_t *vrow, const int32_t *vcol,
                               const uint8_t *unrestricted, int n_index, const int32_t *int_vars, int n_int,
                               int n_opt, const double *opt_obj) {
    if (!t || !matrix || !vrow || !vcol) return fail(JSLP_E_INVALID, "NULL argument");
    if (n_opt < 0 || n_int < 0) return fail(JSLP_E_INVALID, "negative count");
    CK(cudaSetDevice(t->ctx->device));
    cudaStream_t s = t->ctx->stream;
    CK(cudaMemcpy2DAsync(t->hd.M, sizeof(double) * t->stride, matrix, sizeof(double) * t->W,
                         sizeof(double) * t->W, t->H, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(t->hd.vrow, vrow, sizeof(int) * t->H, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(t->hd.vcol, vcol, sizeof(int) * t->W, cudaMemcpyHostToDevice, s));
    t->h_vrow_upload.assign(vrow, vrow + t->H);
    if (n_index > 0) t->n_index = n_index;
    cudaFree(t->hd.unres); t->hd.unres = nullptr;
    bool any_unres = false;
    if (unrestricted) for (int i = 0; i < t->n_index; i++) any_unres |= unrestricted[i] != 0;
    if (any_unres) {
        CK(cudaMalloc(&t->hd.unres, (size_t)t->n_index));
        CK(cudaMemcpyAsync(t->hd.unres, unrestricted, (size_t)t->n_index, cudaMemcpyHostToDevice, s));
    }
    cudaFree(t->hd.intpos); t->hd.intpos = nullptr;
    t->h_intpos.clear();
    t->n_int = n_int;
    if (n_int > 0) {
        if (!int_vars) return fail(JSLP_E_INVALID, "int_var_indices is NULL");
        std::vector<int> pos((size_t)t->n_index, -1);
        for (int i = 0; i < n_int; i++) {
            if (int_vars[i] < 0 || int_vars[i] >= t->n_index) return fail(JSLP_E_INVALID, "integer var index out of range");
            if (pos[int_vars[i]] < 0) pos[int_vars[i]] = i;
        }
        t->h_intpos = pos;
        CK(cudaMalloc(&t->hd.intpos, sizeof(int) * (size_t)t->n_index));
        CK(cudaMemcpyAsync(t->hd.intpos, pos.data(), sizeof(int) * (size_t)t->n_index, cudaMemcpyHostToDevice, s));
        CK(cudaStreamSynchronize(s));
    }
    cudaFree(t->hd.opt); cudaFree(t->hd.optcoef); t->hd.opt = nullptr; t->hd.optcoef = nullptr;
    t->nOpt = n_opt;
    if (n_opt > 0) {
        if (!opt_obj) return fail(JSLP_E_INVALID, "opt_obj is NULL");
        CK(cudaMalloc(&t->hd.opt, sizeof(double) * (size_t)n_opt * t->stride));
        CK(cudaMalloc(&t->hd.optcoef, sizeof(double) * (size_t)n_opt));
        CK(cudaMemsetAsync(t->hd.opt, 0, sizeof(double) * (size_t)n_opt * t->stride, s));
        CK(cudaMemcpy2DAsync(t->hd.opt, sizeof(double) * t->stride, opt_obj, sizeof(double) * t->W,
                             sizeof(double) * t->W, n_opt, cudaMemcpyHostToDevice, s));
    }
    t->feasible = 1; t->bounded = 1; t->simplexIters = 0; t->unboundedVar = -1;
    t->evaluation = 0; t->bestPossibleEval = 0; t->isIntegralFlag = 0; t->bncIterations = 0;
    t->nVars = t->W + t->H - 2;
    t->lastElementIndex = t->nVars;
    t->saved.valid = false;
    t->slots.release();  // slot descriptors copy unres / intpos / sizes of the tableau they were built for
    int rc = push_desc(t);
    if (rc) return rc;
    CK(cudaStreamSynchronize(s));
    return JSLP_OK;
}

static int n_step_variants();

extern "C" int jslp_tab_set_option(jslp_tab *t, int key, double value) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    switch (key) {
        case JSLP_OPT_ENGINE:
            if (value < 0 || value > 4) return fail(JSLP_E_INVALID, "engine must be 0..4");
            t->engine = (int)value;
            return JSLP_OK;
        case JSLP_OPT_BATCH:
            if (value < 1 || value > 4000) return fail(JSLP_E_INVALID, "batch must be 1..4000");
            t->batch = (int)value;
            return JSLP_OK;
        case JSLP_OPT_PIVOT_LOG_CAP:
            t->host_log_cap = (int64_t)value;
            t->host_log.clear();
            return JSLP_OK;
        case JSLP_OPT_STEP_VARIANT:
            if (value < -1 || value >= n_step_variants()) return fail(JSLP_E_INVALID, "step variant out of range");
            t->variant = (int)value;  // -1 = auto
            return JSLP_OK;
        case JSLP_OPT_GRID_PER_SM:
            if (value < 0 || value > 16) return fail(JSLP_E_INVALID, "grid per SM must be 0..16");
            t->grid_per_sm = (int)value;
            return JSLP_OK;
        case JSLP_OPT_LOOKAHEAD:
            t->lookahead = value != 0;
            return JSLP_OK;
        case JSLP_OPT_PINGPONG:
            t->pingpong = value != 0;
            return JSLP_OK;
        case JSLP_OPT_PDL:
            t->pdl = value != 0;  // programmatic-dependent-launch edges inside the graph (measured: no gain)
            return JSLP_OK;
        case JSLP_OPT_NODE_SLOTS:
            if (value < -1 || value > 64) return fail(JSLP_E_INVALID, "node slots must be -1..64");
            t->node_slots = (int)value;
            return JSLP_OK;
        case JSLP_OPT_NODE_LOG_CAP:
            if (value < 2 || value > 65536) return fail(JSLP_E_INVALID, "node log cap must be 2..65536");
            t->node_log_cap = (int)value;
            return JSLP_OK;
        case JSLP_OPT_USE_MIR_CUTS:
            t->use_mir = value != 0;
            return JSLP_OK;
        case JSLP_OPT_SLOT_VARIANT:
            if (value < 0 || value >= n_step_variants()) return fail(JSLP_E_INVALID, "slot variant out of range");
            t->slot_variant = (int)value;
            return JSLP_OK;
        case JSLP_OPT_SLOT_STEPS:
            if (value < 1 || value > 1024) return fail(JSLP_E_INVALID, "slot steps must be 1..1024");
            t->slot_steps = (int)value;
            return JSLP_OK;
        case JSLP_OPT_TIMELINE:
            if (value < 0 || value > 4096) return fail(JSLP_E_INVALID, "timeline launches must be 0..4096");
            t->timeline_cap = (int)value;
            return JSLP_OK;
    }
    return fail(JSLP_E_INVALID, "unknown option");
}

// Debug: per-CTA timeline of the first `launches` pivot steps of the last solve.  8 int64 per CTA
// per launch: globaltimer at start [ns], cycles to {row staged, rows updated, ticket taken, exit},
// SM id, is-last-CTA, rows owned.
extern "C" int jslp_debug_timeline(jslp_tab *t, int64_t *out, int64_t cap_values, int *launches, int *grid) {
    if (!t || !launches || !grid) return fail(JSLP_E_INVALID, "NULL argument");
    *launches = t->hd.dbg ? t->hd.dbg_cap : 0;
    *grid = t->hd.dbg ? t->hd.dbg_grid : 0;
    if (!out || !t->hd.dbg) return JSLP_OK;
    const int64_t n = std::min<int64_t>(cap_values, (int64_t)8 * t->hd.dbg_grid * t->hd.dbg_cap);
    CK(cudaSetDevice(t->ctx->device));
    CK(cudaMemcpyAsync(out, t->hd.dbg, sizeof(int64_t) * (size_t)n, cudaMemcpyDeviceToHost, t->ctx->stream));
    CK(cudaStreamSynchronize(t->ctx->stream));
    return JSLP_OK;
}

namespace jslp {
// The streaming loop of the pivot step without its arithmetic: every CTA owns one contiguous block, each thread
// keeps 4 + 4 128-bit loads in flight (current batch + prefetched batch), like update_rows_pp.
__global__ void __launch_bounds__(256, 2) k_copy_pairs(const double *src, double *dst, size_t n2) {
    constexpr int K = 4;
    const size_t per = (n2 + gridDim.x - 1) / gridDim.x;
    const size_t lo = per * blockIdx.x, hi = lo + per < n2 ? lo + per : n2;
    const int NT = blockDim.x;
    double2 cur[K], nxt[K];
#pragma unroll
    for (int j = 0; j < K; j++) {
        const size_t i = lo + threadIdx.x + (size_t)j * NT;
        if (i < hi) cur[j] = ld_v2(src + 2 * i);
    }
    for (size_t i0 = lo + threadIdx.x; i0 < hi; i0 += (size_t)K * NT) {
#pragma unroll
        for (int j = 0; j < K; j++) {
            const size_t i = i0 + (size_t)(K + j) * NT;
            if (i < hi) nxt[j] = ld_v2(src + 2 * i);
        }
#pragma unroll
        for (int j = 0; j < K; j++) {
            const size_t i = i0 + (size_t)j * NT;
            if (i < hi) st_v2(dst + 2 * i, cur[j]);
        }
#pragma unroll
        for (int j = 0; j < K; j++) cur[j] = nxt[j];
    }
}
}  // namespace jslp

extern "C" int jslp_debug_copy_gbs(jslp_ctx *ctx, int64_t bytes, int iters, double *gbs) {
    if (!ctx || !gbs || bytes < 16 || iters < 1) return fail(JSLP_E_INVALID, "bad argument");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    double *a = nullptr, *b = nullptr;
    const size_t n2 = (size_t)bytes / 16;
    CK(cudaMalloc(&a, n2 * 16));
    CK(cudaMalloc(&b, n2 * 16));
    CK(cudaMemsetAsync(a, 0, n2 * 16, s));
    CK(cudaMemsetAsync(b, 0, n2 * 16, s));
    const int grid = ctx->num_sms * 2;
    for (int i = 0; i < 3; i++) {  // warm-up: both buffers settle where they will live
        k_copy_pairs<<<grid, 256, 0, s>>>(a, b, n2);
        k_copy_pairs<<<grid, 256, 0, s>>>(b, a, n2);
    }
    CK(cudaEventRecord(ctx->ev0, s));
    for (int i = 0; i < iters; i++) {
        k_copy_pairs<<<grid, 256, 0, s>>>(a, b, n2);
        k_copy_pairs<<<grid, 256, 0, s>>>(b, a, n2);
    }
    CK(cudaEventRecord(ctx->ev1, s));
    CK(cudaEventSynchronize(ctx->ev1));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
    cudaFree(a); cudaFree(b);
    *gbs = 2.0 * iters * 2.0 * (double)(n2 * 16) / (ms * 1e-3) / 1e9;
    return JSLP_OK;
}

// ---------------------------------------------------------------------------------------------
// Instantiations of the fused step: <threads, min CTAs/SM, rows per pass, software prefetch>.
typedef void (*step_fn_t)(TabDev *, Rec *, int, const double *, int);
struct StepVariant {
    step_fn_t fn;      // in-place step (two-kernel engine, optional objectives, more than 32 rows per CTA)
    step_fn_t fn_pp;   // ping-pong step: grid = row CTAs + 2 selector CTAs
    int threads, ctas_per_sm;
    const char *name;
};
#define JSLP_VARIANT(T, O, RC, PF) k_pivot_step<T, O, RC, PF, false>, k_pivot_step<T, O, RC, PF, true>, T, O
static const StepVariant STEP_VARIANTS[] = {
    {JSLP_VARIANT(256, 2, 8, false), "t256 occ2 rc8"},
    {JSLP_VARIANT(256, 2, 4, true), "t256 occ2 rc4 prefetch"},
    {JSLP_VARIANT(256, 4, 4, false), "t256 occ4 rc4"},
    {JSLP_VARIANT(512, 1, 8, false), "t512 occ1 rc8"},
    {JSLP_VARIANT(256, 3, 4, true), "t256 occ3 rc4 prefetch"},
    {JSLP_VARIANT(128, 8, 4, false), "t128 occ8 rc4"},
    {JSLP_VARIANT(256, 2, 4, false), "t256 occ2 rc4"},
    {JSLP_VARIANT(256, 2, 2, true), "t256 occ2 rc2 prefetch"},
    {JSLP_VARIANT(256, 1, 8, false), "t256 occ1 rc8"},
    {JSLP_VARIANT(512, 1, 4, false), "t512 occ1 rc4"},
    {JSLP_VARIANT(256, 2, -4, true), "t256 occ2 flat4 prefetch"},
    {JSLP_VARIANT(256, 2, -8, true), "t256 occ2 flat8 prefetch"},
    {JSLP_VARIANT(256, 3, -4, true), "t256 occ3 flat4 prefetch"},
    {JSLP_VARIANT(256, 4, -2, true), "t256 occ4 flat2 prefetch"},
};
static const int N_STEP_VARIANTS = (int)(sizeof(STEP_VARIANTS) / sizeof(STEP_VARIANTS[0]));
static int n_step_variants() { return N_STEP_VARIANTS; }
static const int SMALL_BATCH = 24;  // steps in the first graph of a solve

// Auto: while the ping-pong pair fits L2 the flat loop with 4 + 4 loads in flight per thread is fastest; beyond that
// the flat loop with 8 + 8 loads in flight wins.  us per pivot on an H100 SXM (700 W), variants 1 (per-row) / 10 / 11,
// two runs: dense 1000^2 9.4 / 9.4 / 9.8; dense 1500^2 10.2-10.3 / 9.6-10.0 / 10.5-10.8; knapsack root 1537x1025
// 9.1-9.2 / 8.7-9.1 / 9.1-9.3; dense 2000^2 18.0-18.1 / 18.8-19.4 / 16.0-16.4; dense 2500^2 41.1 / 39.7 / 36.6
// (scripts/variant_bench.py).
static int variant_index(const jslp_tab *t) {
    if (t->variant >= 0) return t->variant;
    return 16.0 * (double)t->rowcap * t->stride > 0.95 * (double)t->ctx->l2_bytes ? 11 : 10;
}
static const StepVariant &step_variant(const jslp_tab *t) { return STEP_VARIANTS[variant_index(t)]; }

static int step_grid(const jslp_tab *t) {
    const int per_sm = t->grid_per_sm > 0 ? t->grid_per_sm : step_variant(t).ctas_per_sm;
    int g = t->ctx->num_sms * per_sm;
    return std::max(1, std::min(g, t->rowcap));
}

// The ping-pong step applies to a whole solve or not at all (the graph holds one kernel): no optional
// objectives, the second tableau buffer, and at most 32 rows per row CTA (one warp runs the look-ahead).
// The selector CTAs of the ping-pong step wait for messages from every row CTA of the same launch, so the whole
// grid has to be co-resident: checked against the occupancy the runtime reports for this instantiation and its
// dynamic shared memory (a wide tableau stages a long pivot row and may fit one CTA per SM only).  When it is not,
// the in-place step -- which has no intra-launch dependency -- runs instead.
static bool pp_coresident(const jslp_tab *t, int grid) {
    const StepVariant &sv = step_variant(t);
    const int smem = t->stride * 8;
    static thread_local int c_key = -1, c_val = 0;
    const int key = variant_index(t) * 1000003 + smem;
    if (key != c_key) {
        int nb = 0;
        cudaFuncSetAttribute(sv.fn_pp, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, sv.fn_pp, sv.threads, (size_t)smem) != cudaSuccess) nb = 0;
        c_key = key; c_val = nb;
    }
    return (int64_t)c_val * t->ctx->num_sms >= grid;
}

static bool use_pp(const jslp_tab *t) {
    const int grid = step_grid(t);
    if (!(t->pingpong && t->lookahead && t->nOpt == 0 && grid >= 3 && t->hd.M2 != nullptr)) return false;
    if (t->H / (grid - 2) + 1 > 32) return false;
    return pp_coresident(t, grid);
}

// (re)allocates the buffers that depend on the step grid: look-ahead partials, debug timeline
static int ensure_step_bufs(jslp_tab *t, int grid) {
    if (grid > t->part_cap) {
        CK(cudaStreamSynchronize(t->ctx->stream));
        cudaFree(t->hd.part);
        CK(cudaMalloc(&t->hd.part, sizeof(Part) * (size_t)grid));
        t->part_cap = grid;
    }
    if (t->timeline_cap > 0 && (t->hd.dbg == nullptr || t->hd.dbg_grid != grid || t->hd.dbg_cap != t->timeline_cap)) {
        CK(cudaStreamSynchronize(t->ctx->stream));
        cudaFree(t->hd.dbg);
        CK(cudaMalloc(&t->hd.dbg, sizeof(long long) * 8 * (size_t)grid * t->timeline_cap));
        CK(cudaMemsetAsync(t->hd.dbg, 0, sizeof(long long) * 8 * (size_t)grid * t->timeline_cap, t->ctx->stream));
        t->hd.dbg_grid = grid;
        t->hd.dbg_cap = t->timeline_cap;
    } else if (t->timeline_cap == 0 && t->hd.dbg) {
        CK(cudaStreamSynchronize(t->ctx->stream));
        cudaFree(t->hd.dbg);
        t->hd.dbg = nullptr; t->hd.dbg_cap = 0;
    }
    return push_desc(t);
}

// Steps in a batch of kind k.  A solve starts with short batches that double (most node LPs of a
// branch-and-cut end inside them, and every step enqueued past the end of a solve is a wasted launch)
// and settles on the configured batch length.
static int batch_steps(const jslp_tab *t, int kind) {
    return kind >= N_KINDS - 1 ? t->batch : std::min(SMALL_BATCH << kind, std::max(1, t->batch));
}

// Validates the graph cache against the current launch geometry (drops it when stale).
static int build_graphs(jslp_tab *t) {
    const int grid = step_grid(t);
    const int smem = t->stride * 8;
    int rc = ensure_step_bufs(t, grid);
    if (rc) return rc;
    const int key = variant_index(t) + 100 * (t->pdl == 1) + 1000 * (use_pp(t) ? 1 : 0);
    if (t->g_batch == t->batch && t->g_grid == grid && t->g_smem == smem && t->g_variant == key) return JSLP_OK;
    drop_graphs(t);
    CK(cudaFuncSetAttribute(step_variant(t).fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CK(cudaFuncSetAttribute(step_variant(t).fn_pp, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    t->g_batch = t->batch; t->g_grid = grid; t->g_smem = smem; t->g_variant = key;
    return JSLP_OK;
}

// The graph of `kind` for engine index eidx (0 = fused, 1 = two kernels per pivot); captured on first use.
static int get_graph(jslp_tab *t, int eidx, int kind, cudaGraphExec_t *out) {
    if (t->graphs[eidx][kind]) { *out = t->graphs[eidx][kind]; return JSLP_OK; }
    const int grid = step_grid(t);
    const int smem = t->stride * 8;
    cudaStream_t s = t->ctx->stream;
    const StepVariant &sv = step_variant(t);
    // ping-pong step: the last two CTAs of the grid are the selectors
    const bool pp = use_pp(t);
    const int fused_mode = pp ? 2 : 1;
    const step_fn_t step_fused = pp ? sv.fn_pp : sv.fn;
    const int nsteps = batch_steps(t, kind);
    cudaGraph_t g;
    CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    k_batch_begin<<<1, 32, 0, s>>>(t->d_rec);
    if (eidx == 0) {  // fused: one launch per pivot, last CTA selects the next pivot
        k_select<<<1, 512, 0, s>>>(t->d_T, t->d_rec, -1, -1);
        for (int i = 0; i < nsteps; i++) {
            if (t->pdl == 1 && i > 0) {
                // programmatic dependent launch: step i's CTAs are scheduled while step i-1
                // drains and block in griddepcontrol.wait until it has completed
                cudaLaunchConfig_t cfg;
                memset(&cfg, 0, sizeof(cfg));
                cfg.gridDim = dim3(grid); cfg.blockDim = dim3(sv.threads);
                cfg.dynamicSmemBytes = smem; cfg.stream = s;
                cudaLaunchAttribute at[1];
                at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
                at[0].val.programmaticStreamSerializationAllowed = 1;
                cfg.attrs = at; cfg.numAttrs = 1;
                TabDev *a0 = t->d_T; Rec *a1 = t->d_rec; int a2 = fused_mode; const double *a3 = t->hd.prow; int a4 = t->stride;
                void *args[] = {&a0, &a1, &a2, &a3, &a4};
                cudaError_t le = cudaLaunchKernelExC(&cfg, (const void *)step_fused, args);
                if (le != cudaSuccess) {
                    cudaGraph_t junk;
                    cudaStreamEndCapture(s, &junk);
                    return fail(JSLP_E_CUDA, std::string("PDL launch: ") + cudaGetErrorString(le));
                }
            } else {
                step_fused<<<grid, sv.threads, smem, s>>>(t->d_T, t->d_rec, fused_mode, t->hd.prow, t->stride);
            }
        }
    } else {  // two kernels per pivot
        for (int i = 0; i < nsteps; i++) {
            k_select<<<1, 512, 0, s>>>(t->d_T, t->d_rec, -1, -1);
            sv.fn<<<grid, sv.threads, smem, s>>>(t->d_T, t->d_rec, 0, t->hd.prow, t->stride);
        }
    }
    cudaError_t e = cudaStreamEndCapture(s, &g);
    if (e != cudaSuccess) return fail(JSLP_E_CUDA, std::string("graph capture: ") + cudaGetErrorString(e));
    cudaGraphExec_t ge;
    e = cudaGraphInstantiate(&ge, g, 0);
    cudaGraphDestroy(g);
    if (e != cudaSuccess) return fail(JSLP_E_CUDA, std::string("graph instantiate: ") + cudaGetErrorString(e));
    t->graphs[eidx][kind] = ge;
    *out = ge;
    return JSLP_OK;
}

// tableau.ts:420-430
static void set_evaluation(jslp_tab *t, double raw) {
    const double rounded = jslp_round_evaluation(raw, t->precision);
    t->evaluation = rounded;
    if (t->simplexIters == 0) t->bestPossibleEval = rounded;
}

#include "jslp_cycles.h"

static int ensure_snapshot(jslp_tab *t, int slot) {
    Snapshot &sn = t->snaps[slot];
    if (sn.M && sn.rowcap == t->rowcap) return JSLP_OK;
    free_snap(sn);
    CK(cudaMalloc(&sn.M, sizeof(double) * (size_t)t->rowcap * t->stride));
    CK(cudaMalloc(&sn.pcol, sizeof(double) * (size_t)t->rowcap));
    CK(cudaMalloc(&sn.vrow, sizeof(int) * (size_t)t->rowcap));
    CK(cudaMalloc(&sn.vcol, sizeof(int) * (size_t)t->stride));
    CK(cudaMalloc(&sn.prow, sizeof(double) * (size_t)t->stride));
    CK(cudaMalloc(&sn.rec, sizeof(Rec)));
    if (t->nOpt > 0) {
        CK(cudaMalloc(&sn.opt, sizeof(double) * (size_t)t->nOpt * t->stride));
        CK(cudaMalloc(&sn.optcoef, sizeof(double) * (size_t)t->nOpt));
    }
    sn.rowcap = t->rowcap;
    return JSLP_OK;
}

static int snapshot_copy(jslp_tab *t, int slot, bool to_snapshot) {
    Snapshot &sn = t->snaps[slot];
    cudaStream_t s = t->ctx->stream;
    auto cp = [&](void *live, void *snap, size_t bytes) {
        return to_snapshot ? cudaMemcpyAsync(snap, live, bytes, cudaMemcpyDeviceToDevice, s)
                           : cudaMemcpyAsync(live, snap, bytes, cudaMemcpyDeviceToDevice, s);
    };
    // the tableau itself: device-side copy of whichever ping-pong buffer is current at that point
    k_copy_current<<<t->ctx->num_sms * 4, 256, 0, s>>>(t->d_T, sn.M, to_snapshot ? 1 : 0);
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cp(t->hd.pcol, sn.pcol, sizeof(double) * (size_t)t->H));
    CK(cp(t->hd.vrow, sn.vrow, sizeof(int) * (size_t)t->H));
    CK(cp(t->hd.vcol, sn.vcol, sizeof(int) * (size_t)t->W));
    CK(cp(t->hd.prow, sn.prow, sizeof(double) * (size_t)t->stride));
    CK(cp(t->d_rec, sn.rec, sizeof(Rec)));
    if (t->nOpt > 0) {
        CK(cp(t->hd.opt, sn.opt, sizeof(double) * (size_t)t->nOpt * t->stride));
        CK(cp(t->hd.optcoef, sn.optcoef, sizeof(double) * (size_t)t->nOpt));
    }
    return JSLP_OK;
}

static void fill_status(jslp_tab *t, jslp_lp_status *o, const Rec &r, int cycled, int cs, int cl, float ms,
                        int64_t launches, int engine) {
    if (!o) return;
    memset(o, 0, sizeof(*o));
    o->feasible = t->feasible; o->bounded = t->bounded; o->cycled = cycled;
    o->cycle_start = cs; o->cycle_length = cl;
    o->phase1_pivots = r.p1; o->phase2_pivots = r.p2;
    o->unbounded_var_index = t->unboundedVar; o->simplex_iters = t->simplexIters;
    o->width = t->W; o->height = t->H; o->engine = engine;
    o->evaluation_raw = r.eval_raw; o->evaluation = t->evaluation;
    o->best_possible_eval = t->bestPossibleEval;
    o->gpu_ms = ms; o->kernel_launches = launches;
}

static size_t node_smem_bytes(int Hcap, int W, int *Ws_out);
template <int MODE>
static int batch_launch(jslp_tab *t, const NodeBatchDev &nb, int n, size_t smem, double *rhs, int32_t *vrow);
static void finish_lp_flags(jslp_tab *t, int only_phase, int cycled, const Rec &last);

// Engine 4: the whole simplex() of a small tableau in ONE launch, tableau resident in shared
// memory (k_node_batch with a single node and no cuts).  The result is written to the snapshot
// buffers and adopted only if the pivot log shows no cycle; otherwise (or when the in-kernel pivot
// cap is hit) *handled = false and the caller runs the HBM path on the untouched tableau.
static int run_lp_resident(jslp_tab *t, int check_cycles, jslp_lp_status *out, bool timed, bool *handled) {
    *handled = false;
    jslp_ctx *ctx = t->ctx;
    cudaStream_t s = ctx->stream;
    int Ws = 0;
    const size_t smem = node_smem_bytes(t->H, t->W, &Ws);
    if (t->nOpt > 0 || smem > (size_t)ctx->max_smem_optin - 4096) return JSLP_OK;
    int rc = ensure_snapshot(t, 0);
    if (rc) return rc;
    const Snapshot &snap = t->snaps[0];
    const int log_cap = 2048;
    rc = t->rbufs.ensure(1, 0, log_cap);
    if (rc) return rc;
    ResidentBufs &rb = t->rbufs;
    const int64_t launches0 = ctx->launches;
    if (timed) CK(cudaEventRecord(ctx->ev0, s));
    rb.h_off[0] = 0; rb.h_off[1] = 0;
    NodeBatchDev nb;
    memset(&nb, 0, sizeof(nb));
    nb.rootM = t->hd.M; nb.root_vrow = t->hd.vrow; nb.root_vcol = t->hd.vcol;
    nb.cuts = rb.dv_cuts; nb.cut_off = rb.dv_off; nb.out = rb.dv_out; nb.logs = rb.d_logs;
    nb.wb_M = snap.M; nb.wb_vrow = snap.vrow; nb.wb_vcol = snap.vcol;
    nb.H0 = t->H; nb.root_stride = t->stride; nb.first_index = t->lastElementIndex;
    nb.Hcap = t->H; nb.Ws = Ws; nb.log_cap = log_cap; nb.max_pivots = log_cap - 2;
    rc = batch_launch<NODE_BRANCH>(t, nb, 1, smem, nullptr, nullptr);
    if (rc) return rc;
    const NodeResult r = rb.h_out[0].r;
    if (r.overflow || r.log_n > log_cap) return JSLP_OK;
    if (r.log_n <= NODE_LOG_HEAD) {
        memcpy(rb.h_logs, rb.h_out[0].log_head, sizeof(int4) * (size_t)r.log_n);
    } else {
        CK(cudaMemcpyAsync(rb.h_logs, rb.d_logs, sizeof(int4) * (size_t)r.log_n, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
    }
    if (check_cycles && first_cycle(rb.h_logs, r.log_n) >= 0)
        return JSLP_OK;  // exact stop-before-repeat semantics: HBM path
    // adopt the result
    CK(cudaMemcpy2DAsync(t->hd.M, sizeof(double) * t->stride, snap.M, sizeof(double) * t->stride,
                         sizeof(double) * t->W, t->H, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(t->hd.vrow, snap.vrow, sizeof(int) * (size_t)t->H, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(t->hd.vcol, snap.vcol, sizeof(int) * (size_t)t->W, cudaMemcpyDeviceToDevice, s));
    float ms = 0.f;
    if (timed) {
        CK(cudaEventRecord(ctx->ev1, s));
        CK(cudaEventSynchronize(ctx->ev1));
        CK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
    }
    if (t->host_log_cap > 0)  // executed pivots = every selection (the last selection always executes)
        for (int k = 0; k < r.p1 + r.p2 && (int64_t)t->host_log.size() < t->host_log_cap; k++)
            t->host_log.push_back(rb.h_logs[k]);
    Rec last;
    memset(&last, 0, sizeof(last));
    last.status = r.status; last.p1 = r.p1; last.p2 = r.p2; last.unbounded_var = r.unbounded_var;
    last.eval_raw = r.eval_raw;
    t->bounded = 1;
    finish_lp_flags(t, 0, 0, last);
    fill_status(t, out, last, 0, 0, 0, ms, ctx->launches - launches0, 4);
    *handled = true;
    return JSLP_OK;
}

// Runs phase1 and/or phase2 on the device.  only_phase: 0 = simplex(), 1 = phase1(), 2 = phase2().
static int run_lp(jslp_tab *t, int only_phase, int check_cycles, jslp_lp_status *out, bool timed) {
    jslp_ctx *ctx = t->ctx;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    int rc;
    if (only_phase == 0 && (t->engine == 4 || (t->engine == 0 && (size_t)t->H * t->W <= 16384))) {
        bool handled = false;
        rc = run_lp_resident(t, check_cycles, out, timed, &handled);
        if (rc || handled) return rc;
    }
    rc = build_graphs(t);
    if (rc) return rc;
    const int engine = (t->engine == 1) ? 1 : 2;
    const int eidx = engine == 1 ? 1 : 0;
    auto launches_of = [&](int k) { return engine == 1 ? 1 + 2 * (int64_t)batch_steps(t, k) : 2 + (int64_t)batch_steps(t, k); };
    const int64_t launches0 = ctx->launches;
    const int cap = t->hd.plog_cap;

    Rec init;
    memset(&init, 0, sizeof(init));
    init.status = ST_RUNNING;
    init.phase = only_phase == 2 ? 2 : 1;
    init.stop_at = -1;
    init.unbounded_var = -1;
    init.only_phase = only_phase;
    init.lookahead = (engine == 2 && t->lookahead && t->nOpt == 0) ? 1 : 0;
    init.next_c = -1;
    *t->h_rec = init;
    if (timed) CK(cudaEventRecord(ctx->ev0, s));
    CK(cudaMemcpyAsync(t->d_rec, t->h_rec, sizeof(Rec), cudaMemcpyHostToDevice, s));
    // look-ahead partial slots: no stale message may carry a sequence tag of this solve
    if (t->hd.part) CK(cudaMemsetAsync(t->hd.part, 0xff, sizeof(Part) * (size_t)t->part_cap, s));
    CK(cudaStreamSynchronize(s));  // h_rec is reused as the read-back buffer below

    if (only_phase != 2) t->bounded = 1;  // simplex.ts:15
    if (check_cycles) {
        rc = ensure_snapshot(t, 0);
        if (rc) return rc;
        rc = ensure_snapshot(t, 1);
        if (rc) return rc;
    }
    CycleHist hist[2];   // (leaving, entering) per phase call (simplex.ts:27,102)
    long selected = 0;   // selections seen so far in this call
    int cycled = 0, cyc_start = 0, cyc_len = 0;
    Rec last = init;
    // Batches are double-buffered: batch i+1 is enqueued before the host waits for batch i, so the
    // read-back, the cycle check and the launch latency hide behind device work.  Kernels of a batch
    // enqueued after the solve has finished exit at once.
    int kind_of[2] = {0, 0};
    auto enqueue = [&](int slot, int kind) -> int {
        if (check_cycles) {
            int e = snapshot_copy(t, slot, true);
            if (e) return e;
        }
        {
            cudaGraphExec_t ge;
            int e = get_graph(t, eidx, kind, &ge);
            if (e) return e;
            CK(cudaGraphLaunch(ge, s));
        }
        ctx->launches += launches_of(kind);
        CK(cudaMemcpyAsync(t->h_rec + slot, t->d_rec, sizeof(Rec), cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(t->h_log + (size_t)slot * cap, t->hd.plog, sizeof(int4) * (size_t)cap, cudaMemcpyDeviceToHost, s));
        CK(cudaEventRecord(t->ev_slot[slot], s));
        kind_of[slot] = kind;
        return JSLP_OK;
    };
    rc = enqueue(0, 0);
    if (rc) return rc;
    for (int i = 0;; i++) {
        const int slot = i & 1;
        // enqueue the next batch ahead of the wait only once the solve has reached the steady-state
        // batch length; while the batches are still growing the next one is enqueued after the wait
        const bool ahead = i >= N_KINDS - 1;
        if (ahead) {
            rc = enqueue(slot ^ 1, N_KINDS - 1);
            if (rc) return rc;
        }
        CK(cudaEventSynchronize(t->ev_slot[slot]));
        last = t->h_rec[slot];
        const int4 *log = t->h_log + (size_t)slot * cap;
        const int n_new = std::min(last.log_n, cap);
        if (last.log_n > cap) return fail(JSLP_E_CAPACITY, "pivot log overflow inside one batch");
        long hit_at = -1;
        if (check_cycles) {
            for (int k = 0; k < n_new; k++) {
                const int4 e = log[k];
                const int phase = (e.x >> 30) & 1 ? 2 : 1;
                if (hist[phase - 1].push_and_check(((long long)e.z << 32) | (unsigned int)e.w, &cyc_start, &cyc_len)) {
                    cycled = phase;
                    hit_at = selected + k;
                    break;
                }
            }
        }
        if (hit_at >= 0) {
            // The reference returns before executing the pivot that completes the repeat: replay
            // this batch from its snapshot and stop after `hit_at` executed pivots.
            CK(cudaStreamSynchronize(s));
            rc = snapshot_copy(t, slot, false);
            if (rc) return rc;
            CK(cudaMemcpyAsync(t->h_rec + slot, t->d_rec, sizeof(Rec), cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            Rec r = t->h_rec[slot];
            // hit_at selections precede the offending one, so exactly hit_at pivots get executed;
            // a pivot pending in the snapshot was selected in an earlier batch, hence done < hit_at.
            r.stop_at = (int)hit_at;
            t->h_rec[slot] = r;
            if (t->hd.part) CK(cudaMemsetAsync(t->hd.part, 0xff, sizeof(Part) * (size_t)t->part_cap, s));
            CK(cudaMemcpyAsync(t->d_rec, t->h_rec + slot, sizeof(Rec), cudaMemcpyHostToDevice, s));
            CK(cudaStreamSynchronize(s));
            cudaGraphExec_t ge;
            rc = get_graph(t, eidx, kind_of[slot], &ge);
            if (rc) return rc;
            CK(cudaGraphLaunch(ge, s));
            ctx->launches += launches_of(kind_of[slot]);
            CK(cudaMemcpyAsync(t->h_rec + slot, t->d_rec, sizeof(Rec), cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            last = t->h_rec[slot];
            if (t->host_log_cap > 0)
                for (long k = selected; k < hit_at && (int64_t)t->host_log.size() < t->host_log_cap; k++)
                    t->host_log.push_back(log[k - selected]);
            break;
        }
        if (t->host_log_cap > 0)
            for (int k = 0; k < n_new && (int64_t)t->host_log.size() < t->host_log_cap; k++)
                t->host_log.push_back(log[k]);
        selected += n_new;
        if (last.status != ST_RUNNING) {
            if (ahead) CK(cudaStreamSynchronize(s));  // drain the (no-op) batch that was enqueued ahead
            break;
        }
        if (!ahead) {
            rc = enqueue(slot ^ 1, std::min(i + 1, N_KINDS - 1));
            if (rc) return rc;
        }
    }
    {   // the ping-pong step swaps TabDev.M / M2 on the device: adopt the device's view of "current"
        TabDev cur;
        CK(cudaMemcpyAsync(&cur, t->d_T, sizeof(TabDev), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        t->hd.M = cur.M;
        t->hd.M2 = cur.M2;
    }
    float ms = 0.f;
    if (timed) {
        CK(cudaEventRecord(ctx->ev1, s));
        CK(cudaEventSynchronize(ctx->ev1));
        CK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
    }
    if (last.status == ST_ERROR) return fail(JSLP_E_CUDA, "ping-pong step: selector CTA timed out waiting for row CTAs");

    finish_lp_flags(t, only_phase, cycled, last);
    fill_status(t, out, last, cycled, cyc_start, cyc_len, ms, ctx->launches - launches0, engine);
    return JSLP_OK;
}

// Tableau flag contract (simplex.ts:51-54,73-76,90-91,265-269,298-303,317-318)
static void finish_lp_flags(jslp_tab *t, int only_phase, int cycled, const Rec &last) {
    if (cycled) {
        t->feasible = 0;
    } else if (last.status == ST_INFEASIBLE) {
        t->feasible = 0;
    } else if (last.status == ST_P1_DONE) {
        t->feasible = 1;
    } else if (last.status == ST_OPTIMAL) {
        if (only_phase != 2) t->feasible = 1;
        set_evaluation(t, last.eval_raw);
        t->simplexIters += 1;
    } else if (last.status == ST_UNBOUNDED) {
        if (only_phase != 2) t->feasible = 1;
        t->evaluation = -INFINITY;
        t->bounded = 0;
        t->unboundedVar = last.unbounded_var;
    }
}

extern "C" int jslp_simplex(jslp_tab *t, int check_cycles, jslp_lp_status *out) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    return run_lp(t, 0, check_cycles, out, true);
}
extern "C" int jslp_phase1(jslp_tab *t, int check_cycles, jslp_lp_status *out) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    return run_lp(t, 1, check_cycles, out, true);
}
extern "C" int jslp_phase2(jslp_tab *t, int check_cycles, jslp_lp_status *out) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    return run_lp(t, 2, check_cycles, out, true);
}

extern "C" int jslp_pivot(jslp_tab *t, int row, int col) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    if (row < 0 || row >= t->H || col < 0 || col >= t->W) return fail(JSLP_E_INVALID, "pivot index out of range");
    jslp_ctx *ctx = t->ctx;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const int smem = t->stride * 8;
    const int grid = step_grid(t);
    int rc = ensure_step_bufs(t, grid);
    if (rc) return rc;
    const StepVariant &sv = step_variant(t);
    CK(cudaFuncSetAttribute(sv.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    Rec init;
    memset(&init, 0, sizeof(init));
    init.status = ST_RUNNING; init.phase = 2; init.stop_at = -1; init.unbounded_var = -1; init.next_c = -1;
    *t->h_rec = init;
    CK(cudaMemcpyAsync(t->d_rec, t->h_rec, sizeof(Rec), cudaMemcpyHostToDevice, s));
    k_select<<<1, 512, 0, s>>>(t->d_T, t->d_rec, row, col);
    sv.fn<<<grid, sv.threads, smem, s>>>(t->d_T, t->d_rec, 0, t->hd.prow, t->stride);
    ctx->launches += 2;
    CK(cudaGetLastError());
    if (t->host_log_cap > 0) {  // explicit pivots are part of the executed-pivot log
        CK(cudaMemcpyAsync(t->h_log, t->hd.plog, sizeof(int4), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        if ((int64_t)t->host_log.size() < t->host_log_cap) t->host_log.push_back(t->h_log[0]);
    }
    CK(cudaStreamSynchronize(s));
    return JSLP_OK;
}

// backup.ts:49-51 (copy): device snapshot
extern "C" int jslp_save(jslp_tab *t) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    CK(cudaSetDevice(t->ctx->device));
    cudaStream_t s = t->ctx->stream;
    Saved &sv = t->saved;
    if (!sv.M || sv.rowcap < t->H) {
        free_saved(sv);
        CK(cudaMalloc(&sv.M, sizeof(double) * (size_t)t->rowcap * t->stride));
        CK(cudaMalloc(&sv.vrow, sizeof(int) * (size_t)t->rowcap));
        CK(cudaMalloc(&sv.vcol, sizeof(int) * (size_t)t->stride));
        if (t->nOpt > 0) CK(cudaMalloc(&sv.opt, sizeof(double) * (size_t)t->nOpt * t->stride));
        sv.rowcap = t->rowcap;
    }
    CK(cudaMemcpyAsync(sv.M, t->hd.M, sizeof(double) * (size_t)t->H * t->stride, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(sv.vrow, t->hd.vrow, sizeof(int) * (size_t)t->H, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(sv.vcol, t->hd.vcol, sizeof(int) * (size_t)t->W, cudaMemcpyDeviceToDevice, s));
    if (t->nOpt > 0)
        CK(cudaMemcpyAsync(sv.opt, t->hd.opt, sizeof(double) * (size_t)t->nOpt * t->stride, cudaMemcpyDeviceToDevice, s));
    sv.H = t->H; sv.nVars = t->nVars; sv.lastElementIndex = t->lastElementIndex;
    sv.valid = true;
    return JSLP_OK;
}

// backup.ts:53-105: feasible/bounded/evaluation are deliberately not restored
extern "C" int jslp_restore(jslp_tab *t) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    Saved &sv = t->saved;
    if (!sv.valid) return JSLP_OK;
    CK(cudaSetDevice(t->ctx->device));
    cudaStream_t s = t->ctx->stream;
    CK(cudaMemcpyAsync(t->hd.M, sv.M, sizeof(double) * (size_t)sv.H * t->stride, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(t->hd.vrow, sv.vrow, sizeof(int) * (size_t)sv.H, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(t->hd.vcol, sv.vcol, sizeof(int) * (size_t)t->W, cudaMemcpyDeviceToDevice, s));
    if (t->nOpt > 0)
        CK(cudaMemcpyAsync(t->hd.opt, sv.opt, sizeof(double) * (size_t)t->nOpt * t->stride, cudaMemcpyDeviceToDevice, s));
    const bool changed = t->H != sv.H;
    t->H = sv.H; t->nVars = sv.nVars; t->lastElementIndex = sv.lastElementIndex;
    if (changed) return push_desc(t);
    return JSLP_OK;
}

static int grow_rows(jslp_tab *t, int need) {
    if (need <= t->rowcap) return JSLP_OK;
    int cap = std::max(need, t->rowcap + t->rowcap / 2 + 8);
    CK(cudaStreamSynchronize(t->ctx->stream));
    int rc = alloc_rows(t, cap);
    if (rc) return rc;
    free_snap(t->snaps[0]);
    free_snap(t->snaps[1]);
    free_snap(t->snaps[2]);
    return JSLP_OK;  // descriptor is pushed by the caller; graphs read pointers through it
}

extern "C" int jslp_add_cuts(jslp_tab *t, const jslp_cut *cuts, int n) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    if (n < 0 || (n > 0 && !cuts)) return fail(JSLP_E_INVALID, "bad cuts");
    if (n == 0) {
        t->nVars = t->W + t->H - 2;  // cutting-strategies.ts:33-34
        return JSLP_OK;
    }
    CK(cudaSetDevice(t->ctx->device));
    cudaStream_t s = t->ctx->stream;
    const int grid_before = step_grid(t);
    int rc = grow_rows(t, t->H + n);
    if (rc) return rc;
    if (n > t->cuts_cap) {
        CK(cudaStreamSynchronize(s));
        cudaFree(t->d_cuts); cudaFreeHost(t->h_cuts);
        t->cuts_cap = std::max(64, n * 2);
        CK(cudaMalloc(&t->d_cuts, sizeof(CutDev) * (size_t)t->cuts_cap));
        CK(cudaMallocHost(&t->h_cuts, sizeof(CutDev) * (size_t)t->cuts_cap));
    } else {
        CK(cudaStreamSynchronize(s));  // h_cuts may still be in flight from the previous call
    }
    for (int i = 0; i < n; i++) {
        t->h_cuts[i].type = cuts[i].type;
        t->h_cuts[i].var_index = cuts[i].var_index;
        t->h_cuts[i].value = cuts[i].value;
    }
    CK(cudaMemcpyAsync(t->d_cuts, t->h_cuts, sizeof(CutDev) * (size_t)n, cudaMemcpyHostToDevice, s));
    const int H0 = t->H;
    t->H = H0 + n;
    rc = push_desc(t);  // kernels below read pointers/sizes through the descriptor
    if (rc) return rc;
    k_add_cuts<<<n, 256, 0, s>>>(t->d_T, t->d_cuts, H0, t->lastElementIndex);
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    t->lastElementIndex += n;
    t->nVars = t->W + t->H - 2 + n;  // cutting-strategies.ts:34,70 (the reference over-counts; kept)
    if (step_grid(t) != grid_before) drop_graphs(t);
    return JSLP_OK;
}

// addLowerBoundMIRCut / addUpperBoundMIRCut (row >= 0) and applyMIRCuts (row < 0), cutting-strategies.ts:74-212
static int mir_cuts(jslp_tab *t, int row, int upper, int *n_added) {
    CK(cudaSetDevice(t->ctx->device));
    cudaStream_t s = t->ctx->stream;
    const int max_cuts = 10;  // cutting-strategies.ts:203
    const int grid_before = step_grid(t);
    int rc = grow_rows(t, t->H + (row >= 0 ? 1 : max_cuts));
    if (rc) return rc;
    rc = push_desc(t);
    if (rc) return rc;
    k_mir_cuts<<<1, 256, 0, s>>>(t->d_T, t->H, t->lastElementIndex, row, upper, max_cuts, t->d_count);
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(t->h_count, t->d_count, sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    const int n = *t->h_count;
    t->H += n;
    t->nVars += n;             // cutting-strategies.ts:106 / 168
    t->lastElementIndex += n;  // getNewElementIndex (tableau.ts:393-401)
    if (n_added) *n_added = n;
    if (n > 0) {
        rc = push_desc(t);
        if (rc) return rc;
    }
    if (step_grid(t) != grid_before) drop_graphs(t);
    return JSLP_OK;
}

extern "C" int jslp_add_mir_cut(jslp_tab *t, int row, int upper_bound, int *added) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    if (row < 0 || row >= t->H) { if (added) *added = 0; return JSLP_OK; }
    return mir_cuts(t, row, upper_bound != 0, added);
}
extern "C" int jslp_apply_mir_cuts(jslp_tab *t, int *n_added) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    return mir_cuts(t, -1, 0, n_added);
}

// computeFractionalVolume (mip-utils.ts:67-98): a product over the basic integer variables in row order --
// an order-dependent fp64 product, so it is evaluated on the host over the downloaded right-hand-side column.
extern "C" int jslp_fractional_volume(jslp_tab *t, int ignore_integer_values, double *volume) {
    if (!t || !volume) return fail(JSLP_E_INVALID, "NULL argument");
    std::vector<double> rhs((size_t)t->H);
    std::vector<int> vrow((size_t)t->H);
    int rc = jslp_download(t, nullptr, rhs.data(), nullptr, vrow.data(), nullptr, nullptr, nullptr, nullptr);
    if (rc) return rc;
    double vol = -1;
    for (int r = 1; r < t->H; r++) {
        const int v = vrow[r];
        if (v < 0 || v >= (int)t->h_intpos.size() || t->h_intpos[v] < 0) continue;
        const double distance = std::fabs(rhs[r]);
        const double a = distance - std::floor(distance), b = std::floor(distance + 1);
        if ((a < b ? a : b) < t->precision) {
            if (!ignore_integer_values) { *volume = 0; return JSLP_OK; }
        } else if (vol == -1) {
            vol = distance;
        } else {
            vol *= distance;
        }
    }
    *volume = vol == -1 ? 0 : vol;
    return JSLP_OK;
}

// simplex() followed, under model.useMIRCuts, by the loop of branch-and-cut.ts:38-51.  Reports how many of the
// simplex() calls ended optimal and the evaluation of the first one (Tableau.simplexIters / bestPossibleEval).
static int simplex_with_mir(jslp_tab *t, int check_cycles, jslp_lp_status *out, bool timed, int *n_optimal, double *first_eval) {
    const int it0 = t->simplexIters;
    int rc = run_lp(t, 0, check_cycles, out, timed);
    if (rc) return rc;
    bool have_first = t->simplexIters != it0;
    double first = t->evaluation;
    int p1 = out ? out->phase1_pivots : 0, p2 = out ? out->phase2_pivots : 0;
    if (t->use_mir) {
        bool improved = true;
        while (improved) {
            double before = 0, after = 0;
            rc = jslp_fractional_volume(t, 1, &before);
            if (rc) return rc;
            rc = mir_cuts(t, -1, 0, nullptr);
            if (rc) return rc;
            const int it1 = t->simplexIters;
            rc = run_lp(t, 0, check_cycles, out, false);
            if (rc) return rc;
            if (!have_first && t->simplexIters != it1) { have_first = true; first = t->evaluation; }
            if (out) { p1 += out->phase1_pivots; p2 += out->phase2_pivots; }
            rc = jslp_fractional_volume(t, 1, &after);
            if (rc) return rc;
            if (after >= 0.9 * before) improved = false;
        }
        if (out) { out->phase1_pivots = p1; out->phase2_pivots = p2; }
    }
    if (n_optimal) *n_optimal = t->simplexIters - it0;
    if (first_eval) *first_eval = first;
    return JSLP_OK;
}

extern "C" int jslp_apply_cuts(jslp_tab *t, const jslp_cut *cuts, int n, int check_cycles, jslp_lp_status *out) {
    int rc = jslp_restore(t);
    if (rc) return rc;
    rc = jslp_add_cuts(t, cuts, n);
    if (rc) return rc;
    return simplex_with_mir(t, check_cycles, out, true, nullptr, nullptr);
}

static int mip_scan(jslp_tab *t, MipOut *o) {
    if (t->n_int <= 0) { o->is_integral = 1; o->var_index = -1; o->value = 0; return JSLP_OK; }
    CK(cudaSetDevice(t->ctx->device));
    cudaStream_t s = t->ctx->stream;
    k_mip_scan<<<1, 256, 0, s>>>(t->d_T, t->d_mip);
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(t->h_mip, t->d_mip, sizeof(MipOut), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    *o = *t->h_mip;
    return JSLP_OK;
}

extern "C" int jslp_is_integral(jslp_tab *t, int *is_integral) {
    if (!t || !is_integral) return fail(JSLP_E_INVALID, "NULL argument");
    MipOut o;
    int rc = mip_scan(t, &o);
    if (rc) return rc;
    *is_integral = o.is_integral;
    return JSLP_OK;
}
extern "C" int jslp_most_fractional(jslp_tab *t, int32_t *var_index, double *value) {
    if (!t || !var_index || !value) return fail(JSLP_E_INVALID, "NULL argument");
    MipOut o;
    int rc = mip_scan(t, &o);
    if (rc) return rc;
    *var_index = o.var_index;
    *value = o.value;
    return JSLP_OK;
}

extern "C" int jslp_download(jslp_tab *t, double *matrix, double *rhs_col, double *cost_row, int32_t *vrow,
                             int32_t *vcol, double *opt_obj, int32_t *width, int32_t *height) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    CK(cudaSetDevice(t->ctx->device));
    cudaStream_t s = t->ctx->stream;
    if (width) *width = t->W;
    if (height) *height = t->H;
    if (matrix)
        CK(cudaMemcpy2DAsync(matrix, sizeof(double) * t->W, t->hd.M, sizeof(double) * t->stride,
                             sizeof(double) * t->W, t->H, cudaMemcpyDeviceToHost, s));
    if (rhs_col)  // column 0 of every row: a strided D2H copy (8 bytes per row)
        CK(cudaMemcpy2DAsync(rhs_col, sizeof(double), t->hd.M, sizeof(double) * t->stride, sizeof(double), t->H,
                             cudaMemcpyDeviceToHost, s));
    if (cost_row) CK(cudaMemcpyAsync(cost_row, t->hd.M, sizeof(double) * t->W, cudaMemcpyDeviceToHost, s));
    if (vrow) CK(cudaMemcpyAsync(vrow, t->hd.vrow, sizeof(int) * t->H, cudaMemcpyDeviceToHost, s));
    if (vcol) CK(cudaMemcpyAsync(vcol, t->hd.vcol, sizeof(int) * t->W, cudaMemcpyDeviceToHost, s));
    if (opt_obj && t->nOpt > 0)
        CK(cudaMemcpy2DAsync(opt_obj, sizeof(double) * t->W, t->hd.opt, sizeof(double) * t->stride,
                             sizeof(double) * t->W, t->nOpt, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return JSLP_OK;
}

extern "C" int jslp_pivot_log(jslp_tab *t, int32_t *entries, int cap, int *n) {
    if (!t || !n) return fail(JSLP_E_INVALID, "NULL argument");
    const int m = (int)std::min<int64_t>((int64_t)t->host_log.size(), cap);
    for (int i = 0; i < m && entries; i++) {
        entries[4 * i + 0] = t->host_log[i].x & 0x3fffffff;
        entries[4 * i + 1] = t->host_log[i].y;
        entries[4 * i + 2] = t->host_log[i].z;
        entries[4 * i + 3] = t->host_log[i].w;
    }
    *n = (int)t->host_log.size();
    t->host_log.clear();
    return JSLP_OK;
}

#include "jslp_dynamic.cuh"
#include "jslp_comm.cuh"
#include "jslp_bnb_enhanced.cuh"
#include "jslp_batch.cuh"
#include "jslp_bnb.cuh"
#include "jslp_sensitivity.cuh"
#include "jslp_iis.cuh"
#include "jslp_parametric.cuh"
#include "jslp_scenario.cuh"
#include "jslp_recourse.cuh"
#include "jslp_crash.cuh"
#include "jslp_frontier.cuh"
#include "jslp_face.cuh"
#include "jslp_bound.cuh"
#include "jslp_lex.cuh"
#include "jslp_elastic.cuh"
#include "jslp_cone.cuh"
#include "jslp_pool.cuh"
#include "jslp_conflict.cuh"
#include "jslp_forest.cuh"
