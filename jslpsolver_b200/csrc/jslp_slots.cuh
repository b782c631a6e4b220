// jslpsolver_b200/csrc/jslp_slots.cuh -- K3: HBM-resident node batch (included by jslp_api.cu).
//
// Branch-and-cut nodes whose tableau does not fit shared memory (BASELINE config 5: 1537 x 1025 + cut rows,
// 12.6 MB) used to be solved strictly one after the other, each paying restore + cut rows + a host poll per
// batch of pivots, with ONE tableau in flight -- so every pivot cost the full selector chain although streaming
// its 25 MB takes a fraction of that.  Here B node LPs run side by side in B *slots*: each slot owns a ping-pong tableau
// pair, descriptor, pivot record and side buffers, and ONE launch of k_pivot_step with grid (G + 2, B) executes
// one pivot of every running slot -- while slot A's selectors walk their chain, slot B's rows stream.  A node is
// applyCuts (branch-and-cut.ts:33-52): restore the root snapshot (backup.ts:53-105), append its cut rows
// (cutting-strategies.ts:36-71), simplex(); then isIntegral / getMostFractionalVar (mip-utils.ts:43-61,100-126).
//
// One CUDA graph = k_slot_begin (restore + cut rows + record init for slots that were handed a new node, all on
// the device) -> k_select (first pivot of those) -> S x k_pivot_step -> k_slot_end (integrality scan + result
// record into mapped host memory).  The host polls once per graph for ALL slots, runs the cycle detector over
// the new log entries, retires finished nodes and hands free slots their next node: no per-node host work
// beyond writing its cut list.  Results are a pure function of (root snapshot, cut list) (SURVEY.md 3.8), so
// the frontier manager commits them in the reference's order exactly as before.
#pragma once

namespace jslp {

enum { SLOT_IDLE = 0, SLOT_CONTINUE = 1, SLOT_LOAD = 2 };

struct SlotCtl {  // host -> device, one per slot, mapped pinned memory
    int cmd, n_cuts, cut_off, pad;
};
struct SlotOut {  // device -> host, one per slot, mapped pinned memory
    Rec rec;
    MipOut mip;
    int scanned, pad[3];
};
struct SlotBatchDev {
    TabDev *T;            // [B] descriptors
    Rec *rec;             // [B] pivot records
    const SlotCtl *ctl;   // [B]
    const CutDev *cuts;   // cut lists of the nodes being loaded
    SlotOut *out;         // [B]
    const double *rootM;  // root snapshot (Saved), row stride = the tableau's stride
    const int *root_vrow, *root_vcol;
    int H0, first_index, part_n, lookahead;
};

// Start of a graph.  LOAD: slot := root snapshot + the node's cut rows, fresh record (what jslp_restore,
// jslp_add_cuts and the head of run_lp do for a single tableau).  CONTINUE: new log window.  IDLE: parked.
__global__ void __launch_bounds__(256) k_slot_begin(const __grid_constant__ SlotBatchDev sb) {
    __shared__ int s_row, s_col;
    const int slot = blockIdx.y, tid = threadIdx.x, NT = blockDim.x;
    const SlotCtl ctl = sb.ctl[slot];
    Rec *rec = sb.rec + slot;
    if (ctl.cmd == SLOT_IDLE) {
        if (blockIdx.x == 0 && tid == 0) { rec->status = ST_P1_DONE; rec->has_pivot = 0; rec->log_n = 0; }
        return;
    }
    if (ctl.cmd == SLOT_CONTINUE) {
        if (blockIdx.x == 0 && tid == 0) rec->log_n = 0;
        return;
    }
    TabDev *Tp = sb.T + slot;
    const TabDev T = *Tp;
    const int H0 = sb.H0, stride = T.stride;
    {   // restore (backup.ts:53-105): matrix, varIndexByRow, varIndexByCol
        const size_t n2 = ((size_t)H0 * stride) >> 1;
        const double2 *src = reinterpret_cast<const double2 *>(sb.rootM);
        double2 *dst = reinterpret_cast<double2 *>(T.M);
        for (size_t i = (size_t)blockIdx.x * NT + tid; i < n2; i += (size_t)gridDim.x * NT) dst[i] = src[i];
        for (int i = blockIdx.x * NT + tid; i < H0; i += gridDim.x * NT) T.vrow[i] = sb.root_vrow[i];
        for (int i = blockIdx.x * NT + tid; i < T.W; i += gridDim.x * NT) T.vcol[i] = sb.root_vcol[i];
        // no message of the slot's previous node may carry a sequence tag of this solve (tags restart at 1)
        unsigned long long *pp = reinterpret_cast<unsigned long long *>(T.part);
        const int nw = sb.part_n * (int)(sizeof(Part) / sizeof(unsigned long long));
        for (int i = blockIdx.x * NT + tid; i < nw; i += gridDim.x * NT) pp[i] = ~0ull;
    }
    // addCutConstraints (cutting-strategies.ts:36-71): cut rows in the ROOT basis, read from the snapshot
    for (int h = blockIdx.x; h < ctl.n_cuts; h += gridDim.x) {
        const CutDev cut = sb.cuts[ctl.cut_off + h];
        __syncthreads();
        if (tid == 0) { s_row = -1; s_col = -1; }
        __syncthreads();
        int row, col;
        cut_lookup(sb.root_vrow, H0, sb.root_vcol, T.W, cut.var_index, tid, NT, row, col);
        if (row >= 0) s_row = row;
        if (col >= 0) s_col = col;
        __syncthreads();
        const double *vr = s_row < 0 ? nullptr : sb.rootM + (size_t)s_row * stride;
        double *cutrow = T.M + (size_t)(H0 + h) * stride;
        for (int c = tid; c < stride; c += NT) cutrow[c] = cut_entry(cut, c, s_col, c < T.W ? vr : nullptr);
        if (tid == 0) T.vrow[H0 + h] = sb.first_index + h;
    }
    if (blockIdx.x == 0 && tid == 0) {
        Tp->H = H0 + ctl.n_cuts;
        Rec r;
        memset(&r, 0, sizeof(r));
        r.status = ST_RUNNING; r.phase = 1; r.stop_at = -1; r.unbounded_var = -1; r.only_phase = 0;
        r.lookahead = sb.lookahead; r.next_c = -1;
        *rec = r;
    }
}

// End of a graph: integrality scan of slots whose LP ended optimal, record copy for the host.
__global__ void __launch_bounds__(256) k_slot_end(const __grid_constant__ SlotBatchDev sb) {
    __shared__ RedSmem red;
    __shared__ TabDev T;
    __shared__ MipOut mo;
    const int slot = blockIdx.x, tid = threadIdx.x;
    if (sb.ctl[slot].cmd == SLOT_IDLE) return;
    const Rec *rec = sb.rec + slot;
    if (tid == 0) { T = sb.T[slot]; mo.is_integral = 0; mo.var_index = -1; mo.value = 0.0; }
    __syncthreads();
    const int status = rec->status;
    const bool scan = (status == ST_OPTIMAL || status == ST_UNBOUNDED) && T.intpos != nullptr;
    if (scan) cta_mip_scan(T, &mo, red);
    __syncthreads();
    SlotOut *o = sb.out + slot;
    if (tid < (int)(sizeof(Rec) / 16)) reinterpret_cast<int4 *>(&o->rec)[tid] = reinterpret_cast<const int4 *>(rec)[tid];
    if (tid == 32) { o->mip = mo; o->scanned = scan ? 1 : 0; }
}

}  // namespace jslp

// ---- host side ----------------------------------------------------------------------------------
struct NodeSlots {
    using TabDev = jslp::TabDev; using Rec = jslp::Rec; using Part = jslp::Part; using SlotCtl = jslp::SlotCtl;
    using SlotOut = jslp::SlotOut; using CutDev = jslp::CutDev;
    int B = 0, rowcap = 0, G = 0, steps = 0, key = -1;
    TabDev *d_T = nullptr;
    Rec *d_rec = nullptr;
    double *M = nullptr, *M2 = nullptr, *prow = nullptr, *pcol = nullptr;
    int *vrow = nullptr, *vcol = nullptr;
    Part *part = nullptr;
    int4 *plog = nullptr, *h_logs = nullptr;
    int plog_cap = 0;
    SlotCtl *h_ctl = nullptr, *dv_ctl = nullptr;
    SlotOut *h_out = nullptr, *dv_out = nullptr;
    CutDev *h_cuts = nullptr, *dv_cuts = nullptr;
    int cuts_cap = 0;
    cudaGraphExec_t graph = nullptr;
    void release() {
        if (graph) cudaGraphExecDestroy(graph);
        graph = nullptr;
        cudaFree(d_T); cudaFree(d_rec); cudaFree(M); cudaFree(M2); cudaFree(prow); cudaFree(pcol);
        cudaFree(vrow); cudaFree(vcol); cudaFree(part); cudaFree(plog);
        cudaFreeHost(h_logs); cudaFreeHost(h_ctl); cudaFreeHost(h_out); cudaFreeHost(h_cuts);
        *this = NodeSlots();
    }
};
