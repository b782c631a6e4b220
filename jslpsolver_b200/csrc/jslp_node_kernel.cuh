// jslpsolver_b200/csrc/jslp_node_kernel.cuh -- shared-memory-resident node LPs.
//
// One CTA solves one branch-and-cut node (or one small LP) start to finish with the whole tableau
// in shared memory: restore from the root snapshot (backup.ts:53-105), append the node's cut rows
// (cutting-strategies.ts:36-71), run phase 1 / phase 2 to completion (simplex.ts:14-325) and
// report the summary the frontier needs (evaluation, isIntegral, most fractional variable;
// mip-utils.ts:43-61,100-126).  A launch evaluates a whole batch of open nodes, one CTA each:
// this is what makes the node frontier GPU-resident.  Selection is done by ONE warp with shuffle
// reductions (no CTA barrier): the same rules as cta_select, restated at warp scope; the parity tests
// run every fixture through both paths.
#pragma once
#include "jslp_kernels.cuh"

namespace jslp {

struct NodeResult {
    int status;       // ST_* at exit
    int p1, p2;       // pivots per phase
    int log_n;        // pivot-log entries written (selections)
    int overflow;     // pivot cap reached or log overflow: host re-evaluates on the HBM path
    int is_integral;
    int branch_var;   // -1 = none
    int unbounded_var;
    double eval_raw;
    double branch_value;
    long long t_ns;   // CTA lifetime by %globaltimer (reporting only)
    long long pad;
    long long cy[6];  // warp-0 cycles: select, barrier A, division passes, row update, look-ahead pricing, barrier B
    long long tl[6];  // ns since CTA start: offsets read, restored, cut rows built, pivots done, mip scan done, (unused)
};

// What a CTA reports: the summary plus the head of its pivot log (enough for the cycle check of
// almost every node), written straight into mapped pinned host memory -- no D2H copy per round.
constexpr int NODE_LOG_HEAD = 64;
struct NodeOut {
    NodeResult r;
    int4 log_head[NODE_LOG_HEAD];
};

constexpr int NODE_INLINE_OFF = 64;

// Launch modes of k_node_batch (a template parameter: each mode's instantiation carries only its own prologue)
enum NodeMode : int {
    NODE_BRANCH = 0,    // branch-and-cut nodes and engine 4: every root row, then the node's cuts
    NODE_SCENARIO = 2,  // one list of right-hand-side / cost edits of the root per CTA (jslp_scenario_batch)
    NODE_COLUMNS = 3,   // one column subset of the root per CTA, the others zeroed (jslp_column_batch)
    NODE_POOL = 4,      // one region of a solution-pool search per CTA: fixed columns, then cut rows (jslp_pool_batch)
    NODE_CONFLICT = 5,  // one row subset of the root per CTA, then cut rows, phase 1 only, and the integrality scan
                        // over an integer mask (jslp_conflict_batch; jslp_feasibility_batch without cuts or mask)
    NODE_FOREST = 6,    // the roots and nodes of many branch-and-cut trees at once (jslp_bnb_batch): each CTA's own
                        // column 0 and row 0 over the root, or each node restored from its tree's root slot
};

// One resolved scenario edit (DESIGN.md 2e): where updateRightHandSide / updateCost (dynamic-modification.ts:78-160)
// write on the root tableau, and the difference.
enum EditKind : int {
    EDIT_RHS_COL = 0,   // slack non-basic in column pos: M[r,0] -= d * M[r,pos] for every row, row 0 included
    EDIT_RHS_ROW = 1,   // slack basic in row pos: M[pos,0] -= d
    EDIT_COST_ROW = 2,  // variable basic in row pos: M[0,c] += d * M[pos,c] for every column, column 0 included
    EDIT_COST_COL = 3,  // variable non-basic in column pos: M[0,pos] -= d
    EDIT_FIX_COL = 4,   // variable non-basic in column pos held at d (DESIGN.md 2m): M[r,0] -= d * M[r,pos], then
                        // M[r,pos] = +0, for every row, row 0 included
};
struct EditDev {
    int kind, pos;
    double d;
};

struct NodeBatchDev {
    const double *rootM;   // root snapshot, row stride = root_stride
    const int *root_vrow, *root_vcol;
    const CutDev *cuts;    // all cuts of the batch, node n owns [cut_off[n], cut_off[n+1]); may be mapped host memory
    const int *cut_off;    // (NODE_SCENARIO: the same offsets into edits)
    NodeOut *out;          // one record per node; may be mapped host memory
    int4 *logs;            // log_cap entries per node (device memory)
    double *wb_M;          // optional write-back of node 0's final tableau (stride = root_stride)
    int *wb_vrow, *wb_vcol;
    int H0, root_stride, first_index, Hcap, Ws, log_cap, max_pivots;
    // row-subset launches (NODE_CONFLICT): node n keeps the root rows whose bits are set in keep[n * keep_words ...]
    // (device memory; row 0 is always kept).  Column-subset launches (NODE_COLUMNS, jslp_column_batch) read the same
    // bits as columns: node n writes +0 over every column whose bit is clear, in every row.  Not read by the other
    // modes.
    const uint32_t *keep;
    int keep_words;
    // scenario launches (NODE_SCENARIO, jslp_scenario_batch): node n applies edits[cut_off[n] .. cut_off[n+1]) (device
    // memory; every right-hand-side edit before every cost edit) to the restored root, solves, and writes its final
    // column 0 and row labels to out_rhs / out_vrow + n * Hcap (NODE_COLUMNS writes them too).  Not read by the other
    // modes.
    // Pool launches (NODE_POOL: jslp_pool_batch, jslp_target_batch, jslp_box_batch) apply edits[edit_off[n] ..
    // edit_off[n+1]) (device memory) to the restored root: the EDIT_RHS_COL / EDIT_RHS_ROW / EDIT_FIX_COL edits in list
    // order as one row pass, then, when cost_edits is set, the
    // EDIT_COST_ROW / EDIT_COST_COL edits in list order as NODE_SCENARIO applies them; then they append node n's cut
    // rows as NODE_BRANCH does.  They write column 0 and the row labels too.  The final columns go to out_rhs /
    // out_vrow + n * Hcap.
    const EditDev *edits;
    const int *edit_off;
    double *out_rhs;
    int *out_vrow;
    // scenario launches with cert_u set (jslp_recourse_batch): node n writes the multipliers of its certificate row
    // (row 0 at an optimum, the row phase 1 stopped at when infeasible) to cert_u + n * cert_n, entry cert_pos[l] for
    // every label l < cert_labels with cert_pos[l] >= 0: the row's entry when l is non-basic, its unit entry when l is
    // basic; +0 throughout when there is no certificate (device memory).  Not read by the other modes.
    double *cert_u;
    const int *cert_pos;
    int cert_n, cert_labels;
    int cost_edits;
    int n_inline;         // > 0: cut_off_inline holds the n_inline + 1 offsets (saves a PCIe round trip)
    int cut_off_inline[NODE_INLINE_OFF + 1];
    // Row-subset launches (NODE_CONFLICT: jslp_conflict_batch, and jslp_feasibility_batch without cuts, mask or
    // outputs) append the node's cut rows after its kept rows and stop with ST_P1_DONE where phase 1 finds no leaving
    // row; Hcap counts the kept rows plus the cuts of the largest node.  With int_keep set, the integrality scan reads
    // only the integer positions p whose bit is set in int_keep[n * int_words ...] (device memory); with it null there
    // is no scan.  With out_rhs set, column 0 and the row labels go to out_rhs / out_vrow + n * Hcap.  Not read by the
    // other modes.
    const uint32_t *int_keep;
    int int_words;
    // Forest launches (NODE_FOREST, jslp_bnb_batch).  Tree s owns root slot s: slot_M + s * slot_pitch (H0 rows at
    // root_stride), slot_vrow + s * H0 and slot_vcol + s * W.  A root launch (col0 set) restores rootM, writes
    // col0 + s * H0 over rows 1.. of column 0 and row0 + s * W over row 0 for s = root_of[n], solves, and writes its
    // whole final tableau and labels to slot s.  A node launch (col0 null) restores slot root_of[n] and appends node n's cut rows
    // as NODE_BRANCH does.  Either writes column 0 and the row labels to out_rhs / out_vrow + n * Hcap when out_rhs is
    // set.  Not read by the other modes.
    double *slot_M;
    int *slot_vrow, *slot_vcol;
    size_t slot_pitch;
    const int *root_of;
    const double *col0, *row0;
};

constexpr int NODE_THREADS = 256;

__device__ __forceinline__ long long globaltimer_ns() {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// ---- warp-level selection ----------------------------------------------------------------------
// In the resident kernel one warp decides every pivot.  A lone warp issues a dependent instruction
// every ~8 cycles, so the reductions avoid shuffle trees: values are mapped to order-preserving
// integer keys and reduced with redux.sync (three to four REDUX per arg-min instead of five shuffle
// levels of fp64 compares), and the scans issue their loads and divisions four at a time.
// Phase-2 pricing of the cost row (simplex.ts:140-219 without optional objectives): first batch with
// an improving column, arg-max inside it, lowest column on ties.  Returns the column (0 = none).
// One copy each of the bulky helpers: the pivot loop has to stay inside the instruction cache (an
// earlier fully-inlined build had a 64 KB loop body and spent most of its time fetching instructions).
__device__ __noinline__ int warp_price(const TabDev &T, const double *cost, const int *vcol, int W, int lane, int *neg_out) {
    const int bsz = T.use_partial ? T.batch_size : max(1, W - 1);
    const bool has_unres = T.unres != nullptr;
    PriceAcc acc;
    price_init(acc, T.prec);
#pragma unroll 1
    for (int c = 1 + lane; c < W; c += 32) {
        const double nc = cost[c];
        int label = -1;
        if (has_unres && nc < 0) label = vcol[c];
        price_consider(T, acc, c, nc, label, bsz);
    }
    // lexicographic (batch asc, value desc, column asc)
    const int mb = __reduce_min_sync(0xffffffffu, acc.myb);
    if (mb == INT_MAX) { *neg_out = 0; return 0; }
    const bool in = acc.myb == mb;
    const unsigned long long k = dkey(acc.x.v);
    const unsigned int hi = (unsigned int)(k >> 32), lo = (unsigned int)k;
    const unsigned int mhi = __reduce_max_sync(0xffffffffu, in ? hi : 0u);
    const unsigned int mlo = __reduce_max_sync(0xffffffffu, (in && hi == mhi) ? lo : 0u);
    const bool win = in && hi == mhi && lo == mlo;
    const int col = __reduce_min_sync(0xffffffffu, win ? acc.x.i : INT_MAX);
    *neg_out = __reduce_max_sync(0xffffffffu, (win && acc.x.i == col) ? acc.myneg : 0);
    return col;
}

struct NodePivot {   // warp 0 -> CTA
    int go, r, c, flush;
    double q;
};
struct NodeScan {    // warp 0 -> CTA: which division scan to run (1 = phase-1 column scan of row r, 2 = ratio test of column c)
    int mode, r, c, neg;
};
struct NodePart {    // per-warp partial results of a scan
    double v[8];
    int i[8], d[8], n[8];
};

// MODE = NODE_BRANCH: branch-and-cut nodes and engine 4 (every root row, then the node's cuts).  NODE_SCENARIO: every
// root row, then the CTA's edit list applied to column 0 and row 0 (DESIGN.md 2e) in place of cut rows.  NODE_COLUMNS:
// every root row, with the columns cleared in the CTA's mask set to +0 in every row, row 0 included (DESIGN.md 2l).
// NODE_POOL: every root row, the CTA's fixings applied by the scenario edit loop, then its cut rows (DESIGN.md 2m).
// NODE_CONFLICT: one row subset of the root per CTA (NodeBatchDev.keep), compacted in row order, then the CTA's cut
// rows, phase 1 only, and the integrality scan over the CTA's integer mask if it has one (DESIGN.md 2c, 2n); row
// labels stay the root's, so the unrestricted lookup and the pivot log read as on the whole tableau.  A template
// parameter, so that the node path carries none of the scenario, column, pool or row-subset code.
template <int MODE>
__global__ void __launch_bounds__(NODE_THREADS) k_node_batch(const TabDev *Tp, const __grid_constant__ NodeBatchDev nb) {
    constexpr bool SCENARIO = MODE == NODE_SCENARIO, COLUMNS = MODE == NODE_COLUMNS;
    constexpr bool POOL = MODE == NODE_POOL, CONFLICT = MODE == NODE_CONFLICT, FOREST = MODE == NODE_FOREST;
    extern __shared__ __align__(16) unsigned char smraw[];
    __shared__ TabDev T;
    __shared__ SelSmem sel;
    __shared__ MipOut mip;
    __shared__ NodePivot piv;
    __shared__ NodeScan sc;
    __shared__ NodePart part;
    __shared__ int s_spare, s_kept;
    __shared__ int s_fin[8];   // status, p1, p2, log_n, overflow, unbounded_var
    __shared__ double s_eval;
    __shared__ __align__(8) uint64_t s_bar;
    const int tid = threadIdx.x, NT = blockDim.x;
    const int warp = tid >> 5, lane = tid & 31, NW = NT >> 5;
    const int node = blockIdx.x;
    long long t_start = 0;
    if (tid == 0) t_start = globaltimer_ns();
    const int H0 = nb.H0, Ws = nb.Ws;
    // a forest node restores its tree's root slot; every other launch, and a forest root, the launch's root
    const bool from_slot = FOREST && nb.col0 == nullptr;
    const size_t tree = from_slot ? (size_t)nb.root_of[node] : 0;

    // rows live in Hcap + 1 slots: the normalised pivot row is written to the spare slot and the slot
    // table is swapped, so nobody waits for the old pivot row to be overwritten in place.  Ws is even:
    // rows are 16-byte aligned, which is what lets TMA restore them.
    double *Ms = reinterpret_cast<double *>(smraw);
    double *frow = Ms + (size_t)(nb.Hcap + 1) * Ws;
    double *rhs = frow + Ws;                         // Hcap entries: pivot-column staging, final RHS column
    CutDev *cutS = reinterpret_cast<CutDev *>(rhs + nb.Hcap + (nb.Hcap & 1));
    int *vrow = reinterpret_cast<int *>(cutS + (CONFLICT ? nb.Hcap : nb.Hcap - H0));
    int *slot = vrow + nb.Hcap;
    if (tid == 0) {
        T = *Tp;
        T.vcol = slot + nb.Hcap;
        s_spare = nb.Hcap;
        mbar_init(&s_bar, 1);
        fence_mbar_init();
    }
    __syncthreads();
    int H0k = H0;  // rows restored from the root
    if constexpr (CONFLICT) {
        // compacted position of every kept row: slot[d] = the root row that becomes row d (slot is reset below,
        // once the copies that read it have been issued)
        if (warp == 0) {
            const uint32_t *kw = nb.keep + (size_t)node * nb.keep_words;
            int base = 0;
            for (int r0 = 0; r0 < H0; r0 += 32) {
                const int r = r0 + lane;
                const bool kept = r < H0 && (r == 0 || ((kw[r >> 5] >> (r & 31)) & 1u));
                const unsigned int b = __ballot_sync(0xffffffffu, kept);
                if (kept) slot[base + __popc(b & ((1u << lane) - 1u))] = r;
                base += __popc(b);
            }
            if (lane == 0) s_kept = base;
        }
        __syncthreads();
        H0k = s_kept;
    }
    // restore(): root snapshot -> shared memory, one TMA bulk copy per row (backup.ts:53-105)
    if (tid == 0) mbar_expect_tx(&s_bar, (uint32_t)(H0k * Ws * sizeof(double)));
    __syncthreads();
    for (int r = tid; r < H0k; r += NT) {
        const int src = CONFLICT ? slot[r] : r;
        const double *rootM = from_slot ? nb.slot_M + tree * nb.slot_pitch : nb.rootM;
        tma_bulk_g2s(Ms + (size_t)r * Ws, rootM + (size_t)src * nb.root_stride, (uint32_t)(Ws * sizeof(double)), &s_bar);
    }
    // the cut list may live in mapped host memory: one PCIe round trip, overlapped with the restore
    int c0, nc;
    if (nb.n_inline > 0) { c0 = nb.cut_off_inline[node]; nc = nb.cut_off_inline[node + 1] - c0; }
    else { c0 = nb.cut_off[node]; nc = nb.cut_off[node + 1] - c0; }
    long long tl0 = 0, tl1 = 0, tl2 = 0, tl3 = 0, tl4 = 0;
    const int W = T.W;
    const double prec = T.prec;
    int *vcol = T.vcol;
    for (int h = tid; !SCENARIO && !COLUMNS && h < nc; h += NT) cutS[h] = nb.cuts[c0 + h];
    for (int r = tid; r < H0k; r += NT)
        vrow[r] = __ldg((from_slot ? nb.slot_vrow + tree * H0 : nb.root_vrow) + (CONFLICT ? slot[r] : r));
    for (int c = tid; c < W; c += NT) vcol[c] = __ldg((from_slot ? nb.slot_vcol + tree * W : nb.root_vcol) + c);
    if (!CONFLICT)
        for (int r = tid; r < nb.Hcap; r += NT) slot[r] = r;
    const int Hn = (SCENARIO || COLUMNS) ? H0k : H0k + nc;
    if (tid == 0) tl0 = globaltimer_ns() - t_start;
    mbar_wait(&s_bar, 0);
    __syncthreads();
    if (CONFLICT)  // nobody reads slot until the barrier after the cut rows
        for (int r = tid; r < nb.Hcap; r += NT) slot[r] = r;
    if (tid == 0) tl1 = globaltimer_ns() - t_start;
    if constexpr (FOREST) {
        // a forest root: the tree's right-hand sides and costs are written over the base's (DESIGN.md 2p); rows 1.. of
        // column 0 and row 0 are disjoint, and the next reader waits at the barrier after the (absent) cut rows
        if (nb.col0 != nullptr) {
            const size_t s = (size_t)nb.root_of[node];
            const double *c0 = nb.col0 + s * H0, *r0 = nb.row0 + s * W;
            for (int r = 1 + tid; r < H0; r += NT) Ms[(size_t)r * Ws] = c0[r];
            for (int c = tid; c < W; c += NT) Ms[c] = r0[c];
        }
    }
    if constexpr (SCENARIO || POOL) {
        // setRightHandSide / setCost on the restored root (DESIGN.md 2e): every edit writes column 0 or row 0 only and
        // reads columns >= 1 / rows >= 1, so the right-hand-side edits run as one pass over rows (each thread applies
        // all of them to its M[r,0] in order) and the cost edits, after them, as one pass over columns.  A fixing
        // (DESIGN.md 2m) reads and then clears its own column of the thread's row, so it joins the row pass.  A pool
        // launch without cost edits (jslp_pool_batch) skips the column pass.
        int e0 = c0, ne = nc;
        if constexpr (POOL) { e0 = nb.edit_off[node]; ne = nb.edit_off[node + 1] - e0; }
        const EditDev *ed = nb.edits + e0;
        for (int r = tid; r < H0k; r += NT) {
            double *row = Ms + (size_t)r * Ws;
            double x = row[0];
            for (int k = 0; k < ne; k++) {
                const EditDev e = ed[k];
                if (e.kind == EDIT_RHS_COL) x = edit_axpy_sub(x, e.d, row[e.pos]);
                else if (e.kind == EDIT_RHS_ROW && e.pos == r) x = edit_sub(x, e.d);
                else if (POOL && e.kind == EDIT_FIX_COL) { x = edit_axpy_sub(x, e.d, row[e.pos]); row[e.pos] = 0.0; }
            }
            row[0] = x;
        }
        __syncthreads();
        if (SCENARIO || nb.cost_edits)
            for (int c = tid; c < W; c += NT) {
                double x = Ms[c];
                for (int k = 0; k < ne; k++) {
                    const EditDev e = ed[k];
                    if (e.kind == EDIT_COST_ROW) x = edit_axpy_add(x, e.d, Ms[(size_t)e.pos * Ws + c]);
                    else if (e.kind == EDIT_COST_COL && e.pos == c) x = edit_sub(x, e.d);
                }
                Ms[c] = x;
            }
    }
    if constexpr (COLUMNS) {
        // the cleared columns of this CTA's mask are +0 in every row: a zero column prices at 0, so it never
        // enters, and a pivot leaves it zero
        const uint32_t *kw = nb.keep + (size_t)node * nb.keep_words;
        for (int r = warp; r < Hn; r += NW) {
            double *row = Ms + (size_t)r * Ws;
            for (int c = 1 + lane; c < W; c += 32)
                if (!((kw[c >> 5] >> (c & 31)) & 1u)) row[c] = 0.0;
        }
    }
    // addCutConstraints(): every cut row is expressed in the ROOT basis, so the rows are independent:
    // one warp per cut, no CTA barrier inside (a scenario's nc counts edits; a column launch has none)
    for (int h = warp; !SCENARIO && !COLUMNS && h < nc; h += NW) {
        const CutDev cut = cutS[h];
        int s_row, s_col;
        cut_lookup(vrow, H0k, vcol, W, cut.var_index, lane, 32, s_row, s_col);
        s_row = __reduce_max_sync(0xffffffffu, s_row);
        s_col = __reduce_max_sync(0xffffffffu, s_col);
        const double *vr = s_row < 0 ? nullptr : Ms + (size_t)s_row * Ws;
        double *cutrow = Ms + (size_t)(H0k + h) * Ws;
        if (vr != nullptr)  // one loop per case: neither tests the case per entry
            for (int c = lane; c < W; c += 32) cutrow[c] = cut_entry(cut, c, s_col, vr);
        else
            for (int c = lane; c < W; c += 32) cutrow[c] = cut_entry(cut, c, s_col, nullptr);
        if (lane == 0) vrow[H0k + h] = nb.first_index + h;
    }
    __syncthreads();
    if (tid == 0) tl2 = globaltimer_ns() - t_start;

    // warp 0's registers: the solve state
    int phase = 1, p1 = 0, p2 = 0, log_n = 0, status = ST_RUNNING, overflow = 0, unb = -1;
    int next_c = -1, next_neg = 0;      // look-ahead pricing of the updated cost row (-1 = not priced)
    int rstar = -1, cstar = -1, isneg = 0;
    int4 *plog = nb.logs + (size_t)node * nb.log_cap;
    const bool has_unres = T.unres != nullptr;
    long long cy[6] = {0, 0, 0, 0, 0, 0}, cprev = clock64();
// per-phase cycle counters of warp 0 (S1, S2, S3, D, U, barrier): compile with -DJSLP_NODE_CYCLES to fill them
#ifdef JSLP_NODE_CYCLES
#define NODE_CY(k) do { const long long cnow = clock64(); cy[k] += cnow - cprev; cprev = cnow; } while (0)
#else
#define NODE_CY(k) do { (void)cprev; } while (0)
#endif
    double *pcol = rhs;  // old pivot-column entries of the pivot in flight (the RHS copy is only made at the end)

    // One pivot = five CTA barriers.  fp64 division has a latency of several hundred cycles and does not
    // interleave (each one carries a slow-path branch), so every pass that divides is spread over the
    // whole CTA, one element per thread: (S2) the phase-1 column scan / the ratio test, (D) pivot-row
    // normalisation + pivot-column rewrite.  The cheap decisions (S1, S3) stay in warp 0's registers.
    for (;;) {
        // ---- S1 (warp 0): leaving row (phase 1: simplex.ts:38-54) or entering column (phase 2: 129-269)
        if (warp == 0) {
            const double *cost = Ms + (size_t)slot[0] * Ws;
            int go = 1;
            rstar = -1; cstar = -1; isneg = 0;
            if (p1 + p2 >= nb.max_pivots || log_n >= nb.log_cap) { overflow = 1; go = 0; }
            if (go && phase == 1) {
                VI b = {-prec, INT_MAX};
#pragma unroll 2
                for (int r = 1 + lane; r < Hn; r += 32) {
                    const double v = Ms[(size_t)slot[r] * Ws];
                    if (v < b.v) { b.v = v; b.i = r; }
                }
                b = warp_reduce_vi<true>(b);
                if (b.i == INT_MAX) {  // feasible (simplex.ts:51-54)
                    if (CONFLICT) { status = ST_P1_DONE; go = 0; }
                    else phase = 2;
                } else {
                    rstar = b.i;
                }
            }
            if (go && rstar < 0) {  // phase 2
                if (next_c < 0) next_c = warp_price(T, cost, vcol, W, lane, &next_neg);
                if (next_c == 0) { status = ST_OPTIMAL; go = 0; }  // simplex.ts:265-269
                else { cstar = next_c; isneg = next_neg; }
            }
            if (lane == 0) {
                sc.mode = !go ? 0 : (rstar >= 0 ? 1 : 2);
                sc.r = rstar; sc.c = cstar; sc.neg = isneg;
                if (!go) {
                    s_fin[0] = status; s_fin[1] = p1; s_fin[2] = p2; s_fin[3] = log_n; s_fin[4] = overflow; s_fin[5] = unb;
                    s_eval = cost[0];
                }
            }
        }
        NODE_CY(0);
        __syncthreads();
        const int mode = sc.mode;
        if (mode == 0) break;
        // ---- S2 (CTA): the scan that divides, one element per thread --------------------------------
        if (mode == 1) {  // entering column of a phase-1 pivot (simplex.ts:56-76)
            const double *cost = Ms + (size_t)slot[0] * Ws;
            const double *lrow = Ms + (size_t)slot[sc.r] * Ws;
            VI e = {-INFINITY, INT_MAX};
#pragma unroll 1
            for (int c = 1 + tid; c < W; c += NT)
                entering_step<ddiv_z>(c, lrow[c], has_unres && is_unres(T, vcol[c]), prec, e, [&] { return cost[c]; });
            e = warp_reduce_vi<false>(e);
            if (lane == 0) { part.v[warp] = e.v; part.i[warp] = e.i; }
        } else {          // ratio test (simplex.ts:271-296)
            const int cs = sc.c, neg = sc.neg;
            VI m = {INFINITY, INT_MAX};
            int dmin = INT_MAX, cnt = 0;
#pragma unroll 1
            for (int r = tid; r < Hn; r += NT) {
                const double *row = Ms + (size_t)slot[r] * Ws;
                ratio_step<ddiv_z>(r, row[cs], row[0], neg, prec, dmin, m, cnt);
            }
            dmin = __reduce_min_sync(0xffffffffu, dmin);
            cnt = __reduce_add_sync(0xffffffffu, cnt);
            m = warp_reduce_vi<true>(m);
            if (lane == 0) { part.v[warp] = m.v; part.i[warp] = m.i; part.d[warp] = dmin; part.n[warp] = cnt; }
        }
        NODE_CY(1);
        __syncthreads();
        // ---- S3 (warp 0): combine the partials, stage the pivot ------------------------------------
        if (warp == 0) {
            int go = 1, cnt = 0;
            if (mode == 1) {
                VI e = {-INFINITY, INT_MAX};
                if (lane < NW) { e.v = part.v[lane]; e.i = part.i[lane]; }
                e = warp_reduce_vi<false>(e);
                if (e.i == INT_MAX) { status = ST_INFEASIBLE; go = 0; }  // simplex.ts:73-76
                else {
                    cstar = e.i;
#pragma unroll 1
                    for (int r = lane; r < Hn; r += 32)  // non-zero pivot-column entries (lazy-flush flag)
                        if (nz16(Ms[(size_t)slot[r] * Ws + cstar])) cnt++;
                    cnt = __reduce_add_sync(0xffffffffu, cnt);
                }
            } else {
                VI m = {INFINITY, INT_MAX};
                int dmin = INT_MAX;
                if (lane < NW) { m.v = part.v[lane]; m.i = part.i[lane]; dmin = part.d[lane]; cnt = part.n[lane]; }
                dmin = __reduce_min_sync(0xffffffffu, dmin);
                cnt = __reduce_add_sync(0xffffffffu, cnt);
                if (dmin != INT_MAX) rstar = dmin;
                else {
                    m = warp_reduce_vi<true>(m);
                    if (m.i != INT_MAX) rstar = m.i;
                    else { status = ST_UNBOUNDED; unb = vcol[cstar]; go = 0; }  // simplex.ts:298-303
                }
            }
            if (go) {
                const double q = Ms[(size_t)slot[rstar] * Ws + cstar];
                if (lane == 0) {  // log_n < log_cap: checked in S1
                    log_pivot(plog, log_n, nb.log_cap, vrow, vcol, phase, rstar, cstar, vrow[rstar], vcol[cstar]);
                    piv.go = 1; piv.r = rstar; piv.c = cstar; piv.q = q;
                    piv.flush = flush_flag(cnt, q);
                }
                log_n++;
                if (phase == 1) p1++; else p2++;
                next_c = -1;
            } else if (lane == 0) {
                piv.go = 0;
                s_fin[0] = status; s_fin[1] = p1; s_fin[2] = p2; s_fin[3] = log_n; s_fin[4] = overflow; s_fin[5] = unb;
                s_eval = Ms[(size_t)slot[0] * Ws];
            }
        }
        NODE_CY(2);
        __syncthreads();
        if (!piv.go) break;
        const int prs = piv.r, pcs = piv.c, flush = piv.flush, spare = s_spare;
        const double q = piv.q;
        // ---- D (CTA): both division passes at once: the lower half of the CTA normalises the pivot row
        // (simplex.ts:352-364 + lazy flush 380-382), the upper half rewrites the pivot column
        // (simplex.ts:371-374,386) after staging its old entries for the row updates.
        if (tid < NT / 2) {
            const double *praw = Ms + (size_t)slot[prs] * Ws;
#pragma unroll 1
            for (int c = tid; c < W; c += NT / 2) frow[c] = norm_entry<ddiv_z>(praw[c], c == pcs, q, flush);
        } else {
#pragma unroll 1
            for (int r = tid - NT / 2; r < Hn; r += NT / 2) {
                if (r == prs) { pcol[r] = 0.0; continue; }
                double *e = Ms + (size_t)slot[r] * Ws + pcs;
                const double coef = *e;
                pcol[r] = coef;
                if (nz16(coef)) *e = ddiv_z(-coef, q);  // else untouched (simplex.ts:371; :389-391 is dead code)
            }
        }
        NODE_CY(3);
        __syncthreads();
        // ---- U (CTA): simplex.ts:367-391.  Warp 0 owns the cost row and then prices it (look-ahead, off
        // the other warps' critical path); rows 1.. are dealt over the other warps.  A lane's columns are
        // the same for every row, so its share of the normalised pivot row lives in registers.
#pragma unroll 1
        for (int cb = 0; cb < W; cb += 128) {
            double fr[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int c = cb + lane + 32 * k;
                fr[k] = c < W ? frow[c] : 0.0;
            }
            const int rfirst = warp == 0 ? 0 : warp, rstep = warp == 0 ? Hn : NW - 1;
#pragma unroll 1
            for (int r = rfirst; r < Hn; r += rstep) {
                if (r == prs) {
                    double *dst = Ms + (size_t)spare * Ws;
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        const int c = cb + lane + 32 * k;
                        if (c < W) dst[c] = fr[k];
                    }
                    continue;
                }
                const double coef = pcol[r];
                if (!nz16(coef)) continue;
                double *row = Ms + (size_t)slot[r] * Ws;
                double v[4];
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const int c = cb + lane + 32 * k;
                    v[k] = c < W ? row[c] : 0.0;
                }
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const int c = cb + lane + 32 * k;
                    if (c < W && c != pcs && nz16(fr[k])) row[c] = __dsub_rn(v[k], __dmul_rn(coef, fr[k]));
                }
            }
        }
        if (warp == 0) {
            __syncwarp();
            next_c = warp_price(T, Ms + (size_t)slot[0] * Ws, vcol, W, lane, &next_neg);
        }
        NODE_CY(4);
        __syncthreads();
        NODE_CY(5);
        if (tid == 0) {
            const int old = slot[prs];
            slot[prs] = spare;
            s_spare = old;
        }
        __syncwarp();  // warp 0 reads the slot table next; every other warp waits at the next barrier
    }

    if (tid == 0) tl3 = globaltimer_ns() - t_start;
    if constexpr (SCENARIO)
        if (nb.cert_u != nullptr) {
            // the certificate row's multipliers of the requested rows, through the final labels (DESIGN.md 2u); sc.r
            // is still the row whose phase-1 column scan found no entering column
            const int st = s_fin[0], cr = st == ST_OPTIMAL ? 0 : st == ST_INFEASIBLE ? sc.r : -1;
            double *u = nb.cert_u + (size_t)node * nb.cert_n;
            if (cr < 0) {
                for (int i = tid; i < nb.cert_n; i += NT) u[i] = 0.0;
            } else {
                const double *crow = Ms + (size_t)slot[cr] * Ws;
                for (int c = 1 + tid; c < W; c += NT) {
                    const int l = vcol[c], i = l >= 0 && l < nb.cert_labels ? nb.cert_pos[l] : -1;
                    if (i >= 0) u[i] = crow[c];
                }
                for (int r = 1 + tid; r < Hn; r += NT) {
                    const int l = vrow[r], i = l >= 0 && l < nb.cert_labels ? nb.cert_pos[l] : -1;
                    if (i >= 0) u[i] = r == cr ? 1.0 : 0.0;
                }
            }
        }
    // isIntegral / most fractional variable over the final RHS column
    for (int r = tid; r < Hn; r += NT) rhs[r] = Ms[(size_t)slot[r] * Ws];
    __syncthreads();
    if constexpr (SCENARIO || COLUMNS || POOL || CONFLICT || FOREST)
        if (!(CONFLICT || FOREST) || nb.out_rhs != nullptr)  // row-subset and forest launches write them only when asked
            for (int r = tid; r < Hn; r += NT) {
                nb.out_rhs[(size_t)node * nb.Hcap + r] = rhs[r];
                nb.out_vrow[(size_t)node * nb.Hcap + r] = vrow[r];
            }
    // a row-subset launch without an integer mask has no scan: integral, as a tableau without integer variables
    if (T.intpos != nullptr && (!CONFLICT || nb.int_keep != nullptr)) {
        if (tid == 0) { T.M = rhs; T.stride = 1; T.vrow = vrow; T.H = Hn; }
        __syncthreads();
        cta_mip_scan<CONFLICT>(T, &mip, sel.red, CONFLICT ? nb.int_keep + (size_t)node * nb.int_words : nullptr);
    } else if (tid == 0) { mip.is_integral = 1; mip.var_index = -1; mip.value = 0.0; }
    __syncthreads();
    if (tid == 0) tl4 = globaltimer_ns() - t_start;
    NodeOut *out = nb.out + node;
    {
        const int nlog = min(min(s_fin[3], nb.log_cap), NODE_LOG_HEAD);
        for (int k = tid; k < nlog; k += NT) out->log_head[k] = plog[k];
    }
    if (nb.wb_M != nullptr && node == 0) {
        for (int r = warp; r < Hn; r += NW) {
            const double *row = Ms + (size_t)slot[r] * Ws;
            for (int c = lane; c < W; c += 32) nb.wb_M[(size_t)r * nb.root_stride + c] = row[c];
        }
        for (int r = tid; r < Hn; r += NT) nb.wb_vrow[r] = vrow[r];
        for (int c = tid; c < W; c += NT) nb.wb_vcol[c] = vcol[c];
    }
    if constexpr (FOREST)
        if (nb.col0 != nullptr) {  // a forest root: its final tableau becomes its tree's snapshot (jslp_save)
            const size_t s = (size_t)nb.root_of[node];
            double *dst = nb.slot_M + s * nb.slot_pitch;
            for (int r = warp; r < Hn; r += NW) {
                const double *row = Ms + (size_t)slot[r] * Ws;
                for (int c = lane; c < W; c += 32) dst[(size_t)r * nb.root_stride + c] = row[c];
            }
            for (int r = tid; r < Hn; r += NT) nb.slot_vrow[s * H0 + r] = vrow[r];
            for (int c = tid; c < W; c += NT) nb.slot_vcol[s * W + c] = vcol[c];
        }
    if (tid == 0) {
        NodeResult r;
        r.status = s_fin[0]; r.p1 = s_fin[1]; r.p2 = s_fin[2]; r.log_n = s_fin[3]; r.overflow = s_fin[4];
        r.is_integral = mip.is_integral; r.branch_var = mip.var_index; r.unbounded_var = s_fin[5];
        r.eval_raw = s_eval; r.branch_value = mip.value;
        r.t_ns = globaltimer_ns() - t_start; r.pad = 0;
        r.tl[0] = tl0; r.tl[1] = tl1; r.tl[2] = tl2; r.tl[3] = tl3; r.tl[4] = tl4; r.tl[5] = 0;
        for (int k = 0; k < 6; k++) r.cy[k] = cy[k];
        out->r = r;
    }
}

}  // namespace jslp
