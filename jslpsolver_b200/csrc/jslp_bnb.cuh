// jslpsolver_b200/csrc/jslp_bnb.cuh -- branch-and-cut frontier manager (included by jslp_api.cu).
//
// Replaces BranchAndCutService.branchAndCut (branch-and-cut.ts:54-199) and BranchMinHeap
// (min-heap.ts).  The commit order is the reference's: best-first on relaxedEvaluation, most
// recently pushed first on ties.  A node's LP result is a pure function of (root snapshot, cut
// list) (SURVEY.md 3.8), so the frontier is evaluated speculatively: every round takes the next K
// open nodes in exact pop order, evaluates them together on the device (one CTA per node when the
// tableau fits shared memory, else one after the other on the HBM path; sharded round-robin over
// ranks with an all-gather of the 128-byte summaries when n_ranks > 1), then COMMITS results
// sequentially in pop order exactly as the reference loop would.  A popped node without a cached
// result ends the round.  Speculation that is never popped is wasted work, never wrong work.
#pragma once

#include <chrono>
#include <map>
#include <memory>

#include "jslp_frontier.h"

// ---- node evaluation back-ends ---------------------------------------------------------------
// HBM path: applyCuts (branch-and-cut.ts:33-52) in place, exactly as the reference does it.
static int eval_node_streaming(jslp_tab *t, const jslp_bnb::Branch &b, int check_cycles, jslp_bnb::NodeEval &ev) {
    jslp_lp_status st;
    static const bool dbg = getenv("JSLP_DEBUG") != nullptr;
    auto tnow = [] { return std::chrono::steady_clock::now(); };
    auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b2) {
        return std::chrono::duration<double, std::micro>(b2 - a).count();
    };
    const auto t_0 = tnow();
    int rc = jslp_restore(t);
    if (rc) return rc;
    if (dbg) cudaStreamSynchronize(t->ctx->stream);
    const auto t_1 = tnow();
    rc = jslp_add_cuts(t, b.cuts.data(), (int)b.cuts.size());
    if (rc) return rc;
    if (dbg) cudaStreamSynchronize(t->ctx->stream);
    const auto t_2 = tnow();
    const double prevBest = t->bestPossibleEval;
    const int prevIters = t->simplexIters;
    int n_optimal = 0;
    double first_eval = 0;
    rc = simplex_with_mir(t, check_cycles, &st, false, &n_optimal, &first_eval);
    if (rc) return rc;
    const auto t_3 = tnow();
    // simplexIters / bestPossibleEval are frontier state: the commit loop owns them
    ev.optimal = n_optimal > 0;
    ev.n_optimal = t->use_mir ? n_optimal : -1;
    ev.first_eval = first_eval;
    t->simplexIters = prevIters;
    t->bestPossibleEval = prevBest;
    ev.valid = true;
    ev.feasible = t->feasible; ev.bounded = t->bounded; ev.evaluation = t->evaluation;
    ev.pivots = st.phase1_pivots + st.phase2_pivots;
    ev.is_integral = 0; ev.branch_var = -1; ev.branch_value = 0;
    if (ev.feasible) {
        MipOut mo;
        rc = mip_scan(t, &mo);
        if (rc) return rc;
        ev.is_integral = mo.is_integral; ev.branch_var = mo.var_index; ev.branch_value = mo.value;
        if (t->nOpt > 0) {
            std::vector<double> opt((size_t)t->nOpt * t->W);
            rc = jslp_download(t, nullptr, nullptr, nullptr, nullptr, nullptr, opt.data(), nullptr, nullptr);
            if (rc) return rc;
            for (int o = 0; o < t->nOpt && o < 7; o++) ev.opt0[o] = opt[(size_t)o * t->W];
        }
    }
    if (dbg)
        fprintf(stderr, "stream node: cuts %d pivots %d+%d restore %.0f us add_cuts %.0f us run_lp %.0f us rest %.0f us\n",
                (int)b.cuts.size(), st.phase1_pivots, st.phase2_pivots, us(t_0, t_1), us(t_1, t_2), us(t_2, t_3), us(t_3, tnow()));
    return JSLP_OK;
}

// A node LP the device ran on its own (node kernel or node slot) as eval_node_streaming reads it from the tableau:
// the status (ST_OPTIMAL, ST_UNBOUNDED, else infeasible), the raw evaluation, the pivots and the integrality scan,
// which only a feasible node carries.
static jslp_bnb::NodeEval node_eval(int status, double eval_raw, int pivots, int is_integral, int branch_var,
                                    double branch_value, double precision) {
    jslp_bnb::NodeEval ev;
    ev.valid = true;
    ev.pivots = pivots;
    ev.optimal = status == ST_OPTIMAL;
    ev.bounded = status != ST_UNBOUNDED;
    ev.feasible = status == ST_OPTIMAL || status == ST_UNBOUNDED;
    // infeasible: the evaluation is never read by the commit loop; 0 keeps it rank-independent on the wire
    ev.evaluation = status == ST_OPTIMAL ? jslp_round_evaluation(eval_raw, precision)
                                         : (status == ST_UNBOUNDED ? -INFINITY : 0.0);
    if (ev.feasible) { ev.is_integral = is_integral; ev.branch_var = branch_var; ev.branch_value = branch_value; }
    return ev;
}

// ---- K3: HBM-resident node batch (jslp_slots.cuh) ---------------------------------------------
// Largest number of slots for which every slot still runs the ping-pong step (at most 32 rows per row CTA,
// all B * (G + 2) CTAs co-resident), capped by the option and by what keeps the buffers being written in L2.
static int slots_for(const jslp_tab *t, int rowcap, int want) {
    if (t->node_slots == 0 || want < 2) return 0;
    if (!(t->pingpong && t->lookahead && t->nOpt == 0) || t->engine == 1) return 0;
    const StepVariant &sv = STEP_VARIANTS[t->slot_variant];
    int per_sm = t->grid_per_sm > 0 ? t->grid_per_sm : sv.ctas_per_sm;
    {   // every CTA of the slot batch must be co-resident (selectors wait for row CTAs of the same launch)
        int nb = 0;
        cudaFuncSetAttribute(sv.fn_pp, cudaFuncAttributeMaxDynamicSharedMemorySize, t->stride * 8);
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, sv.fn_pp, sv.threads, (size_t)t->stride * 8) != cudaSuccess) nb = 0;
        per_sm = std::min(per_sm, nb);
        if (per_sm < 1) return 0;
    }
    const int C = t->ctx->num_sms * per_sm;
    int geom = 0;
    for (int b = 1; b <= 64; b++) {
        const int G = C / b - 2;
        if (G < 1 || rowcap / G + 1 > 32) break;
        geom = b;
    }
    int cap = geom;
    if (t->node_slots > 0) cap = std::min(cap, t->node_slots);
    else {  // auto: the buffers being WRITTEN by all slots (half of each pair; the dead-load hint lets L2 drop the other
            // half first) should stay in L2: each pivot re-reads what the last one wrote
        const double live_bytes = 8.0 * (double)rowcap * t->stride;
        const int l2 = (int)std::floor(0.55 * (double)t->ctx->l2_bytes / live_bytes);
        cap = std::min(cap, std::max(2, l2));
    }
    return std::min(cap, want) >= 2 ? std::min(cap, want) : 0;
}

static int ensure_slots(jslp_tab *t, int B, int need_rowcap) {
    NodeSlots &ns = t->slots;
    jslp_ctx *ctx = t->ctx;
    cudaStream_t s = ctx->stream;
    const StepVariant &sv = STEP_VARIANTS[t->slot_variant];
    int per_sm = t->grid_per_sm > 0 ? t->grid_per_sm : sv.ctas_per_sm;
    {
        int nb = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, sv.fn_pp, sv.threads, (size_t)t->stride * 8) == cudaSuccess) per_sm = std::min(per_sm, std::max(1, nb));
    }
    const int G = ctx->num_sms * per_sm / B - 2;
    const int S = t->slot_steps;
    const int stride = t->stride;
    if (ns.B != B || ns.rowcap < need_rowcap) {
        CK(cudaStreamSynchronize(s));
        const int rowcap = std::max(need_rowcap + 32, std::max(ns.rowcap, t->saved.H + 64));
        ns.release();
        ns.B = B; ns.rowcap = rowcap;
        ns.plog_cap = 1024;
        const size_t tab = (size_t)rowcap * stride;
        CK(cudaMalloc(&ns.d_T, sizeof(TabDev) * B));
        CK(cudaMalloc(&ns.d_rec, sizeof(Rec) * B));
        CK(cudaMalloc(&ns.M, sizeof(double) * tab * B));
        CK(cudaMalloc(&ns.M2, sizeof(double) * tab * B));
        CK(cudaMalloc(&ns.prow, sizeof(double) * (size_t)stride * B));
        CK(cudaMalloc(&ns.pcol, sizeof(double) * (size_t)rowcap * B));
        CK(cudaMalloc(&ns.vrow, sizeof(int) * (size_t)rowcap * B));
        CK(cudaMalloc(&ns.vcol, sizeof(int) * (size_t)t->W * B));
        CK(cudaMalloc(&ns.part, sizeof(Part) * (size_t)(ctx->num_sms * 16) * B));
        CK(cudaMalloc(&ns.plog, sizeof(int4) * (size_t)ns.plog_cap * B));
        CK(cudaMallocHost(&ns.h_logs, sizeof(int4) * (size_t)ns.plog_cap * B));
        CK(cudaMemsetAsync(ns.M, 0, sizeof(double) * tab * B, s));
        CK(cudaMemsetAsync(ns.M2, 0, sizeof(double) * tab * B, s));
        CK(cudaMemsetAsync(ns.prow, 0, sizeof(double) * (size_t)stride * B, s));
        CK(cudaMemsetAsync(ns.pcol, 0, sizeof(double) * (size_t)rowcap * B, s));
        CK(cudaMemsetAsync(ns.part, 0xff, sizeof(Part) * (size_t)(ctx->num_sms * 16) * B, s));
        int rc;
        if ((rc = ResidentBufs::mapped(&ns.h_ctl, &ns.dv_ctl, sizeof(SlotCtl) * B))) return rc;
        if ((rc = ResidentBufs::mapped(&ns.h_out, &ns.dv_out, sizeof(SlotOut) * B))) return rc;
        ns.cuts_cap = B * (rowcap - t->saved.H);
        if ((rc = ResidentBufs::mapped(&ns.h_cuts, &ns.dv_cuts, sizeof(CutDev) * (size_t)std::max(1, ns.cuts_cap)))) return rc;
        std::vector<TabDev> hd((size_t)B, t->hd);
        std::vector<Rec> hr((size_t)B);
        for (int b = 0; b < B; b++) {
            TabDev &d = hd[b];
            d.M = ns.M + tab * b; d.M2 = ns.M2 + tab * b;
            d.prow = ns.prow + (size_t)stride * b;
            d.pcol = ns.pcol + (size_t)rowcap * b;
            d.vrow = ns.vrow + (size_t)rowcap * b; d.vcol = ns.vcol + (size_t)t->W * b;
            d.part = ns.part + (size_t)(ctx->num_sms * 16) * b;
            d.plog = ns.plog + (size_t)ns.plog_cap * b; d.plog_cap = ns.plog_cap;
            d.opt = nullptr; d.optcoef = nullptr; d.dbg = nullptr; d.dbg_cap = 0; d.dbg_grid = 0; d.nOpt = 0;
            d.W = t->W; d.H = t->saved.H; d.stride = stride; d.rowcap = rowcap;
            d.n_index = t->n_index; d.prec = t->precision;
            memset(&hr[b], 0, sizeof(Rec));
            hr[b].status = ST_P1_DONE;
            ns.h_ctl[b] = SlotCtl{SLOT_IDLE, 0, 0, 0};
        }
        CK(cudaMemcpyAsync(ns.d_T, hd.data(), sizeof(TabDev) * B, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(ns.d_rec, hr.data(), sizeof(Rec) * B, cudaMemcpyHostToDevice, s));
        CK(cudaStreamSynchronize(s));
        ns.key = -1;
    }
    // the graph bakes in the launch geometry and the snapshot it restores from
    const int key = (int)((((size_t)t->saved.M >> 4) * 2654435761u) ^ (size_t)(t->slot_variant * 131 + G * 7 + S * 1009 + t->saved.H * 31 +
                          t->saved.lastElementIndex * 17 + B)) & 0x7fffffff;
    if (ns.graph && ns.key == key && ns.G == G && ns.steps == S) return JSLP_OK;
    if (ns.graph) { cudaGraphExecDestroy(ns.graph); ns.graph = nullptr; }
    if (S + 2 > ns.plog_cap) return fail(JSLP_E_INVALID, "slot steps exceed the slot pivot-log capacity");
    if (G + 2 > ctx->num_sms * 16) return fail(JSLP_E_INVALID, "slot grid exceeds the partial-message buffer");
    const int smem = stride * 8;
    CK(cudaFuncSetAttribute(sv.fn_pp, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    SlotBatchDev sb;
    memset(&sb, 0, sizeof(sb));
    sb.T = ns.d_T; sb.rec = ns.d_rec; sb.ctl = ns.dv_ctl; sb.cuts = ns.dv_cuts; sb.out = ns.dv_out;
    sb.rootM = t->saved.M; sb.root_vrow = t->saved.vrow; sb.root_vcol = t->saved.vcol;
    sb.H0 = t->saved.H; sb.first_index = t->saved.lastElementIndex; sb.part_n = G + 2; sb.lookahead = 1;
    cudaGraph_t g;
    CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    k_slot_begin<<<dim3(std::max(8, G + 2), B), 256, 0, s>>>(sb);
    k_select<<<B, 512, 0, s>>>(ns.d_T, ns.d_rec, -1, -1);
    for (int i = 0; i < S; i++)
        sv.fn_pp<<<dim3(G + 2, B), sv.threads, smem, s>>>(ns.d_T, ns.d_rec, 2, ns.prow, stride);
    k_slot_end<<<B, 256, 0, s>>>(sb);
    cudaMemcpy2DAsync(ns.h_logs, sizeof(int4) * (size_t)(S + 2), ns.plog, sizeof(int4) * (size_t)ns.plog_cap,
                      sizeof(int4) * (size_t)(S + 2), B, cudaMemcpyDeviceToHost, s);
    cudaError_t e = cudaStreamEndCapture(s, &g);
    if (e != cudaSuccess) return fail(JSLP_E_CUDA, std::string("slot graph capture: ") + cudaGetErrorString(e));
    e = cudaGraphInstantiate(&ns.graph, g, 0);
    cudaGraphDestroy(g);
    if (e != cudaSuccess) return fail(JSLP_E_CUDA, std::string("slot graph instantiate: ") + cudaGetErrorString(e));
    ns.key = key; ns.G = G; ns.steps = S;
    return JSLP_OK;
}

// What a round shares between ranks while its node LPs are running (n_ranks > 1): element-wise min.
struct RoundExchange {
    const jslp_bnb_opts *opts;
    int n_ranks;
    std::vector<double> scratch;
    int64_t collectives = 0;
    int min(double *v, int n) {
        collectives++;
        if (opts->comm) return jslp_comm_all_reduce_min(opts->comm, v, n);
        scratch.assign((size_t)n * n_ranks, 0.0);
        memcpy(&scratch[(size_t)opts->rank * n], v, sizeof(double) * n);
        if (opts->all_gather(opts->user, scratch.data(), (int64_t)sizeof(double) * n)) return fail(JSLP_E_INVALID, "all_gather hook failed");
        jslp_bnb::fold_min(scratch.data(), n_ranks, n, v);
        return JSLP_OK;
    }
    int gather(void *buf, int64_t bytes_per_rank) {
        collectives++;
        if (opts->comm) return jslp_comm_all_gather(opts->comm, buf, bytes_per_rank);
        if (opts->all_gather(opts->user, buf, bytes_per_rank)) return fail(JSLP_E_INVALID, "all_gather hook failed");
        return JSLP_OK;
    }
};

// Evaluates nodes[0..n) in B slots side by side.  Nodes whose pivot log shows a cycle are re-evaluated on the
// single-tableau HBM path (exact stop-before-the-repeat semantics there).
//
// *U is the incumbent bound of the round: the smallest evaluation of an integral feasible node known so far
// (committed incumbent, cached results, nodes finished in this call -- on any rank when `ex` is set: one
// all-reduce(min) per poll keeps the ranks' poll loops in lockstep and shares the bound).  A speculative node
// whose relaxedEvaluation exceeds it is dropped or aborted: it sorts after the node that set the bound, so by
// the time the reference's loop pops it bestEvaluation <= U < relaxedEvaluation and it is skipped unevaluated
// (branch-and-cut.ts:90-92).  Pruned nodes keep ev.valid == false.
static int eval_nodes_slots(jslp_tab *t, jslp_bnb::Branch *const *nodes, int n, int B, int check_cycles, double *U,
                            RoundExchange *ex, int64_t *pruned) {
    jslp_ctx *ctx = t->ctx;
    cudaStream_t s = ctx->stream;
    int maxc = 0;
    for (int i = 0; i < n; i++) maxc = std::max(maxc, (int)nodes[i]->cuts.size());
    int rc = ensure_slots(t, B, t->saved.H + maxc);
    if (rc) return rc;
    NodeSlots &ns = t->slots;
    const int S = ns.steps;
    static const bool dbg = getenv("JSLP_DEBUG") != nullptr;
    std::vector<int> node_of((size_t)B, -1), redo;
    std::vector<CycleHist> hist((size_t)2 * B);
    int next = 0, done = 0;
    auto account = [&](int i, int pivots) {
        t->slot_pivots += pivots;
        t->slot_bytes += 16.0 * (double)(t->saved.H + (int)nodes[i]->cuts.size()) * t->stride * pivots;
    };
    bool any = n > 0 || ex != nullptr;
    while (any) {
        if (done < n) {
            int tot = 0;
            for (int b = 0; b < B; b++) {
                if (node_of[b] >= 0 && nodes[node_of[b]]->relaxedEvaluation > *U) {  // abort: the reference skips it
                    account(node_of[b], ns.h_out[b].rec.p1 + ns.h_out[b].rec.p2);
                    node_of[b] = -1; done++; (*pruned)++;
                }
                while (node_of[b] < 0 && next < n && nodes[next]->relaxedEvaluation > *U) { next++; done++; (*pruned)++; }
                if (node_of[b] < 0 && next < n) {
                    const std::vector<jslp_cut> &cuts = nodes[next]->cuts;
                    if (tot + (int)cuts.size() > ns.cuts_cap) return fail(JSLP_E_CAPACITY, "slot cut buffer overflow");
                    ns.h_ctl[b] = SlotCtl{SLOT_LOAD, (int)cuts.size(), tot, 0};
                    for (const jslp_cut &c : cuts) {
                        ns.h_cuts[tot].type = c.type; ns.h_cuts[tot].var_index = c.var_index; ns.h_cuts[tot].value = c.value;
                        tot++;
                    }
                    node_of[b] = next++;
                    hist[2 * b] = CycleHist(); hist[2 * b + 1] = CycleHist();
                } else {
                    ns.h_ctl[b].cmd = node_of[b] >= 0 ? SLOT_CONTINUE : SLOT_IDLE;
                }
            }
        }
        int running = 0;
        for (int b = 0; b < B; b++) running += node_of[b] >= 0;
        if (running > 0) {
            const auto t_g = std::chrono::steady_clock::now();
            CK(cudaGraphLaunch(ns.graph, s));
            ctx->launches += 3 + S;
            CK(cudaStreamSynchronize(s));
            const double us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t_g).count();
            t->slot_ms += 1e-3 * us;
            if (dbg) {
                int loads = 0;
                for (int b = 0; b < B; b++) loads += ns.h_ctl[b].cmd == SLOT_LOAD;
                fprintf(stderr, "slot graph: B %d G %d S %d running %d loads %d: %.0f us\n", B, ns.G, S, running, loads, us);
            }
            for (int b = 0; b < B; b++) {
                const int i = node_of[b];
                if (i < 0) continue;
                const Rec &r = ns.h_out[b].rec;
                if (r.status == ST_ERROR) return fail(JSLP_E_CUDA, "slot batch: selector CTA timed out waiting for row CTAs");
                if (r.log_n > S + 2) return fail(JSLP_E_CAPACITY, "slot pivot log overflow inside one batch");
                bool hit = false;
                if (check_cycles) {
                    const int4 *lg = ns.h_logs + (size_t)b * (S + 2);
                    int cs, cl;
                    for (int k = 0; k < r.log_n && !hit; k++) {
                        CycleHist &h = hist[2 * b + (((lg[k].x >> 30) & 1) ? 1 : 0)];
                        hit = h.push_and_check(((long long)lg[k].z << 32) | (unsigned int)lg[k].w, &cs, &cl);
                    }
                }
                if (hit) { account(i, r.p1 + r.p2); redo.push_back(i); node_of[b] = -1; done++; continue; }
                if (r.status == ST_RUNNING) continue;
                const MipOut &mo = ns.h_out[b].mip;
                const jslp_bnb::NodeEval &ev = nodes[i]->ev =
                    node_eval(r.status, r.eval_raw, r.p1 + r.p2, mo.is_integral, mo.var_index, mo.value, t->precision);
                if (ev.feasible && ev.is_integral && ev.evaluation < *U) *U = ev.evaluation;
                account(i, ev.pivots);
                if (dbg) fprintf(stderr, "slot node: slot %d cuts %d pivots %d+%d status %d\n", b, (int)nodes[i]->cuts.size(), r.p1, r.p2, r.status);
                node_of[b] = -1;
                done++;
            }
        }
        if (ex) {  // share the bound; stay in the loop until every rank has finished its nodes
            double v[2] = {*U, done < n ? -1.0 : 0.0};
            rc = ex->min(v, 2);
            if (rc) return rc;
            *U = v[0];
            any = v[1] < 0;
        } else {
            any = done < n;
        }
    }
    for (int i : redo) {
        if (nodes[i]->relaxedEvaluation > *U) { (*pruned)++; t->cycle_redos_pruned++; continue; }
        t->cycle_redos_slots++;
        rc = eval_node_streaming(t, *nodes[i], check_cycles, nodes[i]->ev);
        if (rc) return rc;
    }
    return JSLP_OK;
}

// Evaluates nodes[0..n) with one CTA each (k_node_batch<NODE_BRANCH>).  Nodes whose log shows a cycle or that hit the
// in-kernel pivot or log cap are re-evaluated on the HBM path (exact cycle semantics there).
static int eval_nodes_resident(jslp_tab *t, jslp_bnb::Branch *const *nodes, int n, int check_cycles) {
    const ResidentBufs &rb = t->rbufs;
    NodeBatchDev nb;
    size_t smem = 0;
    int rc = batch_fill(t, t->saved.M, t->saved.vrow, t->saved.vcol, t->saved.H, t->saved.lastElementIndex, n, nb,
                        &smem);
    if (rc) return rc;
    rc = branch_cuts(t, n, [&](int k) { return nodes[k]; }, nb);
    if (rc) return rc;
    int maxc = 0;
    for (int i = 0; i < n; i++) maxc = std::max(maxc, (int)nodes[i]->cuts.size());
    nb.Hcap = t->saved.H + maxc;
    smem = node_smem_bytes(nb.Hcap, t->W, nullptr);
    rc = batch_launch<NODE_BRANCH>(t, nb, n, smem, nullptr, nullptr);
    if (rc) return rc;
    long long slowest = 0;
    static const bool dbg = getenv("JSLP_DEBUG") != nullptr;  // per-node timeline on stderr (scripts/node_timeline.py)
    for (int i = 0; i < n; i++) {
        const NodeResult &q = rb.h_out[i].r;
        if (dbg)
            fprintf(stderr, "node r%d n%d i%d cuts %d piv %d+%d: off %lld restore %lld cuts %lld pivots %lld mip %lld end %lld cy %lld %lld %lld %lld %lld %lld\n",
                    (int)t->ctx->launches, n, i, (int)nodes[i]->cuts.size(), q.p1, q.p2, q.tl[0], q.tl[1], q.tl[2], q.tl[3], q.tl[4], q.t_ns, q.cy[0], q.cy[1], q.cy[2], q.cy[3], q.cy[4], q.cy[5]);
        slowest = std::max(slowest, q.t_ns);
    }
    t->node_kernel_ns += slowest;
    std::vector<int> hit, redo;
    rc = batch_screen(t, n, [&](int i) { return check_cycles && !rb.h_out[i].r.overflow; }, hit);
    if (rc) return rc;
    for (int i = 0; i < n; i++) {
        const NodeResult &r = rb.h_out[i].r;
        if (r.overflow || hit[i] >= 0) {
            t->cycle_redos_kernel += hit[i] >= 0;
            redo.push_back(i);  // second pass: the HBM path may reuse rb's buffers
            continue;
        }
        nodes[i]->ev =
            node_eval(r.status, r.eval_raw, r.p1 + r.p2, r.is_integral, r.branch_var, r.branch_value, t->precision);
    }
    for (int i : redo) {
        rc = eval_node_streaming(t, *nodes[i], check_cycles, nodes[i]->ev);
        if (rc) return rc;
    }
    return JSLP_OK;
}

// The starts of jslp_branch_and_cut_start (DESIGN.md section 2t): start i is cuts[off[i] .. off[i + 1]).
struct StartSet {
    const jslp_cut *cuts;
    const int32_t *off;
    int n;
    int64_t max_nodes;
    jslp_start_status *st;
};

// jslp_branch_and_cut, seeded by the starts of ss when it is set.
static int branch_and_cut(jslp_tab *t, const jslp_bnb_opts *opts, const StartSet *ss, jslp_bnb_status *out,
                          jslp_cut *best_cuts, int best_cuts_cap) {
    using namespace jslp_bnb;
    if (!t || !opts) return fail(JSLP_E_INVALID, "NULL argument");
    if (t->n_int <= 0) return fail(JSLP_E_INVALID, "branch_and_cut needs integer variables (upload int_var_indices)");
    const int n_ranks = std::max(1, opts->n_ranks), rank = opts->rank;
    if (n_ranks > 1 && !opts->all_gather && !opts->comm) return fail(JSLP_E_INVALID, "n_ranks > 1 needs a communicator or an all_gather hook");
    if (n_ranks > 1 && t->nOpt > 7) return fail(JSLP_E_UNSUPPORTED, "more than 7 optional objectives across ranks");
    if (opts->service == 1 || opts->service == 2) return bnb_enhanced(t, opts, out, best_cuts, best_cuts_cap);  // sequential by construction
    if (opts->service != 0) return fail(JSLP_E_UNSUPPORTED, "unknown branch-and-cut service");
    jslp_ctx *ctx = t->ctx;
    CK(cudaSetDevice(ctx->device));
    const int64_t launches0 = ctx->launches;
    CK(cudaEventRecord(ctx->ev0, ctx->stream));
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto ms_since = [](std::chrono::steady_clock::time_point t0) {
        return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    };
    const auto t_start = now();
    const double timeout_ms = opts->timeout_ms > 0 ? opts->timeout_ms : 0;  // branch-and-cut.ts:61-63
    auto time_up = [&] { return timeout_ms > 0 && ms_since(t_start) >= timeout_ms; };

    Tree tree(t->nOpt);
    Frontier &branches = tree.branches;
    const int &iterations = tree.iterations;
    int rounds = 0;
    const int check_cycles = opts->check_cycles;
    bool timed_out = false;
    int64_t nodes = 0, pruned = 0;
    t->node_log.clear();
    t->solutions.clear();
    t->saved.valid = false;
    t->isIntegralFlag = 0;
    t->slot_pivots = 0; t->slot_ms = 0; t->slot_bytes = 0;
    t->cycle_redos_kernel = 0; t->cycle_redos_slots = 0; t->cycle_redos_pruned = 0;
    int K = opts->max_spec_batch > 0 ? opts->max_spec_batch : 16;  // any width commits in the same order
    std::vector<double> wire;
    RoundExchange ex{opts, n_ranks, {}, 0};
    const Tree::Rule rule{opts->tolerance, opts->is_minimization, t->nOpt, opts->max_nodes};

    // keep_solutions (branch-and-cut.ts:143-153): the incumbent's tableau state, as generateSolutionSet reads it.
    // Node evaluators return summaries only, so the node is solved once more in place (incumbents are rare).
    auto store_solution = [&](const Branch &b) -> int {
        NodeEval ev;
        int rc = eval_node_streaming(t, b, check_cycles, ev);
        if (rc) return rc;
        jslp_tab::StoredSolution sol;
        sol.evaluation = t->evaluation;
        sol.vrow.resize((size_t)t->H);
        sol.rhs.resize((size_t)t->H);
        rc = jslp_download(t, nullptr, sol.rhs.data(), nullptr, sol.vrow.data(), nullptr, nullptr, nullptr, nullptr);
        if (rc) return rc;
        t->solutions.push_back(std::move(sol));
        return JSLP_OK;
    };

    // The tab's scalars as the call finds them become the tree's (the root's log row reads Tableau.evaluation when the
    // root is infeasible); from then on the tree's are the authority and store() copies them to the tab after every
    // round and commit.  A node LP run in place on the single-tableau path sets the tab's evaluation when it runs, not
    // when its turn to commit comes, and keep_solutions' re-solves set it again: neither may reach the tree.
    auto load = [&] {
        tree.feasible = t->feasible; tree.bounded = t->bounded; tree.evaluation = t->evaluation;
        tree.bestPossibleEval = t->bestPossibleEval; tree.simplexIters = t->simplexIters; tree.isIntegral = t->isIntegralFlag;
    };
    auto store = [&] {
        t->feasible = tree.feasible; t->bounded = tree.bounded; t->evaluation = tree.evaluation;
        t->bestPossibleEval = tree.bestPossibleEval; t->simplexIters = tree.simplexIters; t->isIntegralFlag = tree.isIntegral;
    };

    // One round's node LPs, todo in pop order, on the path their heights and the options choose: shared-memory node
    // batch, node slots or one after another on the single-tableau path, sharded over the ranks as the options ask.  U
    // is the round's incumbent bound (see eval_nodes_slots); count gains this rank's node LPs.
    auto eval_round = [&](std::vector<Branch *> &todo, double &U, int64_t &count) -> int {
        int maxc_all = 0;
        for (Branch *b : todo) maxc_all = std::max(maxc_all, (int)b->cuts.size());
        // every rank takes the same decisions from the same (rank-independent) quantities
        // useMIRCuts: the MIR loop (fractional volume, cut rows, re-solves) runs on the single-tableau path
        const bool resident = iterations > 0 && t->saved.valid && t->engine != 1 && t->engine != 2 && !t->use_mir &&
                              resident_fits(t, t->saved.H + maxc_all);
        const int nslots = (!resident && !t->use_mir && iterations > 0 && t->saved.valid && todo.size() >= 2)
                               ? slots_for(t, t->saved.H + maxc_all, std::max(K, (int)todo.size())) : 0;
        // The root round is NOT sharded: every rank needs the solved root in its own tableau, it is what
        // jslp_save snapshots and what every later node is derived from.  Rounds of nodes that fit shared
        // memory are not sharded either unless asked: a whole round costs less than one collective.
        const bool sharded = n_ranks > 1 && iterations > 0 && !t->use_mir && (opts->shard_policy == 1 || !resident);
        std::vector<Branch *> mine;
        for (size_t i = 0; i < todo.size(); i++)
            if (!sharded || deal_rank(i, n_ranks) == rank) mine.push_back(todo[i]);
        if (resident) {
            if (!mine.empty()) {
                int rc = eval_nodes_resident(t, mine.data(), (int)mine.size(), check_cycles);
                if (rc) return rc;
            }
        } else if (nslots >= 2) {
            int rc = eval_nodes_slots(t, mine.data(), (int)mine.size(), nslots, check_cycles, &U, sharded ? &ex : nullptr, &pruned);
            if (rc) return rc;
        } else {
            for (Branch *b : mine) {
                if (b->relaxedEvaluation > U) { pruned++; continue; }
                int rc = eval_node_streaming(t, *b, check_cycles, b->ev);
                if (rc) return rc;
                if (b->ev.feasible && b->ev.is_integral && b->ev.evaluation < U) U = b->ev.evaluation;
            }
        }
        count += (int64_t)mine.size();
        if (sharded) {  // all-gather the summaries: rank-major blocks of `per` records
            const WireDeal deal(todo.size(), n_ranks);
            wire.assign((size_t)deal.per * n_ranks * WIRE_DOUBLES, 0.0);
            for (size_t i = 0; i < todo.size(); i++)
                if (deal_rank(i, n_ranks) == rank) to_wire(todo[i]->ev, &wire[deal.slot(i) * WIRE_DOUBLES]);
            int rc = ex.gather(wire.data(), (int64_t)deal.per * WIRE_DOUBLES * 8);
            if (rc) return rc;
            for (size_t i = 0; i < todo.size(); i++) from_wire(todo[i]->ev, &wire[deal.slot(i) * WIRE_DOUBLES]);
        }
        return JSLP_OK;
    };

    // The seed stage (DESIGN.md section 2t), run where the root was committed fractional and snapshotted: every
    // start's node from the snapshot, then depth-first dives from the feasible fractional ones, one node of every live
    // dive per wave, each wave one eval_round.  The best integral node becomes the incumbent; the tableau and the
    // tab's scalar state are then put back as the root left them.
    auto seed_stage = [&]() -> int {
        struct Dive {
            std::vector<std::unique_ptr<Branch>> stack;  // top = back
            std::unique_ptr<Branch> found;
            bool live = true;
        };
        std::vector<Dive> dives((size_t)ss->n);
        for (int i = 0; i < ss->n; i++) {
            dives[i].stack.emplace_back(new Branch{
                -INFINITY, std::vector<jslp_cut>(ss->cuts + ss->off[i], ss->cuts + ss->off[i + 1]), NodeEval()});
            ss->st[i].status = JSLP_START_INFEASIBLE;
        }
        for (;;) {
            std::vector<Branch *> wave;
            std::vector<int> who;
            for (int i = 0; i < ss->n; i++) {
                Dive &d = dives[i];
                if (!d.live) continue;
                if (d.stack.empty()) { d.live = false; continue; }
                if (ss->st[i].nodes >= ss->max_nodes) { ss->st[i].status = JSLP_START_INCOMPLETE; d.live = false; continue; }
                wave.push_back(d.stack.back().get());
                who.push_back(i);
            }
            if (wave.empty()) break;
            double U = INFINITY;  // a start node sorts before nothing: none is dropped
            int64_t count = 0;
            int rc = eval_round(wave, U, count);
            if (rc) return rc;
            for (int i : who) {
                Dive &d = dives[i];
                jslp_start_status &st = ss->st[i];
                std::unique_ptr<Branch> b = std::move(d.stack.back());
                d.stack.pop_back();
                const NodeEval ev = b->ev;
                st.nodes++;
                st.pivots += ev.pivots;
                if (!ev.feasible) continue;
                if (ev.is_integral) {
                    st.status = JSLP_START_FEASIBLE;
                    st.evaluation = ev.evaluation;
                    st.n_cuts = (int)b->cuts.size();
                    d.found = std::move(b);
                    d.live = false;
                    continue;
                }
                std::unique_ptr<Branch> high, low;
                Tree::children(*b, ev.branch_var, ev.branch_value, -INFINITY, high, low);
                const bool up = ev.branch_value - std::floor(ev.branch_value) >= 0.5;  // the nearer child on top
                d.stack.push_back(std::move(up ? low : high));
                d.stack.push_back(std::move(up ? high : low));
            }
        }
        int best = -1;
        for (int i = 0; i < ss->n; i++)
            if (dives[i].found && (best < 0 || ss->st[i].evaluation < ss->st[best].evaluation)) best = i;
        if (best >= 0) {
            ss->st[best].status = JSLP_START_SEED;
            tree.seed(std::move(dives[best].found->cuts), ss->st[best].evaluation);
            if (opts->keep_solutions) {
                int rc = store_solution(*tree.bestBranch);
                if (rc) return rc;
            }
        }
        int rc = jslp_restore(t);
        if (rc) return rc;
        store();
        return JSLP_OK;
    };

    double eval_ms = 0, commit_ms = 0, root_ms = 0, final_ms = 0;
    t->node_kernel_ns = 0;
    bool stop = false;
    load();
    while (!stop && !branches.empty() && tree.toleranceFlag) {
        // ---- speculate: evaluate the next K un-evaluated open nodes in pop order ---------------
        const int width = iterations == 0 ? 1 : K;  // the root decides everything: alone
        std::vector<Frontier::Entry> taken;
        std::vector<Branch *> todo;
        double U = tree.speculate(width, taken, todo, pruned);  // the round's incumbent bound (see eval_nodes_slots)
        const auto t_eval = now();
        if (!todo.empty()) {
            rounds++;
            int rc = eval_round(todo, U, nodes);
            if (rc) return rc;
            store();  // a speculated node's evaluation is the commit's to write
        }
        tree.put_back(taken);
        if (iterations == 0) root_ms += ms_since(t_eval);
        eval_ms += ms_since(t_eval);
        const auto t_commit = now();

        // Date.now() < terminalTime (branch-and-cut.ts:76).  One rank: tested before every commit, like the
        // reference's loop condition.  Several ranks: tested once per round and agreed on (min-reduce), so that
        // every rank stops at the same commit.
        bool round_time_up = false;
        if (n_ranks > 1 && timeout_ms > 0) {
            double v = time_up() ? -1.0 : 0.0;
            int rc = ex.min(&v, 1);
            if (rc) return rc;
            round_time_up = v < 0;
        }

        // ---- commit sequentially in the reference's exact order ---------------------------------
        for (;;) {
            const Tree::Step st = tree.step(rule, [&] { return n_ranks > 1 ? round_time_up : time_up(); });
            store();
            if (st == Tree::DONE || st == Tree::ROUND) break;
            if (st == Tree::LIMIT || st == Tree::EARLY) { stop = true; break; }
            if (st == Tree::TIMED_OUT) { timed_out = true; stop = true; break; }
            if (st == Tree::SNAPSHOT) {  // snapshot = optimal root tableau (branch-and-cut.ts:155-157)
                int rc = jslp_save(t);
                if (rc) return rc;
                if (ss && tree.bounded) {
                    rc = seed_stage();
                    if (rc) return rc;
                }
            } else if (st == Tree::INCUMBENT && opts->keep_solutions) {
                int rc = store_solution(*tree.lastCommitted);
                if (rc) return rc;
            }
        }
        commit_ms += ms_since(t_commit);
    }

    // Final tableau: the reference re-solves the winner (branch-and-cut.ts:195-197); without a
    // winner it is left at the last evaluated node.  In place on the HBM path.
    int n_best = 0;
    int64_t pivots = tree.pivots;
    const std::unique_ptr<Branch> &bestBranch = tree.bestBranch;
    if (const Branch *fin = tree.final_branch()) {
        const auto t_fin = now();
        NodeEval ev;
        int rc = eval_node_streaming(t, *fin, check_cycles, ev);
        if (rc) return rc;
        nodes++;
        if (bestBranch) {
            pivots += ev.pivots;
            if (ev.optimal) t->simplexIters += ev.n_optimal >= 0 ? ev.n_optimal : 1;
        }
        final_ms = ms_since(t_fin);
    }
    if (bestBranch && !tree.early_return) {
        n_best = (int)bestBranch->cuts.size();
        if (best_cuts)
            for (int i = 0; i < n_best && i < best_cuts_cap; i++) best_cuts[i] = bestBranch->cuts[i];
    }
    t->bncIterations = iterations;
    t->node_log = std::move(tree.node_log);

    float ms = 0.f;
    CK(cudaEventRecord(ctx->ev1, ctx->stream));
    CK(cudaEventSynchronize(ctx->ev1));
    CK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
    if (out) {
        memset(out, 0, sizeof(*out));
        out->feasible = t->feasible; out->bounded = t->bounded; out->is_integral = t->isIntegralFlag;
        out->iterations = iterations; out->n_best_cuts = n_best; out->rounds = rounds;
        out->nodes_evaluated = nodes; out->pivots = pivots; out->evaluation = t->evaluation;
        out->best_possible_eval = t->bestPossibleEval; out->gpu_ms = ms;
        out->kernel_launches = ctx->launches - launches0;
        out->host_eval_ms = eval_ms; out->host_commit_ms = commit_ms;
        out->host_root_ms = root_ms; out->host_final_ms = final_ms; out->node_kernel_ms = 1e-6 * (double)t->node_kernel_ns;
        out->timed_out = timed_out ? 1 : 0; out->n_solutions = (int)t->solutions.size();
        out->nodes_pruned = pruned; out->collectives = ex.collectives;
        out->slot_pivots = t->slot_pivots; out->slot_ms = t->slot_ms; out->slot_bytes = t->slot_bytes;
        out->cycle_redos_kernel = t->cycle_redos_kernel; out->cycle_redos_slots = t->cycle_redos_slots;
        out->cycle_redos_pruned = t->cycle_redos_pruned;
    }
    return JSLP_OK;
}

extern "C" int jslp_branch_and_cut(jslp_tab *t, const jslp_bnb_opts *opts, jslp_bnb_status *out,
                                   jslp_cut *best_cuts, int best_cuts_cap) {
    return branch_and_cut(t, opts, nullptr, out, best_cuts, best_cuts_cap);
}

extern "C" int jslp_branch_and_cut_start(jslp_tab *t, const jslp_bnb_opts *opts, const jslp_cut *start_cuts,
                                         const int32_t *start_offsets, int n_starts, int64_t start_nodes,
                                         jslp_start_status *starts, jslp_bnb_status *out, jslp_cut *best_cuts,
                                         int best_cuts_cap) {
    if (n_starts == 0) return branch_and_cut(t, opts, nullptr, out, best_cuts, best_cuts_cap);
    if (!t || !opts) return fail(JSLP_E_INVALID, "NULL argument");
    if (n_starts < 0 || !start_offsets || !starts) return fail(JSLP_E_INVALID, "branch_and_cut_start: bad starts / offsets / status arguments");
    if (start_nodes < 1) return fail(JSLP_E_INVALID, "branch_and_cut_start: start_nodes must be at least 1");
    if (opts->service != 0) return fail(JSLP_E_UNSUPPORTED, "branch_and_cut_start: MIP starts need the default branch-and-cut service");
    if (opts->n_ranks > 1) return fail(JSLP_E_UNSUPPORTED, "branch_and_cut_start: MIP starts run on one GPU (n_ranks must be 1)");
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, "branch_and_cut_start: optional objectives are not supported");
    int rc = batch_check_offsets({start_offsets}, n_starts, "branch_and_cut_start", "start_offsets[0]");
    if (rc) return rc;
    if (start_offsets[n_starts] > 0 && !start_cuts) return fail(JSLP_E_INVALID, "branch_and_cut_start: start_cuts is NULL");
    for (int k = 0; k < start_offsets[n_starts]; k++) {
        const int v = start_cuts[k].var_index;
        if ((start_cuts[k].type != 0 && start_cuts[k].type != 1) || v < 0 || v >= (int)t->h_intpos.size() ||
            t->h_intpos[v] < 0)
            return fail(JSLP_E_INVALID, "branch_and_cut_start: a start cut is type 0 (min) or 1 (max) on an integer label");
    }
    for (int i = 0; i < n_starts; i++) starts[i] = jslp_start_status{JSLP_START_SKIPPED, 0, 0, 0, NAN};
    const StartSet ss{start_cuts, start_offsets, n_starts, start_nodes, starts};
    return branch_and_cut(t, opts, &ss, out, best_cuts, best_cuts_cap);
}

extern "C" int jslp_bnb_solution(jslp_tab *t, int i, double *evaluation, int32_t *height, int32_t *vrow, double *rhs, int cap) {
    if (!t) return fail(JSLP_E_INVALID, "tab is NULL");
    if (i < 0 || i >= (int)t->solutions.size()) return fail(JSLP_E_INVALID, "solution index out of range");
    const jslp_tab::StoredSolution &s = t->solutions[(size_t)i];
    if (evaluation) *evaluation = s.evaluation;
    if (height) *height = (int32_t)s.vrow.size();
    const size_t n = std::min<size_t>((size_t)std::max(0, cap), s.vrow.size());
    if (vrow) memcpy(vrow, s.vrow.data(), sizeof(int32_t) * n);
    if (rhs) memcpy(rhs, s.rhs.data(), sizeof(double) * n);
    return JSLP_OK;
}

extern "C" int jslp_bnb_node_log(jslp_tab *t, double *entries, int64_t cap, int64_t *n) {
    if (!t || !n) return fail(JSLP_E_INVALID, "NULL argument");
    const int64_t m = std::min<int64_t>((int64_t)t->node_log.size(), cap);
    for (int64_t i = 0; i < m && entries; i++) memcpy(entries + 8 * i, t->node_log[i].v, sizeof(double) * 8);
    *n = (int64_t)t->node_log.size();
    return JSLP_OK;
}
