// jslpsolver_b200/csrc/jslp_forest.cuh -- the branch and cut of many right-hand-side / cost scenarios of one model side
// by side (included by jslp_api.cu after jslp_pool.cuh; no reference counterpart).  DESIGN.md section 2p is the
// contract: tree s is jslp_branch_and_cut's default service over the tab's tableau with rows 1.. of column 0 and row 0
// replaced by scenario s's, committed through the same jslp_bnb::Tree.
//
// Every round takes the next `width` open nodes of every live tree in pop order and evaluates them together: nodes
// whose rows fit shared memory run one CTA each in k_node_batch<NODE_FOREST> launches, each restoring its own tree's
// root slot; the others, and any node whose log shows a cycle or that hits the pivot or log cap, run one after another
// on the single-tableau path (the slot copied into the snapshot, then eval_node_streaming).  Roots run the same way
// from the base tableau, and each root's final tableau becomes its tree's slot: the snapshot jslp_branch_and_cut takes
// at iteration 1.
#pragma once

namespace jslp {

// Rows 1.. of column 0 and row 0 of an H x W tableau at `stride` from c0 / r0 (a single-tableau forest root).
__global__ void __launch_bounds__(256) k_write_edges(double *M, int stride, int H, int W, const double *c0,
                                                     const double *r0) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= 1 && i < H) M[(size_t)i * stride] = c0[i];
    if (i < W) M[i] = r0[i];
}

}  // namespace jslp

// Tree groups are sized so that their root slots stay within this many bytes of device memory (DESIGN.md 2p).
static const size_t FOREST_SLOT_BYTES = (size_t)1 << 30;

struct Forest {
    jslp_tab *t;
    int H0, W, G, check_cycles;   // G = trees in the current group
    double *baseM;                // the tab's tableau on entry (device copy)
    int *base_vrow, *base_vcol;
    double *slotM;                // root slots of the current group: pitch doubles each
    int *slot_vrow, *slot_vcol;
    double *d_edges;              // the group's columns 0 (H0 each), then its rows 0 (W each)
    size_t pitch;
    int nVars, lastElementIndex;  // the tab's on entry

    const double *col0(int s) const { return d_edges + (size_t)s * H0; }
    const double *row0(int s) const { return d_edges + (size_t)G * H0 + (size_t)s * W; }

    // The snapshot <- H0 rows and labels (device) at the tab's entry size, for the single-tableau path and for the
    // restore of the caller's tableau.
    int load_saved(const double *M, const int *vrow, const int *vcol) {
        cudaStream_t s = t->ctx->stream;
        Saved &sv = t->saved;
        sv.valid = true; sv.H = H0; sv.nVars = nVars; sv.lastElementIndex = lastElementIndex;
        CK(cudaMemcpyAsync(t->saved.M, M, sizeof(double) * (size_t)H0 * t->stride, cudaMemcpyDeviceToDevice, s));
        CK(cudaMemcpyAsync(t->saved.vrow, vrow, sizeof(int) * (size_t)H0, cudaMemcpyDeviceToDevice, s));
        CK(cudaMemcpyAsync(t->saved.vcol, vcol, sizeof(int) * (size_t)W, cudaMemcpyDeviceToDevice, s));
        return JSLP_OK;
    }
};

struct ForestNode {
    int tree;                  // index within the group
    jslp_bnb::Branch *b;       // cuts in, ev out
    double *rhs;               // final column 0 and labels when set (roots and the final round)
    int32_t *vrow;
};

// One node on the single-tableau path: eval_node_streaming from the tree's slot, or, for a root, from the base with the
// tree's column 0 and row 0 written over it; a root's final tableau then becomes its slot.
static int forest_hbm(Forest &f, const ForestNode &n, bool root) {
    jslp_tab *t = f.t;
    cudaStream_t s = t->ctx->stream;
    int rc = root ? f.load_saved(f.baseM, f.base_vrow, f.base_vcol)
                  : f.load_saved(f.slotM + (size_t)n.tree * f.pitch, f.slot_vrow + (size_t)n.tree * f.H0,
                                 f.slot_vcol + (size_t)n.tree * f.W);
    if (rc) return rc;
    if (root) {
        k_write_edges<<<(std::max(f.H0, f.W) + 255) / 256, 256, 0, s>>>(t->saved.M, t->stride, f.H0, f.W, f.col0(n.tree),
                                                                       f.row0(n.tree));
        t->ctx->launches += 1;
        CK(cudaGetLastError());
    }
    rc = eval_node_streaming(t, *n.b, f.check_cycles, n.b->ev);
    if (rc) return rc;
    if (root) {
        CK(cudaMemcpyAsync(f.slotM + (size_t)n.tree * f.pitch, t->hd.M, sizeof(double) * (size_t)f.H0 * t->stride,
                           cudaMemcpyDeviceToDevice, s));
        CK(cudaMemcpyAsync(f.slot_vrow + (size_t)n.tree * f.H0, t->hd.vrow, sizeof(int) * (size_t)f.H0,
                           cudaMemcpyDeviceToDevice, s));
        CK(cudaMemcpyAsync(f.slot_vcol + (size_t)n.tree * f.W, t->hd.vcol, sizeof(int) * (size_t)f.W,
                           cudaMemcpyDeviceToDevice, s));
    }
    if (n.rhs) return read_column(t, 0, n.rhs, n.vrow);
    return JSLP_OK;
}

// Nodes nodes[idx[0..n)] in one k_node_batch<NODE_FOREST> launch (roots when `root`); those whose log shows a cycle
// or that hit the pivot or log cap go to redo.
static int forest_resident(Forest &f, const std::vector<ForestNode> &nodes, const int *idx, int n, bool root,
                           bool outputs, std::vector<int> &redo) {
    jslp_tab *t = f.t;
    const ResidentBufs &rb = t->rbufs;
    auto node = [&](int k) -> const ForestNode & { return nodes[idx[k]]; };
    std::vector<int> root_of((size_t)n);
    int maxc = 0;
    for (int k = 0; k < n; k++) {
        root_of[k] = node(k).tree;
        maxc = std::max(maxc, (int)node(k).b->cuts.size());
    }
    NodeBatchDev nb;
    size_t smem = 0;
    int rc = batch_fill(t, f.baseM, f.base_vrow, f.base_vcol, f.H0, t->saved.lastElementIndex, n, nb, &smem);
    if (rc) return rc;
    rc = branch_cuts(t, n, [&](int k) { return node(k).b; }, nb);
    if (rc) return rc;
    nb.Hcap = f.H0 + maxc;
    smem = node_smem_bytes(nb.Hcap, t->W, nullptr);
    nb.slot_M = f.slotM; nb.slot_vrow = f.slot_vrow; nb.slot_vcol = f.slot_vcol; nb.slot_pitch = f.pitch;
    if (root) { nb.col0 = f.col0(0); nb.row0 = f.row0(0); }
    // one device block: the slot of each CTA, then the final columns and labels when asked
    ScratchLayout L;
    const size_t b_root = L.take(sizeof(int) * (size_t)n), b_rhs = L.take(sizeof(double) * (size_t)n * nb.Hcap);
    const size_t b_vrow = L.take(sizeof(int) * (size_t)n * nb.Hcap);
    rc = batch_scratch(t, L.bytes);
    if (rc) return rc;
    char *base = (char *)t->d_scratch;
    CK(cudaMemcpyAsync(base + b_root, root_of.data(), sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, t->ctx->stream));
    nb.root_of = (const int *)(base + b_root);
    std::vector<double> rhs;
    std::vector<int32_t> vrow;
    if (outputs) {
        nb.out_rhs = (double *)(base + b_rhs); nb.out_vrow = (int *)(base + b_vrow);
        rhs.resize((size_t)n * nb.Hcap);
        vrow.resize((size_t)n * nb.Hcap);
    }
    rc = batch_launch<NODE_FOREST>(t, nb, n, smem, rhs.data(), vrow.data());
    if (rc) return rc;
    std::vector<int> hit;
    rc = batch_screen(t, n, [&](int k) { return f.check_cycles && !rb.h_out[k].r.overflow; }, hit);
    if (rc) return rc;
    for (int k = 0; k < n; k++) {
        const NodeResult &r = rb.h_out[k].r;
        if (r.overflow || hit[k] >= 0) { redo.push_back(idx[k]); continue; }
        node(k).b->ev = node_eval(r.status, r.eval_raw, r.p1 + r.p2, r.is_integral, r.branch_var, r.branch_value,
                                  t->precision);
        if (outputs) {
            const int Hn = f.H0 + (int)node(k).b->cuts.size();
            memcpy(node(k).rhs, rhs.data() + (size_t)k * nb.Hcap, sizeof(double) * (size_t)Hn);
            memcpy(node(k).vrow, vrow.data() + (size_t)k * nb.Hcap, sizeof(int32_t) * (size_t)Hn);
        }
    }
    return JSLP_OK;
}

// Evaluates the nodes of the current group, routed by batch_route on their height (slot rows plus cuts).  Counts the
// CTAs of each launch in *ctas.
static int forest_eval(Forest &f, const std::vector<ForestNode> &nodes, bool root, bool outputs, int64_t *ctas) {
    return batch_route(
        f.t, (int)nodes.size(), [&](int i) { return f.H0 + (int)nodes[i].b->cuts.size(); }, true,
        [&](const int *idx, int m, std::vector<int> &redo) {
            *ctas += m;
            return forest_resident(f, nodes, idx, m, root, outputs, redo);
        },
        [&](int i) { return forest_hbm(f, nodes[i], root); });
}

extern "C" int jslp_bnb_batch(jslp_tab *t, const double *col0, const double *row0, int n_scenarios,
                              const jslp_bnb_opts *opts, int row_stride, jslp_bnb_status *status, double *rhs,
                              int32_t *vrow, int32_t *height) {
    using namespace jslp_bnb;
    if (!t || !opts) return fail(JSLP_E_INVALID, "NULL argument");
    if (n_scenarios < 0 || (n_scenarios > 0 && (!col0 || !row0 || !status || !rhs || !vrow || !height)))
        return fail(JSLP_E_INVALID, "bnb_batch: bad scenario / output arguments");
    if (t->nOpt > 0) return fail(JSLP_E_UNSUPPORTED, "bnb_batch: optional objectives are not supported");
    if (opts->service != 0 || opts->keep_solutions || opts->timeout_ms > 0 || opts->n_ranks > 1 || t->use_mir)
        return fail(JSLP_E_UNSUPPORTED, "bnb_batch runs the default service only: no enhanced or incremental service, "
                                        "useMIRCuts, keep_solutions, timeout or ranks");
    const int H0 = t->H, W = t->W;
    if (row_stride < H0 + 2 * t->n_int)
        return fail(JSLP_E_INVALID, "bnb_batch: row_stride is below the height plus two cuts per integer variable");
    if (n_scenarios == 0) return JSLP_OK;
    jslp_ctx *ctx = t->ctx;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const CallerState caller(t);
    const Saved kept = t->saved;
    const int kept_iflag = t->isIntegralFlag, kept_iters = t->bncIterations, kept_nvars = t->nVars;
    std::vector<NodeLogEntry> kept_log = std::move(t->node_log);
    std::vector<jslp_tab::StoredSolution> kept_solutions = std::move(t->solutions);
    t->saved = Saved{};
    int rc = jslp_save(t);  // the snapshot the single-tableau path restores from, the base until a slot is loaded
    if (rc) {
        t->saved = kept; t->node_log = std::move(kept_log); t->solutions = std::move(kept_solutions);
        return rc;
    }

    const size_t pitch = (size_t)H0 * t->stride;
    // A base tableau beyond shared memory has no resident node at all: its scenarios run one after another through
    // jslp_branch_and_cut itself (K3 node slots included), each on the base with its column 0 and row 0 written over.
    const bool sequential = !resident_fits(t, H0);
    const int G = sequential ? 1 : (int)std::max<size_t>(1, std::min<size_t>(n_scenarios, FOREST_SLOT_BYTES /
                                                                                             (sizeof(double) * pitch)));
    Forest f{t, H0, W, G, opts->check_cycles, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, pitch,
             t->nVars, t->lastElementIndex};
    auto release = [&] {
        cudaFree(f.baseM); cudaFree(f.base_vrow); cudaFree(f.base_vcol);
        cudaFree(f.slotM); cudaFree(f.slot_vrow); cudaFree(f.slot_vcol); cudaFree(f.d_edges);
    };
    auto run = [&]() -> int {
        CK(cudaMalloc(&f.baseM, sizeof(double) * pitch));
        CK(cudaMalloc(&f.base_vrow, sizeof(int) * (size_t)H0));
        CK(cudaMalloc(&f.base_vcol, sizeof(int) * (size_t)W));
        CK(cudaMemcpyAsync(f.baseM, t->saved.M, sizeof(double) * pitch, cudaMemcpyDeviceToDevice, s));
        CK(cudaMemcpyAsync(f.base_vrow, t->saved.vrow, sizeof(int) * (size_t)H0, cudaMemcpyDeviceToDevice, s));
        CK(cudaMemcpyAsync(f.base_vcol, t->saved.vcol, sizeof(int) * (size_t)W, cudaMemcpyDeviceToDevice, s));
        CK(cudaMalloc(&f.slotM, sizeof(double) * pitch * G));
        CK(cudaMalloc(&f.slot_vrow, sizeof(int) * (size_t)H0 * G));
        CK(cudaMalloc(&f.slot_vcol, sizeof(int) * (size_t)W * G));
        CK(cudaMalloc(&f.d_edges, sizeof(double) * (size_t)(H0 + W) * G));
        const int K = opts->max_spec_batch > 0 ? opts->max_spec_batch : 16;
        const Tree::Rule rule{opts->tolerance, opts->is_minimization, 0, opts->max_nodes};
        for (int k = 0; sequential && k < n_scenarios; k++) {
            f.G = 1;
            CK(cudaMemcpyAsync(f.d_edges, col0 + (size_t)k * H0, sizeof(double) * (size_t)H0, cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(f.d_edges + H0, row0 + (size_t)k * W, sizeof(double) * (size_t)W, cudaMemcpyHostToDevice, s));
            rc = f.load_saved(f.baseM, f.base_vrow, f.base_vcol);
            if (rc) return rc;
            rc = jslp_restore(t);
            if (rc) return rc;
            k_write_edges<<<(std::max(H0, W) + 255) / 256, 256, 0, s>>>(t->hd.M, t->stride, H0, W, f.col0(0), f.row0(0));
            ctx->launches += 1;
            CK(cudaGetLastError());
            // the scalar state of a freshly uploaded tableau, as Solve() starts from
            t->feasible = 1; t->bounded = 1; t->evaluation = 0; t->bestPossibleEval = 0; t->simplexIters = 0;
            t->isIntegralFlag = 0;
            jslp_bnb_status &o = status[k];
            memset(&o, 0, sizeof(o));
            if (t->n_int > 0) {
                jslp_bnb_opts one = *opts;
                rc = jslp_branch_and_cut(t, &one, &o, nullptr, 0);
                if (rc) return rc;
            } else {  // Solve() runs simplex() on a continuous LP
                jslp_lp_status st;
                rc = run_lp(t, 0, opts->check_cycles, &st, false);
                if (rc) return rc;
                o.feasible = t->feasible; o.bounded = t->bounded; o.evaluation = t->evaluation;
                o.best_possible_eval = t->bestPossibleEval; o.nodes_evaluated = 1; o.rounds = 1;
                o.pivots = st.phase1_pivots + st.phase2_pivots;
            }
            height[k] = t->H;
            rc = read_column(t, 0, rhs + (size_t)k * row_stride, vrow + (size_t)k * row_stride);
            if (rc) return rc;
        }
        for (int g0 = 0; !sequential && g0 < n_scenarios; g0 += G) {
            const int n = std::min(G, n_scenarios - g0);
            f.G = n;
            CK(cudaMemcpyAsync(f.d_edges, col0 + (size_t)g0 * H0, sizeof(double) * (size_t)n * H0, cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(f.d_edges + (size_t)n * H0, row0 + (size_t)g0 * W, sizeof(double) * (size_t)n * W,
                               cudaMemcpyHostToDevice, s));
            std::vector<Tree> trees((size_t)n);
            std::vector<int64_t> nodes((size_t)n, 0), rounds((size_t)n, 0), pruned((size_t)n, 0);
            std::vector<char> stop((size_t)n, 0);
            std::vector<int64_t> ctas((size_t)n, 0);
            int64_t launch_ctas = 0;
            auto out_rhs = [&](int k) { return rhs + (size_t)(g0 + k) * row_stride; };
            auto out_vrow = [&](int k) { return vrow + (size_t)(g0 + k) * row_stride; };
            // the root round: every tree's root in one set of launches; its final column 0 and labels are the
            // answer of a tree that ends without a final re-solve
            std::vector<ForestNode> batch;
            for (int k = 0; k < n; k++) {
                trees[k].branches.h[0].b->ev = NodeEval();
                batch.push_back(ForestNode{k, trees[k].branches.h[0].b.get(), out_rhs(k), out_vrow(k)});
                height[g0 + k] = H0;
            }
            rc = forest_eval(f, batch, true, true, &launch_ctas);
            if (rc) return rc;
            for (int k = 0; k < n; k++) { nodes[k] = 1; rounds[k] = 1; }
            if (t->n_int <= 0) {  // a continuous LP: Solve() runs simplex() on the tableau, which is the root
                for (int k = 0; k < n; k++) {
                    const NodeEval &ev = batch[k].b->ev;
                    jslp_bnb_status &o = status[g0 + k];
                    memset(&o, 0, sizeof(o));
                    o.feasible = ev.feasible; o.bounded = ev.bounded;
                    o.evaluation = ev.feasible ? ev.evaluation : 0.0;
                    o.best_possible_eval = ev.optimal ? ev.evaluation : 0.0;
                    o.nodes_evaluated = 1; o.pivots = ev.pivots; o.rounds = 1;
                }
                continue;
            }
            for (;;) {
                // commit every tree in its own pop order
                for (int k = 0; k < n; k++) {
                    Tree &tr = trees[k];
                    while (!stop[k]) {
                        const Tree::Step st = tr.step(rule, [] { return false; });
                        if (st == Tree::DONE) stop[k] = 1;
                        if (st == Tree::DONE || st == Tree::ROUND) break;
                        if (st == Tree::LIMIT || st == Tree::EARLY) { stop[k] = 1; break; }
                    }
                }
                // speculate: the next K un-evaluated open nodes of every live tree in pop order
                batch.clear();
                std::vector<std::vector<Frontier::Entry>> taken((size_t)n);
                std::vector<Branch *> todo;
                for (int k = 0; k < n; k++) {
                    if (stop[k]) continue;
                    trees[k].speculate(K, taken[k], todo, pruned[k]);
                    for (Branch *b : todo) batch.push_back(ForestNode{k, b, nullptr, nullptr});
                    if (!todo.empty()) { rounds[k]++; nodes[k] += (int64_t)todo.size(); }
                }
                if (batch.empty()) break;
                rc = forest_eval(f, batch, false, false, &launch_ctas);
                if (rc) return rc;
                for (int k = 0; k < n; k++) trees[k].put_back(taken[k]);
            }
            // the final tableau: the reference re-solves the winner, or the last evaluated node (branch-and-cut.ts:195-197)
            batch.clear();
            std::vector<NodeEval> keep((size_t)n);
            std::vector<std::unique_ptr<Branch>> fins((size_t)n);
            for (int k = 0; k < n; k++) {
                const Branch *fin = trees[k].final_branch();
                if (!fin) continue;
                fins[k].reset(new Branch{fin->relaxedEvaluation, fin->cuts, NodeEval()});
                batch.push_back(ForestNode{k, fins[k].get(), out_rhs(k), out_vrow(k)});
                height[g0 + k] = H0 + (int)fin->cuts.size();
                nodes[k]++;
            }
            rc = forest_eval(f, batch, false, true, &launch_ctas);
            if (rc) return rc;
            for (int k = 0; k < n; k++) {
                Tree &tr = trees[k];
                if (fins[k]) {  // what run_lp leaves in the Tableau flags after the re-solve
                    const NodeEval &ev = fins[k]->ev;
                    if (tr.bestBranch) {
                        tr.pivots += ev.pivots;
                        if (ev.optimal) tr.simplexIters += 1;
                    }
                    tr.feasible = ev.feasible; tr.bounded = ev.bounded;
                    if (ev.feasible) tr.evaluation = ev.evaluation;
                }
                jslp_bnb_status &o = status[g0 + k];
                memset(&o, 0, sizeof(o));
                o.feasible = tr.feasible; o.bounded = tr.bounded; o.is_integral = tr.isIntegral;
                o.iterations = tr.iterations;
                o.n_best_cuts = tr.bestBranch && !tr.early_return ? (int)tr.bestBranch->cuts.size() : 0;
                o.rounds = (int)rounds[k]; o.nodes_evaluated = nodes[k]; o.pivots = tr.pivots;
                o.evaluation = tr.evaluation; o.best_possible_eval = tr.bestPossibleEval;
                o.nodes_pruned = pruned[k];
            }
        }
        return JSLP_OK;
    };
    const int64_t launches0 = ctx->launches;
    rc = run();
    if (rc == JSLP_OK && n_scenarios > 0) status[0].kernel_launches = ctx->launches - launches0;
    // the tab as it was: its tableau from the base copy, its snapshot, scalar state, node log and stored solutions
    int rc2 = f.baseM ? f.load_saved(f.baseM, f.base_vrow, f.base_vcol) : JSLP_OK;
    if (rc2 == JSLP_OK) rc2 = jslp_restore(t);
    cudaStreamSynchronize(s);
    release();
    free_saved(t->saved);
    t->saved = kept;
    caller.restore(t);
    t->isIntegralFlag = kept_iflag; t->bncIterations = kept_iters; t->nVars = kept_nvars;
    t->node_log = std::move(kept_log);
    t->solutions = std::move(kept_solutions);
    return rc ? rc : rc2;
}
