// jslpsolver_b200/csrc/jslp_frontier.h -- host-only data structures of the branch-and-cut frontier
// (included by jslp_bnb.cuh; also compiled on its own by tests/test_host_cpu.py with g++).
//
// Frontier replaces BranchMinHeap (min-heap.ts:18-119): best-first on relaxedEvaluation, most recently
// pushed first on ties (min-heap.ts:43-49).  Branch / NodeEval replace Branch / BranchCut (types.ts:17-26)
// plus the cached result of a speculative evaluation; to_wire / from_wire are the 128-byte record the
// ranks all-gather per node.
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <utility>
#include <vector>

namespace jslp_bnb {

struct NodeEval {  // what the commit loop needs from one node LP
    bool valid = false;
    int feasible = 0, bounded = 1, optimal = 0, is_integral = 0, branch_var = -1, pivots = 0;
    double evaluation = 0, branch_value = 0;
    // useMIRCuts only (never on the wire: such models are not sharded): simplex() calls of this node that ended
    // optimal (Tableau.simplexIters) and the evaluation of the first one (Tableau.bestPossibleEval at the root)
    int n_optimal = -1;  // -1 = one solve: use `optimal`
    double first_eval = 0;
    double opt0[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // optionalObjectives[o].reducedCosts[0]
};

struct Branch {
    double relaxedEvaluation;
    std::vector<jslp_cut> cuts;
    NodeEval ev;  // cached speculative result
};

// Total order of min-heap.ts:43-49: lower relaxedEvaluation first, then higher seq (LIFO).
struct Frontier {
    struct Entry {
        std::unique_ptr<Branch> b;
        long seq;
    };
    std::vector<Entry> h;
    long seqCounter = 0;
    static bool before(const Entry &a, const Entry &b) {
        if (a.b->relaxedEvaluation != b.b->relaxedEvaluation) return a.b->relaxedEvaluation < b.b->relaxedEvaluation;
        return a.seq > b.seq;
    }
    bool empty() const { return h.empty(); }
    void push_entry(Entry e) {
        h.push_back(std::move(e));
        size_t i = h.size() - 1;
        while (i > 0) {
            const size_t p = (i - 1) / 2;
            if (!before(h[i], h[p])) break;
            std::swap(h[i], h[p]);
            i = p;
        }
    }
    void push(std::unique_ptr<Branch> br) { push_entry(Entry{std::move(br), seqCounter++}); }
    Entry pop_entry() {
        Entry top = std::move(h[0]);
        if (h.size() > 1) h[0] = std::move(h.back());
        h.pop_back();
        size_t i = 0;
        const size_t n = h.size();
        for (;;) {
            size_t l = 2 * i + 1, r = l + 1, m = i;
            if (l < n && before(h[l], h[m])) m = l;
            if (r < n && before(h[r], h[m])) m = r;
            if (m == i) break;
            std::swap(h[i], h[m]);
            i = m;
        }
        return top;
    }
};

// One committed node of the trace jslp_bnb_node_log reads: iteration, nCuts, feasible, evaluation, integral (-1/0/1),
// branchVar, branchValue, pivots.
struct NodeLogEntry {
    double v[8];
};

// One tree of the default branch-and-cut service (branch-and-cut.ts:54-199): its frontier, its incumbent and the
// Tableau scalars the reference's loop reads and writes.  step() is one pass of that loop's body (:76-192) over a node
// whose LP result is cached in Branch::ev; speculate() picks the nodes of a round and final_branch() the node re-solved
// at the end.  jslp_branch_and_cut and jslp_bnb_batch both run their trees through it.
struct Tree {
    Frontier branches;
    int iterations = 0;
    bool toleranceFlag = true, early_return = false;
    double bestEvaluation = INFINITY;
    std::unique_ptr<Branch> bestBranch, lastCommitted;
    std::vector<double> bestOpt;
    // Tableau.feasible / bounded / evaluation / bestPossibleEval / simplexIters / __isIntegral
    int feasible = 1, bounded = 1, simplexIters = 0, isIntegral = 0;
    double evaluation = 0, bestPossibleEval = 0;
    std::vector<NodeLogEntry> node_log;
    int64_t pivots = 0;  // pivots of the committed nodes

    struct Rule {
        double tolerance;
        int is_minimization, nOpt;
        int64_t max_nodes;  // 0 = none
    };
    enum Step {
        DONE,       // the loop condition fails: the frontier is empty or the tolerance was reached
        ROUND,      // the next node to pop has no cached result: evaluate another round first
        LIMIT,      // max_nodes nodes are committed
        TIMED_OUT,  // time_up() said so before the pop
        EARLY,      // the root was integral: the reference returns at once (:134-137)
        NEXT,       // a node was popped (and committed unless the incumbent skips it)
        SNAPSHOT,   // the root was committed fractional: the caller snapshots the tableau now (:155-157)
        INCUMBENT,  // a new incumbent: lastCommitted is it (keep_solutions stores it here, :143-153)
    };

    explicit Tree(int nOpt = 0) : bestOpt((size_t)nOpt, INFINITY) {
        branches.push(std::unique_ptr<Branch>(new Branch{-INFINITY, {}, NodeEval()}));
    }

    template <typename TimeUp>
    Step step(const Rule &r, TimeUp time_up) {
        if (branches.empty() || !toleranceFlag) return DONE;
        if (r.max_nodes > 0 && iterations >= r.max_nodes) return LIMIT;
        if (time_up()) return TIMED_OUT;
        const double acceptableThreshold = r.is_minimization ? bestPossibleEval * (1 + r.tolerance)
                                                             : bestPossibleEval * (1 - r.tolerance);
        // the reference checks the tolerance BEFORE popping, and still processes that pop
        const bool tolHit = r.tolerance > 0 && bestEvaluation < acceptableThreshold;
        if (branches.h[0].b->relaxedEvaluation <= bestEvaluation && !branches.h[0].b->ev.valid) return ROUND;
        if (tolHit) toleranceFlag = false;
        Frontier::Entry e = branches.pop_entry();
        if (e.b->relaxedEvaluation > bestEvaluation) return NEXT;
        pivots += e.b->ev.pivots;
        return commit(std::move(e.b), r.nOpt);
    }

    // The nodes of a round: pops open nodes in the order step() will, into taken, until todo holds width nodes
    // without a cached result or the scan has popped 4 * width + 32 entries.  Returns the round's incumbent bound U,
    // bestEvaluation lowered by every cached integral result on the way.  A node above U is counted in pruned and
    // never evaluated: it sorts after the node that set U, so by the time step() pops it bestEvaluation <= U <
    // relaxedEvaluation and it is skipped (branch-and-cut.ts:90-92).  The scan is bounded because once the
    // un-evaluated nodes thin out it would otherwise walk the whole heap every round; candidates that far down are not
    // popped before the next round anyway.
    double speculate(int width, std::vector<Frontier::Entry> &taken, std::vector<Branch *> &todo, int64_t &pruned) {
        taken.clear();
        todo.clear();
        double U = bestEvaluation;
        const size_t scan_cap = (size_t)width * 4 + 32;
        while (!branches.empty() && (int)todo.size() < width && taken.size() < scan_cap) {
            Frontier::Entry e = branches.pop_entry();
            if (e.b->ev.valid) {
                if (e.b->ev.feasible && e.b->ev.is_integral && e.b->ev.evaluation < U) U = e.b->ev.evaluation;
            } else if (!(e.b->relaxedEvaluation > U)) {
                todo.push_back(e.b.get());
            } else {
                pruned++;
            }
            taken.push_back(std::move(e));
        }
        return U;
    }
    // The entries speculate() took back into the frontier, with their original sequence numbers: the pop order is as
    // it was.
    void put_back(std::vector<Frontier::Entry> &taken) {
        for (Frontier::Entry &e : taken) branches.push_entry(std::move(e));
        taken.clear();
    }

    // A known integral plan as the incumbent (MIP starts, DESIGN.md section 2t): it is not a node of the loop, so it
    // counts no iteration and writes no node-log entry.
    void seed(std::vector<jslp_cut> cuts, double eval) {
        bestEvaluation = eval;
        isIntegral = 1;
        bestBranch.reset(new Branch{eval, std::move(cuts), NodeEval()});
    }

    // The two children of a fractional node (branch-and-cut.ts:166-188): a cut on the branching variable goes to low
    // when it is a `min` cut and to high when it is a `max` cut, every other cut to both, then each child's new cut.
    static void children(const Branch &b, int varIndex, double value, double relaxed, std::unique_ptr<Branch> &high,
                         std::unique_ptr<Branch> &low) {
        high.reset(new Branch{relaxed, {}, NodeEval()});
        low.reset(new Branch{relaxed, {}, NodeEval()});
        for (const jslp_cut &cut : b.cuts) {
            if (cut.var_index == varIndex) {
                if (cut.type == 0) low->cuts.push_back(cut); else high->cuts.push_back(cut);
            } else {
                high->cuts.push_back(cut);
                low->cuts.push_back(cut);
            }
        }
        high->cuts.push_back(jslp_cut{0, varIndex, std::ceil(value)});
        low->cuts.push_back(jslp_cut{1, varIndex, std::floor(value)});
    }

    // The node the reference re-solves once the loop ends (branch-and-cut.ts:195-197): the incumbent, else the last
    // committed node when more than one was committed; null after the early return at an integral root.
    const Branch *final_branch() const {
        if (early_return) return nullptr;
        if (bestBranch) return bestBranch.get();
        return iterations > 1 ? lastCommitted.get() : nullptr;
    }

  private:
    Step commit(std::unique_ptr<Branch> active, int nOpt) {
        const NodeEval ev = active->ev;
        iterations++;
        feasible = ev.feasible; bounded = ev.bounded;
        // Tableau.evaluation is what the node's last optimal (or unbounded) solve set; an infeasible node keeps the
        // previous value, except under useMIRCuts when a solve before the infeasible one was optimal
        if (ev.feasible || ev.optimal) evaluation = ev.evaluation;
        if (ev.optimal) {  // setEvaluation + simplexIters (tableau.ts:420-430, simplex.ts:266-267)
            if (simplexIters == 0) bestPossibleEval = ev.n_optimal >= 0 ? ev.first_eval : ev.evaluation;
            simplexIters += ev.n_optimal >= 0 ? ev.n_optimal : 1;
        }
        NodeLogEntry nl;
        nl.v[0] = iterations; nl.v[1] = (double)active->cuts.size(); nl.v[2] = ev.feasible;
        nl.v[3] = evaluation; nl.v[4] = -1; nl.v[5] = -1; nl.v[6] = 0; nl.v[7] = ev.pivots;
        auto done = [&](std::unique_ptr<Branch> keep) {
            node_log.push_back(nl);
            lastCommitted = std::move(keep);
        };
        if (!ev.feasible) { done(std::move(active)); return NEXT; }
        const double value = ev.evaluation;
        if (value > bestEvaluation) { done(std::move(active)); return NEXT; }
        if (value == bestEvaluation) {  // branch-and-cut.ts:107-127
            bool worse = true;
            for (int o = 0; o < nOpt; o++) {
                if (ev.opt0[o] > bestOpt[o]) break;
                if (ev.opt0[o] < bestOpt[o]) { worse = false; break; }
            }
            if (worse) { done(std::move(active)); return NEXT; }
        }
        if (ev.is_integral) {
            nl.v[4] = 1;
            isIntegral = 1;
            if (iterations == 1) { node_log.push_back(nl); early_return = true; return EARLY; }
            bestEvaluation = value;
            for (int o = 0; o < nOpt; o++) bestOpt[o] = ev.opt0[o];
            node_log.push_back(nl);
            bestBranch.reset(new Branch{active->relaxedEvaluation, active->cuts, NodeEval()});
            lastCommitted = std::move(active);
            return INCUMBENT;
        }
        const int varIndex = ev.branch_var;
        nl.v[4] = 0; nl.v[5] = varIndex; nl.v[6] = ev.branch_value;
        std::unique_ptr<Branch> high, low;
        children(*active, varIndex, ev.branch_value, value, high, low);
        branches.push(std::move(high));
        branches.push(std::move(low));
        const bool root = iterations == 1;
        done(std::move(active));
        return root ? SNAPSHOT : NEXT;
    }
};

// The deal of a sharded round (n_ranks > 1): node i of the round, in pop order, is evaluated by rank i % n_ranks.
static inline int deal_rank(size_t i, int n_ranks) { return (int)(i % (size_t)n_ranks); }

// Where a sharded round's results meet: a rank-major buffer of n_ranks blocks of `per` records, per = ceil(n / n_ranks)
// for a round of n nodes.  Node i's record is the (i / n_ranks)-th of its rank's block; the last ranks' blocks end in
// unused records when n is not a multiple of n_ranks, and a rank with no node of the round sends only those.
struct WireDeal {
    int n_ranks, per;
    WireDeal(size_t n, int ranks) : n_ranks(ranks), per((int)((n + (size_t)ranks - 1) / (size_t)ranks)) {}
    size_t slot(size_t i) const { return (size_t)deal_rank(i, n_ranks) * per + i / (size_t)n_ranks; }
};

// The element-wise min of a round's all-reduce when it is carried by an all-gather: blocks holds n_ranks rank-major
// blocks of n doubles, v[k] becomes the smallest k-th entry over every rank's block.
static inline void fold_min(const double *blocks, int n_ranks, int n, double *v) {
    for (int r = 0; r < n_ranks; r++)
        for (int k = 0; k < n; k++) v[k] = r == 0 ? blocks[k] : std::min(v[k], blocks[(size_t)r * n + k]);
}

static const int WIRE_DOUBLES = 16;  // all-gather record per node (128 bytes)
static void to_wire(const NodeEval &e, double *w) {
    w[0] = e.valid; w[1] = e.feasible; w[2] = e.bounded; w[3] = e.optimal; w[4] = e.is_integral;
    w[5] = e.branch_var; w[6] = e.pivots; w[7] = e.evaluation;
    memcpy(&w[7], &e.evaluation, 8);
    memcpy(&w[8], &e.branch_value, 8);
    for (int o = 0; o < 7; o++) memcpy(&w[9 + o], &e.opt0[o], 8);
}
static void from_wire(NodeEval &e, const double *w) {
    e.valid = w[0] != 0; e.feasible = (int)w[1]; e.bounded = (int)w[2]; e.optimal = (int)w[3];
    e.is_integral = (int)w[4]; e.branch_var = (int)w[5]; e.pivots = (int)w[6];
    memcpy(&e.evaluation, &w[7], 8);
    memcpy(&e.branch_value, &w[8], 8);
    for (int o = 0; o < 7; o++) memcpy(&e.opt0[o], &w[9 + o], 8);
}

}  // namespace jslp_bnb
