// Drives N simulated ranks of a sharded branch and cut through the PRODUCT's round logic (jslpsolver_b200/csrc/
// jslp_frontier.h): each rank owns a jslp_bnb::Tree, takes its round with Tree::speculate, evaluates only the nodes
// deal_rank() gives it, writes their records with to_wire at WireDeal::slot() into its own block of a rank-major
// buffer, and reads every node of the round back with from_wire from the concatenated blocks (the all-gather) before
// Tree::step commits.  An owning rank's answer is the only one that reaches the other ranks.  Node results come from
// the C oracle over a line protocol, so tests/test_distributed_edges_cpu.py can compare every rank's node log with the
// oracle's sequential branch and cut.  Built with g++ by that test.
//   argv[1] == "selftest": checks the wire record, the deal helpers and fold_min on their own and prints SHARD SELFTEST OK.
//   stdin, first line:  tolerance is_minimization max_nodes width n_ranks n_opt      (n_opt <= 7, as the product asks)
//   stdout "EVAL n type var value ..." (the cuts of the node to evaluate), stdin: feasible bounded optimal is_integral
//   branch_var branch_value evaluation pivots opt0[0] .. opt0[n_opt - 1];  stdout "SAVE", stdin: any line;
//   at the end, for every rank r: "RANK r LOG n", n lines of the 8 node-log doubles, "ITER iterations best_cuts evals".
//   Exit codes: 6 the ranks' trees diverged, 7 a record fell outside its rank's block.
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "jslp_b200.h"
#include "jslp_frontier.h"

using namespace jslp_bnb;

#define CHECK(c) do { if (!(c)) { std::printf("FAILED line %d: %s\n", __LINE__, #c); std::exit(1); } } while (0)

static double from_bits(uint64_t u) { double d; std::memcpy(&d, &u, 8); return d; }
static bool same_bits(double a, double b) { return std::memcmp(&a, &b, 8) == 0; }

static void round_trip(const NodeEval &e) {
    double w[WIRE_DOUBLES];
    std::memset(w, 0, sizeof(w));
    to_wire(e, w);
    NodeEval r;
    r.opt0[7] = 42.5;  // not on the wire: from_wire must leave it alone
    r.n_optimal = 9; r.first_eval = 3.25;  // useMIRCuts only, never sharded
    from_wire(r, w);
    CHECK(r.valid == e.valid && r.feasible == e.feasible && r.bounded == e.bounded && r.optimal == e.optimal);
    CHECK(r.is_integral == e.is_integral && r.branch_var == e.branch_var && r.pivots == e.pivots);
    CHECK(same_bits(r.evaluation, e.evaluation) && same_bits(r.branch_value, e.branch_value));
    for (int o = 0; o < 7; o++) CHECK(same_bits(r.opt0[o], e.opt0[o]));
    CHECK(r.opt0[7] == 42.5 && r.n_optimal == 9 && r.first_eval == 3.25);
}

static int selftest() {
    const double specials[] = {0.0, -0.0, INFINITY, -INFINITY, 5e-324, -5e-324, from_bits(0x000fffffffffffffull),
                               from_bits(0x800123456789abcdull), from_bits(0x7ff8000000000123ull),
                               from_bits(0xfff8dead0000beefull), from_bits(0x7ff0000000000001ull),
                               from_bits(0xfff7ffffffffffffull), 2.5000000000000004, -1e308};
    const int n = (int)(sizeof(specials) / sizeof(specials[0]));
    const int ints[] = {-1, 0, 1, INT_MAX, INT_MAX - 1};
    for (int k = 0; k < n; k++) {
        NodeEval e;
        e.valid = k % 2 == 0; e.feasible = k % 3 != 0; e.bounded = k % 4 != 1; e.optimal = k % 5 == 2;
        e.is_integral = k % 2;
        e.branch_var = ints[k % 5]; e.pivots = ints[(k + 2) % 5] < 0 ? 0 : ints[(k + 2) % 5];
        e.evaluation = specials[k];
        e.branch_value = specials[(k + 5) % n];
        for (int o = 0; o < 8; o++) e.opt0[o] = specials[(k + 3 * o + 1) % n];
        round_trip(e);
    }
    {   // the record is 16 doubles: opt0[7] has no slot, which is why jslp_branch_and_cut refuses nOpt > 7 on ranks
        NodeEval e;
        for (int o = 0; o < 8; o++) e.opt0[o] = o + 0.5;
        double w[WIRE_DOUBLES + 1];
        w[WIRE_DOUBLES] = -7.0;
        to_wire(e, w);
        CHECK(w[WIRE_DOUBLES] == -7.0 && WIRE_DOUBLES == 16 && sizeof(double) * WIRE_DOUBLES == 128);
        for (int o = 0; o < 7; o++) CHECK(w[9 + o] == o + 0.5);
    }
    for (int ranks = 1; ranks <= 8; ranks++) {  // every node of a round gets its own record in its own rank's block
        for (size_t todo = 0; todo <= 40; todo++) {
            const WireDeal d(todo, ranks);
            CHECK((size_t)d.per * ranks >= todo && (size_t)d.per * ranks < todo + ranks);
            std::vector<int> used((size_t)d.per * ranks, 0), per_rank((size_t)ranks, 0);
            for (size_t i = 0; i < todo; i++) {
                const int r = deal_rank(i, ranks);
                CHECK(r == (int)(i % ranks));
                const size_t s = d.slot(i);
                CHECK(s >= (size_t)r * d.per && s < (size_t)(r + 1) * d.per);
                CHECK(s - (size_t)r * d.per == (size_t)per_rank[r]);  // a rank's records in pop order, from the block start
                CHECK(used[s]++ == 0);
                per_rank[r]++;
            }
            for (int r = 0; r < ranks; r++) CHECK(per_rank[r] == (int)(todo / ranks) + (r < (int)(todo % ranks)));
        }
    }
    for (int ranks = 1; ranks <= 8; ranks++) {  // the all-reduce(min) fold reads every rank's block and nothing past them
        for (int n = 1; n <= 3; n++) {
            for (int low = 0; low < ranks; low++) {  // the smallest value in each rank's block in turn
                std::vector<double> blocks((size_t)(ranks + 1) * n, -INFINITY);  // one block of -inf past the end
                for (int r = 0; r < ranks; r++)
                    for (int k = 0; k < n; k++) blocks[(size_t)r * n + k] = 10.0 * (r + 1) + k;
                for (int k = 0; k < n; k++) blocks[(size_t)low * n + k] = -1.0 - k;
                std::vector<double> v((size_t)n, 99.0);
                fold_min(blocks.data(), ranks, n, v.data());
                for (int k = 0; k < n; k++) CHECK(v[k] == -1.0 - k);
            }
        }
    }
    std::printf("SHARD SELFTEST OK\n");
    return 0;
}

int main(int argc, char **argv) {
    if (argc > 1 && std::strcmp(argv[1], "selftest") == 0) return selftest();
    double tol = 0;
    int is_min = 1, width = 1, N = 1, nOpt = 0;
    long long max_nodes = 0;
    if (std::scanf("%lf %d %lld %d %d %d", &tol, &is_min, &max_nodes, &width, &N, &nOpt) != 6 || width < 1 || N < 1 ||
        nOpt < 0 || nOpt > 7)
        return 2;
    const Tree::Rule rule{tol, is_min, nOpt, (int64_t)max_nodes};
    std::vector<Tree> trees;
    for (int r = 0; r < N; r++) trees.emplace_back(nOpt);
    std::vector<std::vector<Frontier::Entry>> taken((size_t)N);
    std::vector<std::vector<Branch *>> todo((size_t)N);
    std::vector<int64_t> evals((size_t)N, 0);
    int64_t pruned = 0;
    for (;;) {
        std::vector<Tree::Step> st;
        for (Tree &t : trees) st.push_back(t.step(rule, [] { return false; }));
        for (int r = 1; r < N; r++)
            if (st[r] != st[0] || trees[r].iterations != trees[0].iterations) return 6;
        if (st[0] == Tree::DONE || st[0] == Tree::LIMIT || st[0] == Tree::EARLY) break;
        if (st[0] == Tree::ROUND) {
            const bool root = trees[0].iterations == 0;
            const int nr = root ? 1 : N;  // the root round is not sharded: every rank solves it
            for (int r = 0; r < N; r++) {
                trees[r].speculate(root ? 1 : width, taken[r], todo[r], pruned);
                if (todo[r].size() != todo[0].size()) return 6;
            }
            const size_t n = todo[0].size();
            if (n == 0) return 5;  // step() asks for a round only when the next pop has no result
            const WireDeal deal(n, nr);
            std::vector<std::vector<double>> own((size_t)N, std::vector<double>((size_t)deal.per * nr * WIRE_DOUBLES, 0.0));
            for (size_t i = 0; i < n; i++) {
                const int owner = deal_rank(i, nr);
                Branch *b = todo[owner][i];
                std::printf("EVAL %d", (int)b->cuts.size());
                for (const jslp_cut &c : b->cuts) std::printf(" %d %d %.17g", c.type, c.var_index, c.value);
                std::printf("\n");
                std::fflush(stdout);
                NodeEval &ev = b->ev;
                if (std::scanf("%d %d %d %d %d %lf %lf %d", &ev.feasible, &ev.bounded, &ev.optimal, &ev.is_integral,
                               &ev.branch_var, &ev.branch_value, &ev.evaluation, &ev.pivots) != 8)
                    return 3;
                for (int o = 0; o < nOpt; o++)
                    if (std::scanf("%lf", &ev.opt0[o]) != 1) return 3;
                ev.valid = true;
                evals[owner]++;
                if (root) continue;
                const size_t s = deal.slot(i);
                if (s < (size_t)owner * deal.per || s >= (size_t)(owner + 1) * deal.per) return 7;
                to_wire(ev, &own[owner][s * WIRE_DOUBLES]);
            }
            if (root) {  // every rank holds the same root result
                for (int r = 1; r < N; r++) todo[r][0]->ev = todo[0][0]->ev;
            } else {
                std::vector<double> gathered((size_t)deal.per * nr * WIRE_DOUBLES);
                const size_t block = (size_t)deal.per * WIRE_DOUBLES;
                for (int r = 0; r < nr; r++)
                    std::memcpy(&gathered[r * block], &own[r][r * block], sizeof(double) * block);
                for (int r = 0; r < N; r++)
                    for (size_t i = 0; i < n; i++) from_wire(todo[r][i]->ev, &gathered[deal.slot(i) * WIRE_DOUBLES]);
            }
            for (int r = 0; r < N; r++) trees[r].put_back(taken[r]);
        } else if (st[0] == Tree::SNAPSHOT) {
            std::printf("SAVE\n");
            std::fflush(stdout);
            char line[16];
            if (std::scanf("%15s", line) != 1) return 4;
        }
    }
    for (int r = 0; r < N; r++) {
        const Tree &t = trees[r];
        std::printf("RANK %d LOG %d\n", r, (int)t.node_log.size());
        for (const NodeLogEntry &e : t.node_log) {
            for (int k = 0; k < 8; k++) std::printf(k ? " %.17g" : "%.17g", e.v[k]);
            std::printf("\n");
        }
        std::printf("ITER %d %d %lld\n", t.iterations, t.bestBranch && !t.early_return ? (int)t.bestBranch->cuts.size() : 0,
                    (long long)evals[r]);
    }
    return 0;
}
