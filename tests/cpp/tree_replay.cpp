// Drives the PRODUCT's speculation and commit rules (jslp_bnb::Tree in jslpsolver_b200/csrc/jslp_frontier.h) over a line
// protocol, so that tests/test_mip_scenarios_cpu.py can feed it node results computed by the C oracle and compare its
// node log with the oracle's own branch and cut.  Rounds are taken as jslp_branch_and_cut takes them: the root alone,
// then `width` nodes in pop order (Tree::speculate), each answered in order before the round commits.  Built with g++ by
// that test.
//   stdin, first line:  tolerance is_minimization max_nodes width
//   stdout "EVAL n type var value ..." (the cuts of the node to evaluate), stdin: feasible bounded optimal is_integral
//   branch_var branch_value evaluation pivots;  stdout "SAVE" (the root was committed fractional), stdin: any line;
//   at the end stdout "LOG n", n lines of the 8 node-log doubles, then "ITER iterations best_cuts".
#include <cstdio>
#include "jslp_b200.h"
#include "jslp_frontier.h"

using namespace jslp_bnb;

int main() {
    double tol = 0;
    int is_min = 1;
    long long max_nodes = 0;
    int width = 1;
    if (std::scanf("%lf %d %lld %d", &tol, &is_min, &max_nodes, &width) != 4 || width < 1) return 2;
    const Tree::Rule rule{tol, is_min, 0, (int64_t)max_nodes};
    Tree tree;
    std::vector<Frontier::Entry> taken;
    std::vector<Branch *> todo;
    int64_t pruned = 0;
    for (;;) {
        const Tree::Step st = tree.step(rule, [] { return false; });
        if (st == Tree::DONE || st == Tree::LIMIT || st == Tree::EARLY) break;
        if (st == Tree::ROUND) {
            tree.speculate(tree.iterations == 0 ? 1 : width, taken, todo, pruned);
            if (todo.empty()) return 5;  // step() asks for a round only when the next pop has no result
            for (Branch *b : todo) {
                std::printf("EVAL %d", (int)b->cuts.size());
                for (const jslp_cut &c : b->cuts) std::printf(" %d %d %.17g", c.type, c.var_index, c.value);
                std::printf("\n");
                std::fflush(stdout);
                NodeEval &ev = b->ev;
                if (std::scanf("%d %d %d %d %d %lf %lf %d", &ev.feasible, &ev.bounded, &ev.optimal, &ev.is_integral,
                               &ev.branch_var, &ev.branch_value, &ev.evaluation, &ev.pivots) != 8)
                    return 3;
                ev.valid = true;
            }
            tree.put_back(taken);
        } else if (st == Tree::SNAPSHOT) {
            std::printf("SAVE\n");
            std::fflush(stdout);
            char line[16];
            if (std::scanf("%15s", line) != 1) return 4;
        }
    }
    std::printf("LOG %d\n", (int)tree.node_log.size());
    for (const NodeLogEntry &e : tree.node_log) {
        for (int k = 0; k < 8; k++) std::printf(k ? " %.17g" : "%.17g", e.v[k]);
        std::printf("\n");
    }
    std::printf("ITER %d %d\n", tree.iterations, tree.bestBranch && !tree.early_return ? (int)tree.bestBranch->cuts.size() : 0);
    return 0;
}
