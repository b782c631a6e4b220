// jslpsolver_b200/csrc/jslp_cycles.h -- host-only cycle detection over the drained pivot log
// (included by jslp_api.cu; also compiled on its own by tests/test_host_cpu.py with g++).
#pragma once

#include <unordered_map>
#include <vector>

// checkForCycles (simplex.ts:415-440) under its calling discipline (called after every push, stops at the first hit):
// a repeated block must end at the newest element, so only suffix squares are examined, and the literal scan reports
// the smallest start = the longest block.  A block of length L that repeats up to the newest element needs
// h[n-1-L] == h[n-1], so only earlier positions of the newest pair are candidate block ends (largest L first): each
// push costs O(occurrences of the newest pair) instead of O(n).
struct CycleHist {
    std::vector<long long> h;
    std::unordered_map<long long, std::vector<int>> pos;
    bool push_and_check(long long v, int *start, int *len) {
        h.push_back(v);
        const long n = (long)h.size();
        std::vector<int> &p = pos[v];
        bool hit = false;
        for (size_t k = 0; k < p.size() && !hit; k++) {
            const long L = (n - 1) - p[k];
            if (2 * L > n) continue;
            const long e1 = n - 2 * L, e2 = n - L;
            bool eq = true;
            for (long i = 0; i < L; i++)
                if (h[e1 + i] != h[e2 + i]) { eq = false; break; }
            if (eq) { *start = (int)e1; *len = (int)L; hit = true; }
        }
        p.push_back((int)(n - 1));
        return hit;
    }
};

// The index of the first entry of a node pivot log that closes a repeat, with one (leaving, entering) history per phase
// (simplex.ts:27,102), or -1.  An entry's .x carries the phase in bit 30, its .z / .w the pair.
template <typename Entry>
static int first_cycle(const Entry *lg, int n) {
    CycleHist h[2];
    int cs, cl;
    for (int k = 0; k < n; k++)
        if (h[(lg[k].x >> 30) & 1].push_and_check(((long long)lg[k].z << 32) | (unsigned int)lg[k].w, &cs, &cl))
            return k;
    return -1;
}
