// The product's cycle detectors (jslpsolver_b200/csrc/jslp_cycles.h: the hashed CycleHist and the per-phase node-log
// screen first_cycle) against a literal restatement of the reference's checkForCycles (simplex.ts:415-440), under
// the reference's calling discipline: the detector runs after every push and the solve stops at the first hit
// (simplex.ts:27-36,102-112), with one history per phase (simplex.ts:27,102).  Built and run by tests/test_host_cpu.py
// with g++; prints CYCLES OK.
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "jslp_cycles.h"

// simplex.ts:415-440, pair (leaving, entering) packed into one 64-bit key
static bool literal(const std::vector<long long> &v, int *start, int *len) {
    const long n = (long)v.size();
    for (long e1 = 0; e1 < n - 1; e1++)
        for (long e2 = e1 + 1; e2 < n; e2++) {
            if (v[e1] != v[e2]) continue;
            if (e2 - e1 > n - e2) break;
            bool found = true;
            for (long i = 1; i < e2 - e1; i++)
                if (v[e1 + i] != v[e2 + i]) { found = false; break; }
            if (found) { *start = (int)e1; *len = (int)(e2 - e1); return true; }
        }
    return false;
}

// A node pivot-log entry as first_cycle reads it: the phase in bit 30 of x, the (leaving, entering) pair in z / w.
struct LogEntry {
    int x, y, z, w;
};

static unsigned long long rng_state = 88172645463325252ull;
static unsigned int rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return (unsigned int)(rng_state >> 11); }

// One random pivot history: a few distinct pairs, so that repeats are frequent; some histories fall into an exact
// cycle after a lead-in, and half of them never repeat the previous pair, so that their first hit is a block of
// length >= 2.
struct History {
    int alphabet, period, lead;
    bool periodic, no_stutter;
    std::vector<long long> h;
    History()
        : alphabet(2 + (int)(rnd() % 9)), period(1 + (int)(rnd() % 7)), lead((int)(rnd() % 12)),
          periodic((rnd() & 3) == 0), no_stutter((rnd() & 1) == 0) {}
    long long next() {
        const int k = (int)h.size();
        long long v;
        if (periodic && k >= lead) v = 1000 + ((k - lead) % period) * 7 + (long long)(((k - lead) % period) % 3) * (1ll << 32);
        else {
            do v = (long long)(rnd() % alphabet) | ((long long)(rnd() % 2) << 32);
            while (no_stutter && !h.empty() && v == h.back());
        }
        h.push_back(v);
        return v;
    }
};

int main() {
    long hits = 0, pushes = 0, long_hits = 0;
    for (int trial = 0; trial < 4000; trial++) {
        History hs;
        CycleHist hist;
        for (int k = 0; k < 200; k++) {
            const long long v = hs.next();
            pushes++;
            int s0 = -1, l0 = -1, s2 = -1, l2 = -1;
            const bool r0 = literal(hs.h, &s0, &l0);
            const bool r2 = hist.push_and_check(v, &s2, &l2);
            if (r0 != r2 || (r0 && (s0 != s2 || l0 != l2))) {
                std::printf("FAILED trial %d push %d: literal %d (%d,%d) hashed %d (%d,%d)\n", trial, k, r0, s0, l0, r2, s2,
                            l2);
                return 1;
            }
            if (r0) { hits++; if (l0 >= 3) long_hits++; break; }   // the reference returns at the first hit
        }
    }
    if (hits < 1000 || long_hits < 200) {
        std::printf("FAILED: %ld hits, %ld of length >= 3: the generator does not exercise the detectors\n", hits, long_hits);
        return 1;
    }
    // first_cycle over node logs that interleave two phase histories at random: the first entry at which the literal
    // scan of that entry's own phase history hits, or -1 when neither history repeats within the log
    long log_hits[2] = {0, 0};
    for (int trial = 0; trial < 4000; trial++) {
        History hs[2];
        std::vector<LogEntry> lg;
        int want = -1;
        const int n = 1 + (int)(rnd() % 120);
        for (int k = 0; k < n; k++) {
            const int ph = (int)(rnd() & 1);
            const long long v = hs[ph].next();
            lg.push_back(LogEntry{(int)(rnd() & 0x3fffffff) | (ph << 30), (int)rnd(), (int)(v >> 32), (int)(unsigned int)v});
            int s0, l0;
            if (want < 0 && literal(hs[ph].h, &s0, &l0)) { want = k; log_hits[ph]++; }
        }
        const int got = first_cycle(lg.data(), n);
        if (got != want) {
            std::printf("FAILED log trial %d (%d entries): first_cycle %d, literal per phase %d\n", trial, n, got, want);
            return 1;
        }
    }
    if (log_hits[0] < 500 || log_hits[1] < 500) {
        std::printf("FAILED: %ld / %ld first hits in phase 1 / 2: the logs do not exercise both histories\n", log_hits[0],
                    log_hits[1]);
        return 1;
    }
    std::printf("CYCLES OK (%ld hits, %ld of block length >= 3, %ld pushes; node logs: %ld / %ld first hits per phase)\n",
                hits, long_hits, pushes, log_hits[0], log_hits[1]);
    return 0;
}
