// jslpsolver_b200/csrc/jslp_kernels.cuh -- sm_90a kernels for the dense-tableau pivot path.
//
// What the reference does per simplex iteration (src/tableau/simplex.ts in JWally/jsLPSolver):
//   phase1 (25-98)   leaving row = arg-min RHS < -precision, entering column = arg-max -cost/coef
//   phase2 (100-325) entering column = arg-max reduced cost > precision inside the first 50-column
//                    batch that has one (partial pricing), ratio test with degenerate early exit
//   pivot  (330-413) normalise pivot row, rank-1 update of every other row incl. the cost row
// All of it is "strict compare, lowest index wins" on IEEE fp64 with separate multiply and
// subtract roundings (JS has no FMA), so every reduction here is on (value,index) pairs and the
// update uses __dmul_rn/__dsub_rn.
//
// Kernels:
//   k_select      one CTA decides the next pivot from the tableau in HBM/L2 and stages the raw
//                 pivot row / pivot column into side buffers (also used for Tableau.pivot()).
//   k_pivot_step  multi-CTA fused step: TMA-stages the raw pivot row into shared memory,
//                 normalises it there, streams its row block with 128-bit loads/stores doing the
//                 rank-1 update; the last CTA to finish (atomic ticket) runs the selection for the
//                 NEXT pivot, so one launch == one simplex iteration and a CUDA graph of N launches
//                 needs no host round trip.  Memory-bound (0.125 flop/B): no tensor cores.
#pragma once
#include <cstddef>
#include <cuda_runtime.h>
#include <stdint.h>
#include <limits.h>
#include <math.h>

namespace jslp {

enum { ST_RUNNING = 0, ST_OPTIMAL = 1, ST_INFEASIBLE = 2, ST_UNBOUNDED = 3, ST_P1_DONE = 4, ST_ERROR = 5 };

struct Part;

// Device-resident description of one tableau (kernels read it through a pointer so that a
// captured CUDA graph stays valid when H grows or buffers are re-allocated).
struct TabDev {
    double *M;             // rowcap x stride, row-major; row 0 = cost row, col 0 = RHS
    int *vrow;             // varIndexByRow [rowcap]
    int *vcol;             // varIndexByCol [W]
    unsigned char *unres;  // unrestrictedVars by var index [n_index] or nullptr
    double *opt;           // optional objective reducedCosts [nOpt x stride]
    double *prow;          // staged raw pivot row [stride]
    double *pcol;          // staged raw pivot column [rowcap]
    double *optcoef;       // staged optional-objective pivot-column entries [nOpt]
    int4 *plog;            // per-batch pivot log (row, col, leaving var, entering var)
    unsigned char *optflag; // scratch [W] for the optional-objective tie-break lists
    int *intpos;           // position in model.integerVariables by var index, -1 otherwise [n_index]
    double *M2;            // ping-pong partner of M (same shape): the fused ping-pong step reads M, writes
                           // M2 and swaps the two pointers in this descriptor
    Part *part;            // per-CTA look-ahead ratio-test partials [grid]
    long long *dbg;        // optional per-CTA timeline (8 x int64 per CTA per launch) or nullptr
    int W, H, stride, rowcap;
    int nOpt, n_index, plog_cap;
    int batch_size, use_partial;  // phase-2 partial pricing (simplex.ts:118-127)
    int dbg_cap, dbg_grid;
    double prec;
};

// Look-ahead partial of one CTA: ratio test (simplex.ts:271-296) over its own freshly updated rows
// against the NEXT entering column, so the last CTA only has to reduce gridDim.x of these.
struct __align__(16) Part {
    double minq;        // smallest admissible quotient among this CTA's rows (INF = none)
    double pad0;        // keeps the four ints below on a 16-byte boundary (read as one int4)
    int minr;           // row of minq (INT_MAX = none)
    int dmin;           // first degenerate row (INT_MAX = none)
    int cnt;            // rows with a non-zero pivot-column entry (for the lazy flush flag)
    int pad;
};

// Pivot record: the decision carried from one launch to the next.  One 128-byte line (arrays of records,
// one per node slot, keep the 16-byte loads of k_pivot_step aligned).
struct __align__(128) Rec {
    int status;      // ST_*
    int phase;       // 1 or 2
    int has_pivot;   // (r, c) is selected and staged but not executed yet
    int r, c;
    int is_neg;      // isReducedCostNegative (simplex.ts:138)
    int flush;       // some row other than r has a non-zero pivot-column entry (simplex.ts:380)
    int done;        // pivots executed in this call
    int p1, p2;      // per-phase pivot counts (return values of phase1()/phase2())
    int stop_at;     // execute at most this many pivots (-1 = no limit); used for cycle rewind
    int log_n;       // entries in plog for the current batch
    int unbounded_var;
    int only_phase;  // 0 = simplex(), 1 = phase1() only, 2 = phase2() only
    unsigned int ticket;
    int pad0;
    int lookahead;   // host switch: 1 = the tail also prices the pivot after next
    int next_c;      // entering column of the NEXT pivot, priced on the cost row as it will be after
                     // the staged pivot: -1 unknown (generic tail), 0 none (optimal), >0 column
    int next_neg;    // its isReducedCostNegative
    int prow_norm;   // 1 = the prow side buffer already holds the NORMALISED pivot row (staged by the
                     // ping-pong selector), 0 = the raw row (every CTA normalises it after the TMA copy)
    int pad1;
    double q;        // raw pivot element
    double eval_raw; // matrix[0] at exit
};

// k_pivot_step reads the record with 16-byte loads
static_assert(offsetof(Rec, c) == 16 && offsetof(Rec, p1) == 32 && offsetof(Rec, unbounded_var) == 48 && offsetof(Rec, lookahead) == 64 &&
              offsetof(Rec, q) == 88, "Rec layout");

struct MipOut {
    int is_integral;
    int var_index;
    double value;
};

// One cut of addCutConstraints (cutting-strategies.ts:36-71): type 0 = "min", 1 = "max".
struct CutDev {
    int type, var_index;
    double value;
};

__device__ __forceinline__ bool nz16(double v) { return !(v >= -1e-16 && v <= 1e-16); }

// IEEE fp64 division.  Inline in the step kernels (a call costs more than the expansion on their
// latency-critical paths); the resident node kernel uses the out-of-line ddiv_z below.
__device__ __forceinline__ double ddiv(double a, double b) { return a / b; }

// One shared copy with a fast path for zero dividends: the compiler's expansion sends 0 / b to its slow
// path (several times the cost of a regular division) and degenerate node tableaux are full of zeros;
// 0 / b = 0 signed (a xor b) for every b that is neither 0 nor NaN.
__device__ __noinline__ double ddiv_z(double a, double b) {
    if (a == 0.0 && b == b && b != 0.0)
        return __longlong_as_double((__double_as_longlong(a) ^ __double_as_longlong(b)) & (long long)0x8000000000000000ull);
    return a / b;
}

// Tableau loads bypass L1: other CTAs may just have rewritten the entry in L2.
__device__ __forceinline__ double ldg_cg(const double *p) { return __ldcg(p); }

// JS Math.round: nearest, ties toward +inf
__device__ __forceinline__ double js_round(double x) {
    if (!(x == x) || isinf(x)) return x;
    const double f = floor(x);
    return (x - f >= 0.5) ? f + 1.0 : f;
}

struct VI {
    double v;
    int i;
};

template <bool IS_MIN>
__device__ __forceinline__ bool better(const VI &b, const VI &a) {
    if (IS_MIN) return b.v < a.v || (b.v == a.v && b.i < a.i);
    return b.v > a.v || (b.v == a.v && b.i < a.i);
}

// ---- element rules of the simplex (simplex.ts), each written once for every kernel ---------------------------
// Values in, values out: the callers issue every load of a pass first and then apply these, so a selector pass stays
// one L2 round trip.  DIV = the fp64 division: the inline ddiv in the step kernels, ddiv_z in k_node_batch.
using DivFn = double (*)(double, double);

// Normalised pivot-row entry from its raw value v (simplex.ts:352-364): v / q where |v| > 1e-16, 1 / q in the pivot
// column, 0 elsewhere.  With `flush` (a row other than the pivot row is updated, simplex.ts:380-382) a quotient that is
// itself within 1e-16 of zero is stored as 0.
template <DivFn DIV = ddiv>
__device__ __forceinline__ double norm_entry(double v, bool is_pc, double q, bool flush) {
    double f = (is_pc || nz16(v)) ? DIV(is_pc ? 1.0 : v, q) : 0.0;
    if (flush && !nz16(f) && f != 0.0) f = 0.0;
    return f;
}

// Entry of a row with a non-zero pivot-column entry coef after the pivot (simplex.ts:376-386): -coef / q in the pivot
// column, old - coef * f (two roundings) where the normalised pivot-row entry f is non-zero, old elsewhere.
template <DivFn DIV = ddiv>
__device__ __forceinline__ double upd_entry(double old, double coef, double f, bool is_pc, double q) {
    if (is_pc) return DIV(-coef, q);
    return nz16(f) ? __dsub_rn(old, __dmul_rn(coef, f)) : old;
}

// Entry (r, c) of the tableau as the pivot (rstar, cstar, q) leaves it, from its old value (simplex.ts:352-391):
// is_prow = r is the pivot row, coef = the row's old pivot-column entry, f = the normalised pivot-row entry of column c.
// A row with |coef| <= 1e-16 is untouched, its pivot-column entry included (:389-391 repeats :371's test: dead code).
template <DivFn DIV = ddiv>
__device__ __forceinline__ double new_entry(double old, bool is_prow, double coef, double f, bool is_pc, double q) {
    if (is_prow) return f;
    return nz16(coef) ? upd_entry<DIV>(old, coef, f, is_pc, q) : old;
}

// Cost-row entry after the staged pivot (cstar, q) from the RAW pivot-row entry v: new_entry on norm_entry(v), and v
// is divided only where the cost row changes (coef0 = the cost row's pivot-column entry).  The flush is left out: an f
// within 1e-16 of zero leaves the entry alone either way.
template <DivFn DIV = ddiv>
__device__ __forceinline__ double priced_cost(double cost, double v, double coef0, bool is_pc, double q) {
    const double f = (nz16(coef0) && !is_pc) ? norm_entry<DIV>(v, false, q, false) : 0.0;
    return new_entry<DIV>(cost, false, coef0, f, is_pc, q);
}

// Lazy-flush flag of a pivot (simplex.ts:380): cnt = rows with a non-zero pivot-column entry, the pivot row included.
__device__ __forceinline__ bool flush_flag(int cnt, double q) { return cnt - (nz16(q) ? 1 : 0) > 0; }

// One row of the ratio test (simplex.ts:271-296); col / rhs = the row's entries in the entering column and column 0.
// Rows with |col| >= prec take part: a degenerate one (col > 0, |rhs| < prec) lowers dmin, and the lowest such row
// wins outright, as the reference's early exit does; any other offers its quotient to best (lowest row on ties when
// rows come in increasing order).  cnt counts the non-zero entries of the column, row 0 included (flush_flag).
template <DivFn DIV = ddiv>
__device__ __forceinline__ void ratio_step(int r, double col, double rhs, bool is_neg, double prec, int &dmin, VI &best,
                                           int &cnt) {
    if (nz16(col)) cnt++;
    if (r == 0 || (-prec < col && col < prec)) return;
    if (col > 0 && prec > rhs && rhs > -prec) { dmin = min(dmin, r); return; }
    const double quo = DIV(is_neg ? -rhs : rhs, col);  // (-rhs) / col == -rhs / col
    if (quo > prec && best.v > quo) { best.v = quo; best.i = r; }
}

// One candidate i of the parametric min-quotient tests (DESIGN.md section 2d): the primal step bound -M[r,0] / D[r]
// (num = -M[r,0], den = D[r]), the dual ratio test M[0,c] / M[r*,c], and the cost step bound -M[0,c] / E[c] (num =
// M[0,c], den = -E[c]; negating the divisor instead of the dividend gives the same IEEE quotient).  A restricted
// candidate takes part when den < -prec, an unrestricted one offers 0 when |den| > prec; a quotient below 0 or -0
// counts as +0 and a NaN quotient takes no part.  Lowest i on ties when candidates come in increasing order.
template <DivFn DIV = ddiv>
__device__ __forceinline__ void param_ratio(int i, double num, double den, bool unres, double prec, VI &best) {
    double q;
    if (unres) {
        if (!(fabs(den) > prec)) return;
        q = 0.0;
    } else {
        if (!(den < -prec)) return;
        q = DIV(num, den);
        if (!(q > 0.0) && q == q) q = 0.0;
    }
    if (q < best.v) { best.v = q; best.i = i; }
}

// One row of the warm-start crash (DESIGN.md section 2f): a row whose basic label the saved basis gives up (`leave`)
// takes part when its entry v in the entering column passes putInBase's test v < -prec || prec < v (a NaN never does),
// and the largest |v| wins (lowest row on ties when rows come in increasing order).  |v| of a candidate is positive and
// finite or +inf, so the double itself is an order-preserving key for block_reduce_vi.
__device__ __forceinline__ void crash_step(int r, double v, bool leave, double prec, VI &best) {
    if (!leave || !(v < -prec || prec < v)) return;
    const double key = fabs(v);
    if (key > best.v) { best.v = key; best.i = r; }
}

// The dynamic-modification edits (dynamic-modification.ts:78-160), each one entry: x - d * y and x + d * y (difference
// times entry, then subtract / add: two roundings), and x - d.  updateRightHandSide and updateCost are built from these
// three, on the HBM tableau (jslp_dynamic.cuh) and in the scenario prologue of k_node_batch alike.
__device__ __forceinline__ double edit_axpy_sub(double x, double d, double y) { return __dsub_rn(x, __dmul_rn(d, y)); }
__device__ __forceinline__ double edit_axpy_add(double x, double d, double y) { return __dadd_rn(x, __dmul_rn(d, y)); }
__device__ __forceinline__ double edit_sub(double x, double d) { return __dsub_rn(x, d); }

// One column of the phase-1 entering-column scan (simplex.ts:56-76): the column qualifies when its variable is
// unrestricted or coef (the leaving row's entry) < -prec, and the largest -cost / coef wins (lowest column on ties when
// columns come in increasing order).  cost() yields the cost-row entry; it runs for qualifying columns only.
template <DivFn DIV = ddiv, class Cost>
__device__ __forceinline__ void entering_step(int c, double coef, bool unres, double prec, VI &e, Cost cost) {
    if (unres || coef < -prec) {
        const double quo = DIV(-cost(), coef);
        if (e.v < quo) { e.v = quo; e.i = c; }
    }
}

// Pivot (r, c) on thread 0 (simplex.ts:339-349): pivot-log entry and label swap; the inverse maps are rebuilt on
// read-back.  leaving / entering = the labels of row r and column c before the swap.
__device__ __forceinline__ void log_pivot(int4 *plog, int log_n, int cap, int *vrow, int *vcol, int phase, int r, int c,
                                          int leaving, int entering) {
    if (log_n < cap) plog[log_n] = make_int4(r | (phase == 2 ? (1 << 30) : 0), c, leaving, entering);
    vrow[r] = entering;
    vcol[c] = leaving;
}

// Stages pivot (r, c) on thread 0: log_pivot plus the record fields every staging site writes.
__device__ __forceinline__ void stage_pivot(const TabDev &T, Rec *rec, int log_n, int phase, int r, int c, int leaving,
                                            int entering, double q, int isneg, bool flush, int next_c, int prow_norm) {
    log_pivot(T.plog, log_n, T.plog_cap, T.vrow, T.vcol, phase, r, c, leaving, entering);
    rec->log_n = log_n + 1;
    rec->phase = phase; rec->r = r; rec->c = c; rec->q = q; rec->is_neg = isneg; rec->flush = flush;
    rec->has_pivot = 1;
    rec->next_c = next_c;        // -1: the pivot after this one has not been priced
    rec->prow_norm = prow_norm;  // 1: the prow side buffer holds the row already normalised
}

// Cut rows (addCutConstraints, cutting-strategies.ts:36-71).  cut_lookup: the row where the cut's variable is basic
// (rows 1 .. H0-1) and its column, -1 where absent, searched from position 1 + first in steps of `step`; the caller
// merges the threads' answers (a label occurs once).
__device__ __forceinline__ void cut_lookup(const int *vrow, int H0, const int *vcol, int W, int var, int first, int step,
                                           int &row, int &col) {
    row = col = -1;
    for (int r = 1 + first; r < H0; r += step) if (vrow[r] == var) row = r;
    for (int c = 1 + first; c < W; c += step) if (vcol[c] == var) col = c;
}
// Entry c of the cut row; vr = the row where the variable is basic, nullptr when it is non-basic (in column col, -1
// when basic) or when c lies in the row padding past W (the entry is then 0).
__device__ __forceinline__ double cut_entry(const CutDev &cut, int c, int col, const double *vr) {
    const double sign = cut.type == 0 ? -1.0 : 1.0;
    if (vr == nullptr) return c == 0 ? sign * cut.value : (c == col ? sign : 0.0);
    return c == 0 ? sign * (cut.value - vr[0]) : -sign * vr[c];
}

struct RedSmem {
    double v[32];
    int i[32];
    int a[32];
    int b[32];
};

// (value,index) arg-min / arg-max over the CTA, lowest index wins ties; result on every thread.
template <bool IS_MIN>
__device__ __forceinline__ VI block_reduce_vi(VI x, const VI init, RedSmem &s) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        VI y;
        y.v = __shfl_xor_sync(0xffffffffu, x.v, o);
        y.i = __shfl_xor_sync(0xffffffffu, x.i, o);
        if (better<IS_MIN>(y, x)) x = y;
    }
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (l == 0) { s.v[w] = x.v; s.i[w] = x.i; }
    __syncthreads();
    if (l < nw) { x.v = s.v[l]; x.i = s.i[l]; } else { x = init; }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        VI y;
        y.v = __shfl_xor_sync(0xffffffffu, x.v, o);
        y.i = __shfl_xor_sync(0xffffffffu, x.i, o);
        if (better<IS_MIN>(y, x)) x = y;
    }
    return x;
}

// op: 0 = min, 1 = sum
template <int OP>
__device__ __forceinline__ int block_reduce_int(int x, RedSmem &s) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const int y = __shfl_xor_sync(0xffffffffu, x, o);
        x = OP == 0 ? min(x, y) : x + y;
    }
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (l == 0) s.i[w] = x;
    __syncthreads();
    x = (l < nw) ? s.i[l] : (OP == 0 ? INT_MAX : 0);
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const int y = __shfl_xor_sync(0xffffffffu, x, o);
        x = OP == 0 ? min(x, y) : x + y;
    }
    return x;
}

__device__ __forceinline__ unsigned long long dkey(double v) {  // order-preserving for non-NaN, -0 == +0
    const unsigned long long b = (unsigned long long)__double_as_longlong(v + 0.0);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double dkey_inv(unsigned long long k) {
    const unsigned long long b = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
    return __longlong_as_double((long long)b);
}

// (value, index) arg-min / arg-max over the warp, lowest index on ties; x.v must not be NaN.
template <bool IS_MIN>
__device__ __forceinline__ VI warp_reduce_vi(VI x) {
    const unsigned long long k = dkey(x.v);
    const unsigned int hi = (unsigned int)(k >> 32), lo = (unsigned int)k;
    unsigned int mhi, mlo;
    if (IS_MIN) {
        mhi = __reduce_min_sync(0xffffffffu, hi);
        mlo = __reduce_min_sync(0xffffffffu, hi == mhi ? lo : 0xffffffffu);
    } else {
        mhi = __reduce_max_sync(0xffffffffu, hi);
        mlo = __reduce_max_sync(0xffffffffu, hi == mhi ? lo : 0u);
    }
    VI r;
    r.i = __reduce_min_sync(0xffffffffu, (hi == mhi && lo == mlo) ? x.i : INT_MAX);
    r.v = dkey_inv(((unsigned long long)mhi << 32) | mlo);
    return r;
}


// ---- CTA-wide reductions built on redux.sync (a third of the latency of the shuffle trees above; used on
// the selectors' critical path).  Results on every thread; one trailing barrier protects s for reuse.
template <bool IS_MIN>
__device__ __forceinline__ VI block_reduce_vi_rx(VI x, const VI init, RedSmem &s) {
    x = warp_reduce_vi<IS_MIN>(x);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    if (l == 0) { s.v[w] = x.v; s.i[w] = x.i; }
    __syncthreads();
    VI y = init;
    if (l < nw) { y.v = s.v[l]; y.i = s.i[l]; }
    y = warp_reduce_vi<IS_MIN>(y);
    __syncthreads();
    return y;
}

// Ratio-test reduction: min first-degenerate row, (quotient,row) arg-min with lowest-row ties, count of
// non-zero pivot-column entries, and an all-ok flag (min).
__device__ __forceinline__ void block_reduce_ratio_rx(int &dmin, VI &m, int &cnt, int &ok, RedSmem &s) {
    m = warp_reduce_vi<true>(m);
    dmin = __reduce_min_sync(0xffffffffu, dmin);
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    ok = __reduce_min_sync(0xffffffffu, ok);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    if (l == 0) { s.v[w] = m.v; s.i[w] = m.i; s.a[w] = dmin; s.b[w] = cnt | (ok ? 0 : (1 << 30)); }
    __syncthreads();
    VI y = {INFINITY, INT_MAX};
    int d = INT_MAX, n = 0, bad = 0;
    if (l < nw) { y.v = s.v[l]; y.i = s.i[l]; d = s.a[l]; n = s.b[l] & ~(1 << 30); bad = (s.b[l] >> 30) & 1; }
    m = warp_reduce_vi<true>(y);
    dmin = __reduce_min_sync(0xffffffffu, d);
    cnt = __reduce_add_sync(0xffffffffu, n);
    ok = __reduce_max_sync(0xffffffffu, bad) ? 0 : 1;
    __syncthreads();
}

__device__ __forceinline__ bool is_unres(const TabDev &T, int varIndex) {
    return T.unres != nullptr && varIndex >= 0 && varIndex < T.n_index && T.unres[varIndex] != 0;
}

// Ratio-test reduction in one pass (two barriers instead of six): min first-degenerate row,
// (quotient,row) arg-min with lowest-row ties, count of non-zero pivot-column entries.
__device__ __forceinline__ void block_reduce_ratio(int &dmin, VI &m, int &cnt, RedSmem &s) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        VI y;
        y.v = __shfl_xor_sync(0xffffffffu, m.v, o);
        y.i = __shfl_xor_sync(0xffffffffu, m.i, o);
        if (better<true>(y, m)) m = y;
        dmin = min(dmin, __shfl_xor_sync(0xffffffffu, dmin, o));
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (l == 0) { s.v[w] = m.v; s.i[w] = m.i; s.a[w] = dmin; s.b[w] = cnt; }
    __syncthreads();
    if (l < nw) { m.v = s.v[l]; m.i = s.i[l]; dmin = s.a[l]; cnt = s.b[l]; }
    else { m.v = INFINITY; m.i = INT_MAX; dmin = INT_MAX; cnt = 0; }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        VI y;
        y.v = __shfl_xor_sync(0xffffffffu, m.v, o);
        y.i = __shfl_xor_sync(0xffffffffu, m.i, o);
        if (better<true>(y, m)) m = y;
        dmin = min(dmin, __shfl_xor_sync(0xffffffffu, dmin, o));
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
}

// Copies the raw row `src` (W entries) into the stride-long side buffer `dst` (zero padded) with
// all loads of a pass issued before its stores: the two may alias as far as the compiler knows,
// and a load/store/load chain would cost one L2 round trip per element.
__device__ __forceinline__ void cta_copy_row(double *dst, const double *src, int W, int stride) {
    const int tid = threadIdx.x, NT = blockDim.x;
    for (int c0 = 0; c0 < stride; c0 += 8 * NT) {
        double v[8];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = c0 + tid + k * NT;
            v[k] = c < W ? ldg_cg(src + c) : 0.0;
        }
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = c0 + tid + k * NT;
            if (c < stride) dst[c] = v[k];
        }
    }
}

struct SelSmem {
    RedSmem red;
    int bc_col, bc_neg;
    double bq, bc0;
};

// Phase-2 pricing (simplex.ts:140-219, no optional objectives) in ONE pass over the cost row: the
// reference scans 50-column batches left to right and stops at the first batch with an improving
// column, taking the arg-max inside it; equivalently: lowest batch index that holds a candidate,
// then (value, column) arg-max with lowest-column ties inside that batch.  PRICED = price the cost
// row as the staged pivot (rowsrc, q, coef0, cstar) WILL leave it (look-ahead); new_label = label of
// column cstar after that pivot's swap; costsrc = the cost row to price (row 0 of the tableau, or a
// scratch copy).  Result on every thread; *found = 0 when nothing prices in.
// Per-thread pricing state: lowest batch index that holds a candidate of this thread's columns, and
// the best (value, column) inside that batch.  Columns must be fed in increasing order.
struct PriceAcc {
    int myb, myneg;
    VI x;
};
__device__ __forceinline__ void price_init(PriceAcc &a, double prec) {
    a.myb = INT_MAX; a.myneg = 0; a.x.v = prec; a.x.i = INT_MAX;
}
// nc = (updated) reduced cost of column c, label = variable labelling it (only read for unrestricted models)
__device__ __forceinline__ void price_consider(const TabDev &T, PriceAcc &a, int c, double nc, int label, int bsz) {
    bool un = false;
    if (T.unres != nullptr && nc < 0) un = is_unres(T, label);
    const double v2 = un ? -nc : nc;
    if (v2 > T.prec) {
        const int b = (c - 1) / bsz;
        if (b < a.myb) { a.myb = b; a.x.v = v2; a.x.i = c; a.myneg = un ? 1 : 0; }
        else if (b == a.myb && v2 > a.x.v) { a.x.v = v2; a.x.i = c; a.myneg = un ? 1 : 0; }
    }
}
// CTA-wide result: first batch with a candidate, arg-max inside it, lowest column on ties.
__device__ __forceinline__ void price_finish(const TabDev &T, SelSmem &s, const PriceAcc &a, int *found_out, int *neg_out) {
    const VI init = {T.prec, INT_MAX};
    const int bstar = block_reduce_int<0>(a.myb, s.red);
    int found = 0;
    if (bstar != INT_MAX) {
        const int mine = (a.myb == bstar) ? a.x.i : INT_MAX;
        VI y = (a.myb == bstar) ? a.x : init;
        y = block_reduce_vi<false>(y, init, s.red);
        found = y.i;
        if (mine == y.i) s.bc_neg = a.myneg;  // exactly one thread owns the winning column
    }
    __syncthreads();
    *found_out = found;
    *neg_out = found > 0 ? s.bc_neg : 0;
    __syncthreads();
}

// price_finish on redux.sync: one lexicographic reduction (batch asc, value desc, column asc).
__device__ __forceinline__ void price_finish_rx(const TabDev &T, SelSmem &s, const PriceAcc &a, int *found_out, int *neg_out) {
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    int b = a.myb, col = a.x.i, neg = a.myneg;
    double v = a.x.v;
#pragma unroll
    for (int stage = 0; stage < 2; stage++) {
        const int mb = __reduce_min_sync(0xffffffffu, b);
        const bool in = b == mb && mb != INT_MAX;
        const unsigned long long k = dkey(v);
        const unsigned int hi = (unsigned int)(k >> 32), lo = (unsigned int)k;
        const unsigned int mhi = __reduce_max_sync(0xffffffffu, in ? hi : 0u);
        const unsigned int mlo = __reduce_max_sync(0xffffffffu, (in && hi == mhi) ? lo : 0u);
        const bool win = in && hi == mhi && lo == mlo;
        const int mc = __reduce_min_sync(0xffffffffu, win ? col : INT_MAX);
        const int mn = __reduce_max_sync(0xffffffffu, (win && col == mc) ? neg : 0);
        b = mb; col = mc; neg = mn; v = dkey_inv(((unsigned long long)mhi << 32) | mlo);
        if (stage == 0) {
            if (l == 0) { s.red.i[w] = b; s.red.v[w] = v; s.red.a[w] = col; s.red.b[w] = neg; }
            __syncthreads();
            if (l < nw) { b = s.red.i[l]; v = s.red.v[l]; col = s.red.a[l]; neg = s.red.b[l]; }
            else { b = INT_MAX; v = T.prec; col = INT_MAX; neg = 0; }
        }
    }
    *found_out = b == INT_MAX ? 0 : col;
    *neg_out = b == INT_MAX ? 0 : neg;
    __syncthreads();
}

template <bool PRICED>
__device__ __noinline__ void cta_price_scan(const TabDev &T, SelSmem &s, const double *costsrc, const double *rowsrc, double q,
                               double coef0, int cstar, int new_label, int *found_out, int *neg_out) {
    const int tid = threadIdx.x, NT = blockDim.x;
    const int W = T.W;
    const int bsz = T.use_partial ? T.batch_size : max(1, W - 1);
    const bool has_unres = T.unres != nullptr;
    PriceAcc acc;
    price_init(acc, T.prec);
    // all loads of a pass are issued before any data-dependent branch: one L2 round trip per 8*NT columns
    for (int c0 = 1; c0 < W; c0 += 8 * NT) {
        double cv[8], rv[8];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = c0 + tid + k * NT;
            cv[k] = c < W ? ldg_cg(costsrc + c) : 0.0;
            rv[k] = (PRICED && c < W) ? ldg_cg(rowsrc + c) : 0.0;
        }
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = c0 + tid + k * NT;
            if (c >= W) continue;
            double nc = cv[k];
            if (PRICED) nc = priced_cost(nc, rv[k], coef0, c == cstar, q);
            int label = -1;
            if (has_unres && nc < 0) label = (PRICED && c == cstar) ? new_label : T.vcol[c];
            price_consider(T, acc, c, nc, label, bsz);
        }
    }
    price_finish(T, s, acc, found_out, neg_out);
}

// Literal, single-thread restatement of the pricing loop with optional objectives
// (simplex.ts:132-263).  Only models with constraint weight/priority have them (tiny fixtures),
// so the rare path trades speed for an exact transcription of the list semantics.
__device__ __noinline__ void price_with_optional_seq(const TabDev &T, int *outCol, int *outNeg) {
    const double prec = T.prec;
    const double *cost = T.M;
    const int lastColumn = T.W - 1;
    int enteringColumn = 0, isNeg = 0;
    double enteringValue = prec;
    unsigned char *flag = T.optflag;  // 1 = column is on the tie-break list
    for (int c = 0; c < T.W; c++) flag[c] = 0;
    int listed = 0;
    auto price = [&](int c, double rc) {
        if (is_unres(T, T.vcol[c]) && rc < 0) {
            if (-rc > enteringValue) { enteringValue = -rc; enteringColumn = c; isNeg = 1; }
            return;
        }
        if (rc > enteringValue) { enteringValue = rc; enteringColumn = c; isNeg = 0; }
    };
    if (T.use_partial) {
        const int nColumns = lastColumn;
        const int totalBatches = (nColumns + T.batch_size - 1) / T.batch_size;
        int batchStart = 1, scanned = 0;
        while (enteringColumn == 0 && scanned < totalBatches) {
            int batchEnd = batchStart + T.batch_size - 1;
            if (batchEnd > lastColumn) batchEnd = lastColumn;
            for (int c = batchStart; c <= batchEnd; c++) {
                const double rc = ldg_cg(cost + c);
                if (-prec < rc && rc < prec) { flag[c] = 1; listed++; continue; }
                price(c, rc);
            }
            batchStart = batchEnd >= lastColumn ? 1 : batchEnd + 1;
            scanned++;
        }
    } else {
        for (int c = 1; c <= lastColumn; c++) {
            const double rc = ldg_cg(cost + c);
            if (-prec < rc && rc < prec) { flag[c] = 1; listed++; continue; }
            price(c, rc);
        }
    }
    int o = 0;
    while (enteringColumn == 0 && listed > 0 && o < T.nOpt) {
        const double *rcs = T.opt + (size_t)o * T.stride;
        enteringValue = prec;
        int kept = 0;
        for (int c = 1; c <= lastColumn; c++) {
            if (!flag[c]) continue;
            const double rc = ldg_cg(rcs + c);
            if (-prec < rc && rc < prec) { kept++; continue; }
            flag[c] = 0;
            price(c, rc);
        }
        listed = kept;
        o++;
    }
    *outCol = enteringColumn;
    *outNeg = isNeg;
}

// Stage pivot (rstar, cstar): raw pivot row -> prow, optional pivot-column entries, label swap,
// pivot log, record.  `cnt` = number of rows r (incl. row 0 and rstar) with a non-zero
// pivot-column entry; pcol must already be staged.
__device__ void cta_stage_pivot(const TabDev &T, Rec *rec, int phase, int rstar, int cstar,
                                int isneg, int cnt) {
    const int tid = threadIdx.x, NT = blockDim.x;
    const double *prowsrc = T.M + (size_t)rstar * T.stride;
    const double q = ldg_cg(prowsrc + cstar);
    int leaving = 0, entering = 0;
    if (tid == 0) {  // only the thread that swaps the labels may read them (no barrier in between)
        leaving = T.vrow[rstar];
        entering = T.vcol[cstar];
    }
    cta_copy_row(T.prow, prowsrc, T.W, T.stride);
    for (int o = tid; o < T.nOpt; o += NT) T.optcoef[o] = ldg_cg(T.opt + (size_t)o * T.stride + cstar);
    if (tid == 0) stage_pivot(T, rec, rec->log_n, phase, rstar, cstar, leaving, entering, q, isneg, flush_flag(cnt, q), -1, 0);
}

// One CTA decides the next pivot from the tableau as it stands in L2/HBM (phase1: simplex.ts:
// 38-76, phase2: 129-303) and stages it.  All tableau reads bypass L1 (__ldcg): in the fused
// kernel this runs after other CTAs have just rewritten the tableau.
__device__ __noinline__ void cta_select(const TabDev &T, Rec *rec, SelSmem &s) {
    const int tid = threadIdx.x, NT = blockDim.x;
    const int W = T.W, H = T.H;
    const size_t stride = (size_t)T.stride;
    const double prec = T.prec;
    const double *M = T.M;
    int phase = rec->phase;
    const int only_phase = rec->only_phase;
    int rstar = -1, cstar = -1, isneg = 0, cnt = 0;
    bool col_staged = false;

    if (phase == 1) {
        const VI init = {-prec, INT_MAX};
        VI b = init;
        for (int rbase = 1; rbase < H; rbase += 8 * NT) {
            double rv[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rbase + tid + k * NT;
                rv[k] = r < H ? ldg_cg(M + r * stride) : 0.0;
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rbase + tid + k * NT;
                if (r < H && rv[k] < b.v) { b.v = rv[k]; b.i = r; }
            }
        }
        b = block_reduce_vi<true>(b, init, s.red);
        if (b.i == INT_MAX) {  // feasible (simplex.ts:51-54)
            if (only_phase == 1) {
                if (tid == 0) { rec->status = ST_P1_DONE; rec->has_pivot = 0; rec->eval_raw = ldg_cg(M); }
                return;
            }
            phase = 2;
        } else {
            rstar = b.i;
            const VI einit = {-INFINITY, INT_MAX};
            VI e = einit;
            const double *lrow = M + rstar * stride;
            const bool has_unres = T.unres != nullptr;
            for (int c0 = 1; c0 < W; c0 += 8 * NT) {  // loads of a pass first, then the tests
                double kv[8], cv[8];
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    const int c = c0 + tid + k * NT;
                    kv[k] = c < W ? ldg_cg(lrow + c) : 0.0;
                    cv[k] = c < W ? ldg_cg(M + c) : 0.0;
                }
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    const int c = c0 + tid + k * NT;
                    if (c < W) entering_step(c, kv[k], has_unres && is_unres(T, T.vcol[c]), prec, e, [&] { return cv[k]; });
                }
            }
            e = block_reduce_vi<false>(e, einit, s.red);
            if (e.i == INT_MAX) {  // simplex.ts:73-76
                if (tid == 0) { rec->status = ST_INFEASIBLE; rec->has_pivot = 0; rec->eval_raw = ldg_cg(M); }
                return;
            }
            cstar = e.i;
        }
    }

    if (rstar < 0) {  // phase 2
        if (T.nOpt == 0) {
            int found, neg;
            cta_price_scan<false>(T, s, T.M, nullptr, 1.0, 0.0, -1, -1, &found, &neg);
            if (found > 0) { cstar = found; isneg = neg; }
        } else {
            if (tid == 0) {
                int c0, n0;
                price_with_optional_seq(T, &c0, &n0);
                s.bc_col = c0;
                s.bc_neg = n0;
            }
            __syncthreads();
            cstar = s.bc_col > 0 ? s.bc_col : -1;
            isneg = s.bc_neg;
            __syncthreads();
        }
        if (cstar < 0) {  // optimal (simplex.ts:265-269); setEvaluation rounding is done on the host
            if (tid == 0) { rec->status = ST_OPTIMAL; rec->phase = 2; rec->has_pivot = 0; rec->eval_raw = ldg_cg(M); }
            return;
        }
        // ratio test (simplex.ts:271-296) fused with staging of the pivot column
        const VI init = {INFINITY, INT_MAX};
        VI m = init;
        int dmin = INT_MAX;
        for (int rbase = 0; rbase < H; rbase += 8 * NT) {  // loads of a pass first, then the tests
            double cv[8], rv[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rbase + tid + k * NT;
                cv[k] = r < H ? ldg_cg(M + r * stride + cstar) : 0.0;
                rv[k] = r < H ? ldg_cg(M + r * stride) : 0.0;
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rbase + tid + k * NT;
                if (r >= H) continue;
                T.pcol[r] = cv[k];
                ratio_step(r, cv[k], rv[k], isneg, prec, dmin, m, cnt);
            }
        }
        block_reduce_ratio(dmin, m, cnt, s.red);
        col_staged = true;
        if (dmin != INT_MAX) rstar = dmin;
        else if (m.i != INT_MAX) rstar = m.i;
        else {  // unbounded (simplex.ts:298-303)
            if (tid == 0) {
                rec->status = ST_UNBOUNDED; rec->phase = 2; rec->has_pivot = 0;
                rec->unbounded_var = T.vcol[cstar];
                rec->eval_raw = ldg_cg(M);
            }
            return;
        }
    }

    if (!col_staged) {
        cnt = 0;
        for (int rbase = 0; rbase < H; rbase += 8 * NT) {  // gather the pivot column: loads, then stores
            double cv[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rbase + tid + k * NT;
                cv[k] = r < H ? ldg_cg(M + r * stride + cstar) : 0.0;
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rbase + tid + k * NT;
                if (r < H) { T.pcol[r] = cv[k]; if (nz16(cv[k])) cnt++; }
            }
        }
        cnt = block_reduce_int<1>(cnt, s.red);
    }
    cta_stage_pivot(T, rec, phase, rstar, cstar, isneg, cnt);
}

__device__ __noinline__ void cta_price_next(const TabDev &T, Rec *rec, SelSmem &s);

// Standalone selection (engine 1, the first pivot of every solve, and Tableau.pivot()).
// force_r/force_c >= 0: stage exactly that pivot (== Tableau.pivot(r, c)).
__global__ void __launch_bounds__(512) k_select(const TabDev *Tp, Rec *rec, int force_r, int force_c) {
    __shared__ SelSmem s;
    __shared__ TabDev T;
    Tp += blockIdx.x;   // one CTA per tableau: node slots launch a row of them (jslp_slots.cuh)
    rec += blockIdx.x;
    if (threadIdx.x == 0) T = *Tp;
    __syncthreads();
    if (force_r >= 0) {
        int cnt = 0;
        for (int r = threadIdx.x; r < T.H; r += blockDim.x) {
            const double col = ldg_cg(T.M + (size_t)r * T.stride + force_c);
            T.pcol[r] = col;
            if (nz16(col)) cnt++;
        }
        cnt = block_reduce_int<1>(cnt, s.red);
        cta_stage_pivot(T, rec, rec->phase, force_r, force_c, 0, cnt);
        return;
    }
    if (rec->status != ST_RUNNING || rec->has_pivot) return;
    if (rec->stop_at >= 0 && rec->done >= rec->stop_at) return;
    cta_select(T, rec, s);
    __syncthreads();
    if (rec->lookahead && rec->has_pivot && rec->phase == 2 && T.nOpt == 0) cta_price_next(T, rec, s);
}

// ---- TMA (1-D bulk copy) + mbarrier helpers: raw pivot row HBM/L2 -> shared memory ----------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

__device__ __forceinline__ double2 ld_v2(const double *p) {
    double2 v;
    asm volatile("ld.global.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p));
    return v;
}
// Load of a tableau entry that is DEAD after this read: the ping-pong step reads buffer M once per launch and never
// again (the next launch reads what this one writes to M2), so these lines should be the first to leave L2.  With
// L1::no_allocate loads (SASS LDG.E.NA) and plain stores L2 keeps the WRITTEN buffer instead of both
// (scripts/micro/copybw.cu compares the load/store flavours by footprint).
__device__ __forceinline__ double2 ld_v2_dead(const double *p) {
    double2 v;
    asm volatile("ld.global.L1::no_allocate.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p));
    return v;
}
__device__ __forceinline__ void st_v2(double *p, double2 v) {
    asm volatile("st.global.v2.f64 [%0], {%1, %2};" ::"l"(p), "d"(v.x), "d"(v.y) : "memory");
}

#include "jslp_step.cuh"

// Start of every enqueued batch: empty the per-batch pivot log.
__global__ void k_batch_begin(Rec *rec) {
    if (threadIdx.x == 0) rec->log_n = 0;
}

// addCutConstraints (cutting-strategies.ts:36-71): one CTA per cut row, expressed in the
// current basis.  Cut h becomes row H0 + h with slack index first_index + h.
__global__ void __launch_bounds__(256) k_add_cuts(const TabDev *Tp, const CutDev *cuts, int H0, int first_index) {
    __shared__ int s_row, s_col;
    const TabDev &T = *Tp;
    const int h = blockIdx.x, tid = threadIdx.x, NT = blockDim.x;
    const CutDev cut = cuts[h];
    if (tid == 0) { s_row = -1; s_col = -1; }
    __syncthreads();
    int row, col;
    cut_lookup(T.vrow, H0, T.vcol, T.W, cut.var_index, tid, NT, row, col);
    if (row >= 0) s_row = row;
    if (col >= 0) s_col = col;
    __syncthreads();
    const double *vr = s_row < 0 ? nullptr : T.M + (size_t)s_row * T.stride;
    double *cutrow = T.M + (size_t)(H0 + h) * T.stride;
    for (int c = tid; c < T.stride; c += NT) cutrow[c] = cut_entry(cut, c, s_col, c < T.W ? vr : nullptr);
    if (tid == 0) T.vrow[H0 + h] = first_index + h;
}

// Math.max(0, x) / Math.min(0, y) with JS semantics (NaN propagates; max(0, -0) = +0; min(0, -0) = -0)
__device__ __forceinline__ double js_max0(double x) { return x != x ? x : (x > 0 ? x : 0.0); }
__device__ __forceinline__ double js_min0(double y) { return y != y ? y : (y < 0 ? y : ((y == 0 && signbit(y)) ? y : 0.0)); }

// addLowerBoundMIRCut / addUpperBoundMIRCut / applyMIRCuts (cutting-strategies.ts:74-212), one CTA.
// row >= 0: try exactly that row (upper = 0 / 1); row < 0: applyMIRCuts -- rows 1 .. H0-1 in ascending order,
// lower-bound cut on each row whose basic variable is integer with a fractional right-hand side, at most
// max_cuts.  Cut k becomes row H0 + k with slack index first_index + k; *n_added = number of rows appended.
__global__ void __launch_bounds__(256) k_mir_cuts(const TabDev *Tp, int H0, int first_index, int row, int upper, int max_cuts,
                                                  int *n_added) {
    __shared__ int s_flag[256];
    __shared__ int s_rows[16];
    __shared__ int s_n;
    const TabDev &T = *Tp;
    const int tid = threadIdx.x, NT = blockDim.x;
    const size_t stride = (size_t)T.stride;
    const double prec = T.prec;
    auto is_int = [&](int v) { return T.intpos != nullptr && v >= 0 && v < T.n_index && T.intpos[v] >= 0; };
    auto eligible = [&](int r) {
        if (r <= 0 || r >= H0) return false;                       // costRowIndex / out of range
        if (!is_int(T.vrow[r])) return false;                      // integerVar undefined or not integer
        const double rhs = T.M[r * stride];
        const double frac = rhs - floor(rhs);
        return !(frac < prec || frac > 1 - prec);
    };
    if (tid == 0) s_n = 0;
    __syncthreads();
    if (row >= 0) {
        if (tid == 0 && eligible(row)) { s_rows[0] = row; s_n = 1; }
        __syncthreads();
    } else {
        if (max_cuts > 16) max_cuts = 16;
        for (int base = 1; base < H0; base += NT) {
            s_flag[tid] = eligible(base + tid) ? 1 : 0;
            __syncthreads();
            if (tid == 0)
                for (int k = 0; k < NT && s_n < max_cuts; k++)
                    if (s_flag[k]) s_rows[s_n++] = base + k;
            __syncthreads();
            if (s_n >= max_cuts) break;
        }
    }
    const int n = s_n;
    for (int k = 0; k < n; k++) {
        const int r = s_rows[k];
        const double *src = T.M + r * stride;
        double *nw = T.M + (size_t)(H0 + k) * stride;
        const double rhs = src[0];
        const double frac = rhs - floor(rhs);
        for (int c = tid; c < T.stride; c += NT) {
            double v = 0.0;
            if (c < T.W) {
                const double coefficient = src[c];
                if (!upper) {
                    if (c == 0) v = floor(rhs);
                    else if (is_int(T.vcol[c])) {
                        const double fl = floor(coefficient);
                        const double a = __dsub_rn(coefficient, fl);
                        const double b = __dsub_rn(a, frac);
                        v = __dadd_rn(fl, ddiv(js_max0(b), __dsub_rn(1.0, frac)));
                    } else {
                        v = js_min0(ddiv(coefficient, __dsub_rn(1.0, frac)));
                    }
                    v = __dsub_rn(v, coefficient);  // cutting-strategies.ts:129-131
                } else {
                    if (c == 0) v = -frac;
                    else {
                        const double termCoeff = __dsub_rn(coefficient, floor(coefficient));
                        if (is_int(T.vcol[c]))
                            v = termCoeff <= frac ? -termCoeff : ddiv(__dmul_rn(-__dsub_rn(1.0, termCoeff), frac), termCoeff);
                        else
                            v = coefficient >= 0 ? -coefficient : ddiv(__dmul_rn(coefficient, frac), __dsub_rn(1.0, frac));
                    }
                }
            }
            nw[c] = v;
        }
        if (tid == 0) T.vrow[H0 + k] = first_index + k;
    }
    if (tid == 0) *n_added = n;
}

// isIntegral + getMostFractionalVar (mip-utils.ts:43-61,100-126) over the RHS column.  MASKED (DESIGN.md 2n): only
// the integer variables whose position p in model.integerVariables has bit p set in imask take part.
template <bool MASKED = false>
__device__ __forceinline__ void cta_mip_scan(const TabDev &T, MipOut *out, RedSmem &red, const uint32_t *imask = nullptr) {
    const VI init = {0.0, INT_MAX};
    VI best = init;  // (fraction, position in model.integerVariables)
    int nonint = 0;
    for (int r = 1 + threadIdx.x; r < T.H; r += blockDim.x) {
        const int v = T.vrow[r];
        if (v < 0 || v >= T.n_index) continue;
        const int p = T.intpos[v];
        if (p < 0) continue;
        if (MASKED && !((imask[p >> 5] >> (p & 31)) & 1u)) continue;
        const double x = T.M[(size_t)r * T.stride];
        const double fr = fabs(x - js_round(x));
        if (fr > T.prec) nonint = 1;
        if (fr > 0.0 && (fr > best.v || (fr == best.v && p < best.i))) { best.v = fr; best.i = p; }
    }
    best = block_reduce_vi<false>(best, init, red);
    nonint = block_reduce_int<1>(nonint, red);
    if (threadIdx.x == 0) { out->is_integral = nonint == 0; out->var_index = -1; out->value = 0.0; }
    __syncthreads();
    if (best.i != INT_MAX && best.v > 0.0) {
        for (int r = 1 + threadIdx.x; r < T.H; r += blockDim.x) {
            const int v = T.vrow[r];
            if (v >= 0 && v < T.n_index && T.intpos[v] == best.i) {
                out->var_index = v;
                out->value = T.M[(size_t)r * T.stride];
            }
        }
    }
    __syncthreads();
}

__global__ void __launch_bounds__(256) k_mip_scan(const TabDev *Tp, MipOut *out) {
    __shared__ RedSmem red;
    __shared__ TabDev T;
    if (threadIdx.x == 0) T = *Tp;
    __syncthreads();
    cta_mip_scan(T, out, red);
}

// Snapshot / restore of the CURRENT tableau buffer.  The ping-pong step swaps TabDev.M / M2 on the
// device, so a host-side memcpy enqueued ahead of time cannot know which buffer will be current.
__global__ void __launch_bounds__(256) k_copy_current(const TabDev *Tp, double *buf, int to_buf) {
    const TabDev &T = *Tp;
    const size_t n2 = ((size_t)T.H * T.stride) >> 1;  // stride is a multiple of 16 doubles
    double2 *m = reinterpret_cast<double2 *>(T.M);
    double2 *b = reinterpret_cast<double2 *>(buf);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += (size_t)gridDim.x * blockDim.x) {
        if (to_buf) b[i] = m[i]; else m[i] = b[i];
    }
}

}  // namespace jslp
