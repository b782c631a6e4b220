/*
 * oracle/jslp_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Single-threaded CPU restatement (plain C, IEEE fp64, no FMA contraction) of the
 * jsLPSolver LP/MIP hot path.  It is the checker the CUDA path is compared with; only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load it.  Nothing under jslpsolver_b200/ may import, link or call it.
 *
 * Reference files restated here (all under /root/reference/src/tableau/):
 *   simplex.ts:14-23    simplex            -> orc_simplex
 *   simplex.ts:25-98    phase1             -> orc_phase1
 *   simplex.ts:100-325  phase2             -> orc_phase2
 *   simplex.ts:330-413  pivot              -> orc_pivot
 *   simplex.ts:415-440  checkForCycles     -> cycles_ref (literal) / cycles_fast (equivalent)
 *   tableau.ts:420-430  setEvaluation      -> set_evaluation
 *   backup.ts:13-105    copy/save/restore  -> orc_save / orc_restore
 *   cutting-strategies.ts:16-72 addCutConstraints -> orc_add_cuts
 *   cutting-strategies.ts:74-212 addLowerBoundMIRCut / addUpperBoundMIRCut / applyMIRCuts -> orc_add_mir_cut / orc_apply_mir_cuts
 *   mip-utils.ts:67-98  computeFractionalVolume -> orc_fractional_volume
 *   enhanced-branch-and-cut.ts:54-437  createEnhancedBranchAndCutService -> orc_enhanced_branch_and_cut
 *   incremental-branch-and-cut.ts:28-499 createIncrementalBranchAndCutService -> orc_enhanced_branch_and_cut(incremental = 1)
 *   dynamic-modification.ts:16-316 putInBase / takeOutOfBase / updateRightHandSide / updateConstraintCoefficient /
 *                       updateCost / addConstraint / removeConstraint / addVariable / removeVariable -> orc_dm_*
 *   mip-utils.ts:43-61,100-126  isIntegral / getMostFractionalVar
 *   min-heap.ts:18-119  BranchMinHeap      -> heap_push / heap_pop
 *   branch-and-cut.ts:33-199    applyCuts / branchAndCut -> apply_cuts / orc_branch_and_cut
 *
 * Parity pinning: the reference cannot run in the build container (no JS engine), so this
 * restatement is pinned against the reference's own golden vectors: the `expects` blocks of
 * the 47 test/test-sanity fixtures (tests/test_oracle_golden.py) and the README known
 * answers.  The pivot sequence / basis arrays are NOT pinned by any reference test
 * ("parity unpinned" for those; see DESIGN.md).
 *
 * Build: gcc -O2 -ffp-contract=off -fno-fast-math -shared -fPIC (oracle/Makefile).
 */
#include <math.h>
#include <stdio.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    int type;       /* 0 = "min" (x >= value), 1 = "max" (x <= value) */
    int varIndex;
    double value;
} orc_cut;

typedef struct {
    double relaxedEvaluation;
    orc_cut *cuts;
    int nCuts;
    /* incremental service only (incremental-branch-and-cut.ts:49-53) */
    void *parentCheckpoint;
    orc_cut newCut;
    int hasNewCut;
} orc_branch;

typedef struct {
    orc_branch *branch;
    long seq;
} heap_entry;

typedef struct {
    int W, H, nVars, lastElementIndex;
    double *M;
    int *vrow, *vcol, *rowOf, *colOf;
    int nOpt;
    double *optRC; /* nOpt * W */
    int mapLen;
    int valid;
} orc_saved;

typedef struct orc_tab {
    int W, H;       /* logical width / height (stride == W, as the reference) */
    int capRows;
    double *M;
    int *vrow;      /* varIndexByRow, capRows entries */
    int *vcol;      /* varIndexByCol, W entries */
    int *rowOf, *colOf; /* rowByVarIndex / colByVarIndex */
    int mapCap;
    unsigned char *unres; /* unrestrictedVars by var index */
    int unresN;
    int *intVars;   /* model.integerVariables[].index in model order */
    int nInt;
    int nOpt;       /* optionalObjectives, sorted by priority asc */
    double *optRC;  /* nOpt * W */
    double precision;
    int checkCycles, fastCycles, isMin;
    double tolerance;
    int nVars, lastElementIndex;
    int feasible, bounded, simplexIters, unboundedVar;
    double evaluation, bestPossibleEval;
    int isIntegralFlag, bncIterations;
    int pricingBatchStart;
    int cyclePhase, cycleStart, cycleLen; /* model.messages restated */
    orc_saved saved;
    /* pivot log (row, col, leavingVar, enteringVar) x cap */
    int *plog;
    long plogCap, plogN;
    long totalPivots;
    long lastP1, lastP2;
    /* node log for branch and cut: 8 doubles per evaluated node */
    double *nlog;
    long nlogCap, nlogN;
    long maxNodes; /* safety cap, 0 = none */
    int useMIR;    /* model.useMIRCuts */
    /* best cuts of the winning branch (for tests) */
    orc_cut *bestCuts;
    int nBestCuts;
    int *nzc; /* pivot scratch: nonZeroColumns (simplex.ts:328) */
    long pivotLimit; /* bench sampling only: stop a phase loop after this many pivots (0 = off) */
    int truncated;
} orc_tab;

/* JS Math.round: nearest integer, ties toward +Infinity */
static double js_round(double x) {
    if (!(x == x) || isinf(x)) return x;
    double f = floor(x);
    return (x - f >= 0.5) ? f + 1.0 : f;
}

static int nz16(double v) { return !(v >= -1e-16 && v <= 1e-16); }

static void ensure_maps(orc_tab *t, int n) {
    if (n <= t->mapCap) return;
    int cap = t->mapCap ? t->mapCap : 16;
    while (cap < n) cap *= 2;
    t->rowOf = (int *)realloc(t->rowOf, sizeof(int) * cap);
    t->colOf = (int *)realloc(t->colOf, sizeof(int) * cap);
    for (int i = t->mapCap; i < cap; i++) { t->rowOf[i] = -1; t->colOf[i] = -1; }
    t->mapCap = cap;
}

static void ensure_rows(orc_tab *t, int rows) {
    if (rows <= t->capRows) return;
    int cap = t->capRows ? t->capRows : 4;
    while (cap < rows) cap *= 2;
    t->M = (double *)realloc(t->M, sizeof(double) * (size_t)cap * t->W);
    memset(t->M + (size_t)t->capRows * t->W, 0, sizeof(double) * (size_t)(cap - t->capRows) * t->W);
    t->vrow = (int *)realloc(t->vrow, sizeof(int) * cap);
    t->capRows = cap;
}

orc_tab *orc_create(int width, int height, double precision) {
    orc_tab *t = (orc_tab *)calloc(1, sizeof(orc_tab));
    t->W = width; t->H = height; t->precision = precision;
    ensure_rows(t, height);
    t->vcol = (int *)calloc(width, sizeof(int));
    t->nVars = width + height - 2;
    t->lastElementIndex = t->nVars;
    ensure_maps(t, t->nVars + 1);
    t->feasible = 1; t->bounded = 1; t->checkCycles = 1; t->isMin = 1;
    t->pricingBatchStart = 1;
    t->unboundedVar = -1;
    return t;
}

void orc_destroy(orc_tab *t) {
    if (!t) return;
    free(t->M); free(t->vrow); free(t->vcol); free(t->rowOf); free(t->colOf);
    free(t->unres); free(t->intVars); free(t->optRC);
    free(t->saved.M); free(t->saved.vrow); free(t->saved.vcol); free(t->saved.rowOf);
    free(t->saved.colOf); free(t->saved.optRC);
    free(t->plog); free(t->nlog); free(t->bestCuts); free(t->nzc);
    free(t);
}

/* upload of the state produced by Tableau._resetMatrix (tableau.ts:319-380) */
void orc_upload(orc_tab *t, const double *matrix, const int *vrow, const int *vcol) {
    memcpy(t->M, matrix, sizeof(double) * (size_t)t->H * t->W);
    memcpy(t->vrow, vrow, sizeof(int) * t->H);
    memcpy(t->vcol, vcol, sizeof(int) * t->W);
    for (int i = 0; i < t->mapCap; i++) { t->rowOf[i] = -1; t->colOf[i] = -1; }
    for (int r = 1; r < t->H; r++) {
        if (vrow[r] < 0 || vrow[r] >= t->mapCap) { fprintf(stderr, "orc_upload: row label %d out of range\n", vrow[r]); abort(); }
        t->rowOf[vrow[r]] = r;
    }
    for (int c = 1; c < t->W; c++) {
        if (vcol[c] < 0 || vcol[c] >= t->mapCap) { fprintf(stderr, "orc_upload: column label %d out of range\n", vcol[c]); abort(); }
        t->colOf[vcol[c]] = c;
    }
}

void orc_set_unrestricted(orc_tab *t, const unsigned char *flags, int n) {
    free(t->unres);
    t->unres = (unsigned char *)malloc(n > 0 ? n : 1);
    if (n > 0) memcpy(t->unres, flags, n);
    t->unresN = n;
}

void orc_set_integers(orc_tab *t, const int *varIdx, int n) {
    free(t->intVars);
    t->intVars = (int *)malloc(sizeof(int) * (n > 0 ? n : 1));
    if (n > 0) memcpy(t->intVars, varIdx, sizeof(int) * n);
    t->nInt = n;
}

void orc_set_optional(orc_tab *t, int n, const double *rc /* n*W, priority order */) {
    free(t->optRC);
    t->nOpt = n;
    t->optRC = (double *)malloc(sizeof(double) * (size_t)(n > 0 ? n : 1) * t->W);
    if (n > 0) memcpy(t->optRC, rc, sizeof(double) * (size_t)n * t->W);
}

void orc_set_options(orc_tab *t, int checkCycles, int fastCycles, int isMin, double tolerance,
                     long maxNodes) {
    t->checkCycles = checkCycles; t->fastCycles = fastCycles; t->isMin = isMin;
    t->tolerance = tolerance; t->maxNodes = maxNodes;
}

void orc_set_use_mir(orc_tab *t, int useMIR) { t->useMIR = useMIR; }

void orc_enable_pivot_log(orc_tab *t, long cap) {
    free(t->plog);
    t->plog = (int *)malloc(sizeof(int) * 4 * (size_t)(cap > 0 ? cap : 1));
    t->plogCap = cap; t->plogN = 0;
}

void orc_enable_node_log(orc_tab *t, long cap) {
    free(t->nlog);
    t->nlog = (double *)malloc(sizeof(double) * 8 * (size_t)(cap > 0 ? cap : 1));
    t->nlogCap = cap; t->nlogN = 0;
}

static int is_unres(const orc_tab *t, int varIndex) {
    return varIndex >= 0 && varIndex < t->unresN && t->unres[varIndex];
}

/* simplex.ts:330-413 */
void orc_pivot(orc_tab *t, int pr, int pc) {
    double *M = t->M;
    const int W = t->W, H = t->H;
    double *prow = M + (size_t)pr * W;
    const double quotient = prow[pc];

    const int leaving = t->vrow[pr];
    const int entering = t->vcol[pc];
    if (t->plog && t->plogN < t->plogCap) {
        int *e = t->plog + 4 * t->plogN;
        e[0] = pr; e[1] = pc; e[2] = leaving; e[3] = entering;
        t->plogN++;
    }
    t->totalPivots++;
    t->vrow[pr] = entering;
    t->vcol[pc] = leaving;
    ensure_maps(t, (leaving > entering ? leaving : entering) + 1);
    t->rowOf[entering] = pr;
    t->rowOf[leaving] = -1;
    t->colOf[entering] = -1;
    t->colOf[leaving] = pc;

    if (!t->nzc) t->nzc = (int *)malloc(sizeof(int) * W);
    int *nzc = t->nzc;
    int nnz = 0;
    for (int c = 0; c < W; c++) {
        double val = prow[c];
        if (nz16(val)) {
            prow[c] = val / quotient;
            nzc[nnz++] = c;
        } else {
            prow[c] = 0;
        }
    }
    prow[pc] = 1 / quotient;

    for (int r = 0; r < H; r++) {
        if (r == pr) continue;
        double *row = M + (size_t)r * W;
        const double coefficient = row[pc];
        if (nz16(coefficient)) {
            for (int i = 0; i < nnz; i++) {
                const int c = nzc[i];
                const double v0 = prow[c];
                if (nz16(v0)) {
                    const double prod = coefficient * v0; /* separate rounding: JS has no FMA */
                    row[c] = row[c] - prod;
                } else if (v0 != 0) {
                    prow[c] = 0;
                }
            }
            row[pc] = -coefficient / quotient;
        }
        /* simplex.ts:389-391: the reference's `else if (coefficient !== 0) matrix[...] = 0` sits INSIDE
         * `if (!(pivotColVal >= -1e-16 && pivotColVal <= 1e-16))` (:371) and tests the same value with the
         * same predicate (:374), so it is dead code: a pivot-column entry with |x| <= 1e-16 (tiny non-zero
         * included) is left untouched.  Round 1 flattened the two ifs and made the branch live, which
         * changed low-order bits and, through them, the B&B path of StockCuttingProblem / Vendor Selection. */
    }

    for (int o = 0; o < t->nOpt; o++) {
        double *rc = t->optRC + (size_t)o * W;
        const double coefficient = rc[pc];
        if (coefficient != 0) {
            for (int i = 0; i < nnz; i++) {
                const int c = nzc[i];
                const double v0 = prow[c];
                if (v0 != 0) {
                    const double prod = coefficient * v0;
                    rc[c] = rc[c] - prod;
                }
            }
            rc[pc] = -coefficient / quotient;
        }
    }
}

/* simplex.ts:415-440, literal restatement. list = pairs (a,b), n entries. returns 1 if found */
static int cycles_ref(const int *list, long n, long *start, long *len) {
    for (long e1 = 0; e1 < n - 1; e1++) {
        for (long e2 = e1 + 1; e2 < n; e2++) {
            if (list[2 * e1] == list[2 * e2] && list[2 * e1 + 1] == list[2 * e2 + 1]) {
                if (e2 - e1 > n - e2) break;
                int found = 1;
                for (long i = 1; i < e2 - e1; i++) {
                    if (list[2 * (e1 + i)] != list[2 * (e2 + i)] ||
                        list[2 * (e1 + i) + 1] != list[2 * (e2 + i) + 1]) { found = 0; break; }
                }
                if (found) { *start = e1; *len = e2 - e1; return 1; }
            }
        }
    }
    return 0;
}

/* Equivalent detector, valid when called after every push with no earlier hit (the only way
 * the reference calls it): any repeated block must then end at the last element, so only
 * suffix squares need checking; the literal scan returns the smallest e1 = the largest L. */
static int cycles_fast(const int *list, long n, long *start, long *len) {
    for (long L = n / 2; L >= 1; L--) {
        const long e1 = n - 2 * L, e2 = n - L;
        int eq = 1;
        for (long i = 0; i < L; i++) {
            if (list[2 * (e1 + i)] != list[2 * (e2 + i)] ||
                list[2 * (e1 + i) + 1] != list[2 * (e2 + i) + 1]) { eq = 0; break; }
        }
        if (eq) { *start = e1; *len = L; return 1; }
    }
    return 0;
}

/* exported for the equivalence test of the two detectors */
int orc_cycles_ref(const int *list, long n, long *s, long *l) { return cycles_ref(list, n, s, l); }
int orc_cycles_fast(const int *list, long n, long *s, long *l) { return cycles_fast(list, n, s, l); }

typedef struct { int *v; long n, cap; } pairlist;
static void pl_push(pairlist *p, int a, int b) {
    if (p->n == p->cap) {
        p->cap = p->cap ? p->cap * 2 : 64;
        p->v = (int *)realloc(p->v, sizeof(int) * 2 * p->cap);
    }
    p->v[2 * p->n] = a; p->v[2 * p->n + 1] = b; p->n++;
}

static int check_cycle(orc_tab *t, pairlist *p, int phase) {
    long s = 0, l = 0;
    int hit = t->fastCycles ? cycles_fast(p->v, p->n, &s, &l) : cycles_ref(p->v, p->n, &s, &l);
    if (hit) { t->cyclePhase = phase; t->cycleStart = (int)s; t->cycleLen = (int)l; }
    return hit;
}

/* simplex.ts:25-98 */
long orc_phase1(orc_tab *t) {
    pairlist pl = {0, 0, 0};
    const int W = t->W;
    const double precision = t->precision;
    long iterations = 0;
    for (;;) {
        const int lastRow = t->H - 1, lastColumn = W - 1;
        double *M = t->M;
        int leavingRow = 0;
        double rhsValue = -precision;
        for (int r = 1; r <= lastRow; r++) {
            const double value = M[(size_t)r * W];
            if (value < rhsValue) { rhsValue = value; leavingRow = r; }
        }
        if (leavingRow == 0) { t->feasible = 1; break; }

        int enteringColumn = 0;
        double maxQuotient = -INFINITY;
        const double *lrow = M + (size_t)leavingRow * W;
        for (int c = 1; c <= lastColumn; c++) {
            const double coefficient = lrow[c];
            if (is_unres(t, t->vcol[c]) || coefficient < -precision) {
                const double quotient = -M[c] / coefficient;
                if (maxQuotient < quotient) { maxQuotient = quotient; enteringColumn = c; }
            }
        }
        if (enteringColumn == 0) { t->feasible = 0; break; }

        if (t->checkCycles) {
            pl_push(&pl, t->vrow[leavingRow], t->vcol[enteringColumn]);
            if (check_cycle(t, &pl, 1)) { t->feasible = 0; break; }
        }
        if (t->pivotLimit > 0 && t->totalPivots >= t->pivotLimit) { t->truncated = 1; t->feasible = 0; break; }
        orc_pivot(t, leavingRow, enteringColumn);
        iterations++;
    }
    free(pl.v);
    t->lastP1 = iterations;
    return iterations;
}

/* tableau.ts:420-430 */
static void set_evaluation(orc_tab *t) {
    const double roundingCoeff = js_round(1 / t->precision);
    const double evaluation = t->M[0];
    const double rounded = js_round((2.220446049250313e-16 + evaluation) * roundingCoeff) / roundingCoeff;
    t->evaluation = rounded;
    if (t->simplexIters == 0) t->bestPossibleEval = rounded;
}

/* one pricing test, simplex.ts:151-177 / 191-217.  returns 1 when the column was deferred
 * to the optional-objective tie-break list */
static void price_col(const orc_tab *t, int c, double reducedCost, double *enteringValue,
                      int *enteringColumn, int *isNeg) {
    if (is_unres(t, t->vcol[c]) && reducedCost < 0) {
        if (-reducedCost > *enteringValue) {
            *enteringValue = -reducedCost; *enteringColumn = c; *isNeg = 1;
        }
        return;
    }
    if (reducedCost > *enteringValue) {
        *enteringValue = reducedCost; *enteringColumn = c; *isNeg = 0;
    }
}

/* simplex.ts:100-325 */
long orc_phase2(orc_tab *t) {
    pairlist pl = {0, 0, 0};
    const int W = t->W;
    const double precision = t->precision;
    const int nOpt = t->nOpt;
    int *optCols = nOpt > 0 ? (int *)malloc(sizeof(int) * W) : 0;
    int *optCols2 = nOpt > 0 ? (int *)malloc(sizeof(int) * W) : 0;
    long iterations = 0;

    const int nColumns = W - 1;
    int batchSize = (int)floor(sqrt((double)nColumns));
    if (batchSize < 50) batchSize = 50;
    if (batchSize > 500) batchSize = 500;
    const int usePartial = nColumns > batchSize * 2;

    for (;;) {
        double *M = t->M;
        const int lastRow = t->H - 1, lastColumn = W - 1;
        int nOptCols = 0;
        int enteringColumn = 0;
        double enteringValue = precision;
        int isNeg = 0;

        if (usePartial) {
            const int startBatch = t->pricingBatchStart;
            int batchesScanned = 0;
            const int totalBatches = (nColumns + batchSize - 1) / batchSize;
            while (enteringColumn == 0 && batchesScanned < totalBatches) {
                const int batchStart = t->pricingBatchStart;
                int batchEnd = batchStart + batchSize - 1;
                if (batchEnd > lastColumn) batchEnd = lastColumn;
                for (int c = batchStart; c <= batchEnd; c++) {
                    const double rc = M[c];
                    if (nOpt > 0 && -precision < rc && rc < precision) { optCols[nOptCols++] = c; continue; }
                    price_col(t, c, rc, &enteringValue, &enteringColumn, &isNeg);
                }
                t->pricingBatchStart = batchEnd >= lastColumn ? 1 : batchEnd + 1;
                batchesScanned++;
            }
            if (enteringColumn != 0) t->pricingBatchStart = startBatch;
        } else {
            for (int c = 1; c <= lastColumn; c++) {
                const double rc = M[c];
                if (nOpt > 0 && -precision < rc && rc < precision) { optCols[nOptCols++] = c; continue; }
                price_col(t, c, rc, &enteringValue, &enteringColumn, &isNeg);
            }
        }

        if (nOpt > 0) {
            int o = 0;
            while (enteringColumn == 0 && nOptCols > 0 && o < nOpt) {
                int n2 = 0;
                const double *rcs = t->optRC + (size_t)o * W;
                enteringValue = precision;
                for (int i = 0; i < nOptCols; i++) {
                    const int c = optCols[i];
                    const double rc = rcs[c];
                    if (-precision < rc && rc < precision) { optCols2[n2++] = c; continue; }
                    price_col(t, c, rc, &enteringValue, &enteringColumn, &isNeg);
                }
                int *tmp = optCols; optCols = optCols2; optCols2 = tmp;
                nOptCols = n2;
                o++;
            }
        }

        if (enteringColumn == 0) {
            set_evaluation(t);
            t->simplexIters++;
            break;
        }

        int leavingRow = 0;
        double minQuotient = INFINITY;
        for (int r = 1; r <= lastRow; r++) {
            const double rhsValue = M[(size_t)r * W];
            const double colValue = M[(size_t)r * W + enteringColumn];
            if (-precision < colValue && colValue < precision) continue;
            if (colValue > 0 && precision > rhsValue && rhsValue > -precision) {
                minQuotient = 0; leavingRow = r; break;
            }
            const double quotient = isNeg ? -rhsValue / colValue : rhsValue / colValue;
            if (quotient > precision && minQuotient > quotient) { minQuotient = quotient; leavingRow = r; }
        }

        if (minQuotient == INFINITY) {
            t->evaluation = -INFINITY;
            t->bounded = 0;
            t->unboundedVar = t->vcol[enteringColumn];
            break;
        }

        if (t->checkCycles) {
            pl_push(&pl, t->vrow[leavingRow], t->vcol[enteringColumn]);
            if (check_cycle(t, &pl, 2)) { t->feasible = 0; break; }
        }
        if (t->pivotLimit > 0 && t->totalPivots >= t->pivotLimit) { t->truncated = 1; break; }
        orc_pivot(t, leavingRow, enteringColumn);
        iterations++;
    }
    free(pl.v); free(optCols); free(optCols2);
    t->lastP2 = iterations;
    return iterations;
}

/* simplex.ts:14-23 */
void orc_simplex(orc_tab *t) {
    t->bounded = 1;
    t->lastP1 = t->lastP2 = 0;
    orc_phase1(t);
    if (t->feasible) orc_phase2(t);
}

/* backup.ts:13-51 */
void orc_save(orc_tab *t) {
    orc_saved *s = &t->saved;
    free(s->M); free(s->vrow); free(s->vcol); free(s->rowOf); free(s->colOf); free(s->optRC);
    s->W = t->W; s->H = t->H; s->nVars = t->nVars; s->lastElementIndex = t->lastElementIndex;
    s->M = (double *)malloc(sizeof(double) * (size_t)t->H * t->W);
    memcpy(s->M, t->M, sizeof(double) * (size_t)t->H * t->W);
    s->vrow = (int *)malloc(sizeof(int) * t->H);
    memcpy(s->vrow, t->vrow, sizeof(int) * t->H);
    s->vcol = (int *)malloc(sizeof(int) * t->W);
    memcpy(s->vcol, t->vcol, sizeof(int) * t->W);
    s->mapLen = t->mapCap;
    s->rowOf = (int *)malloc(sizeof(int) * t->mapCap);
    s->colOf = (int *)malloc(sizeof(int) * t->mapCap);
    memcpy(s->rowOf, t->rowOf, sizeof(int) * t->mapCap);
    memcpy(s->colOf, t->colOf, sizeof(int) * t->mapCap);
    s->nOpt = t->nOpt;
    s->optRC = (double *)malloc(sizeof(double) * (size_t)(t->nOpt > 0 ? t->nOpt : 1) * t->W);
    if (t->nOpt > 0) memcpy(s->optRC, t->optRC, sizeof(double) * (size_t)t->nOpt * t->W);
    s->valid = 1;
}

/* backup.ts:53-105 (feasible/bounded/evaluation are deliberately NOT restored) */
void orc_restore(orc_tab *t) {
    orc_saved *s = &t->saved;
    if (!s->valid) return;
    t->nVars = s->nVars;
    t->lastElementIndex = s->lastElementIndex;
    t->W = s->W; t->H = s->H;
    memcpy(t->M, s->M, sizeof(double) * (size_t)s->H * s->W);
    memcpy(t->vrow, s->vrow, sizeof(int) * s->H);
    memcpy(t->vcol, s->vcol, sizeof(int) * s->W);
    for (int v = 0; v < t->nVars && v < s->mapLen; v++) {
        t->rowOf[v] = s->rowOf[v];
        t->colOf[v] = s->colOf[v];
    }
    if (s->nOpt > 0 && t->nOpt > 0)
        memcpy(t->optRC, s->optRC, sizeof(double) * (size_t)s->nOpt * s->W);
}

static int new_element_index(orc_tab *t) { return t->lastElementIndex++; } /* tableau.ts:393-401 */

/* cutting-strategies.ts:16-72 */
void orc_add_cuts(orc_tab *t, const orc_cut *cuts, int n) {
    const int height = t->H, W = t->W, lastColumn = W - 1;
    ensure_rows(t, height + n);
    double *M = t->M;
    t->H = height + n;
    t->nVars = t->W + t->H - 2;
    for (int h = 0; h < n; h++) {
        const orc_cut *cut = &cuts[h];
        const int cutRow = height + h;
        double *crow = M + (size_t)cutRow * W;
        const double sign = cut->type == 0 ? -1 : 1;
        const int varIndex = cut->varIndex;
        int varRowIndex = t->rowOf[varIndex];
        if (varRowIndex == -1) {
            crow[0] = sign * cut->value;
            for (int c = 1; c <= lastColumn; c++) crow[c] = 0;
            crow[t->colOf[varIndex]] = sign;
        } else {
            const double *vr = M + (size_t)varRowIndex * W;
            const double varValue = vr[0];
            crow[0] = sign * (cut->value - varValue);
            for (int c = 1; c <= lastColumn; c++) crow[c] = -sign * vr[c];
        }
        varRowIndex = new_element_index(t);
        ensure_maps(t, varRowIndex + 1);
        t->vrow[cutRow] = varRowIndex;
        t->rowOf[varRowIndex] = cutRow;
        t->colOf[varRowIndex] = -1;
        t->nVars += 1;
    }
}

static int var_is_integer(const orc_tab *t, int varIndex) {
    for (int v = 0; v < t->nInt; v++)
        if (t->intVars[v] == varIndex) return 1;
    return 0;
}

/* Math.max(0, x) / Math.min(0, y) with JS semantics (NaN propagates; max(0,-0) = +0; min(0,-0) = -0) */
static double js_max0(double x) { return x != x ? x : (x > 0 ? x : 0.0); }
static double js_min0(double y) { return y != y ? y : (y < 0 ? y : (y == 0 && signbit(y) ? y : 0.0)); }

/* cutting-strategies.ts:74-134 (upper == 0) and 136-196 (upper != 0); returns 1 when a cut row was added */
int orc_add_mir_cut(orc_tab *t, int rowIndex, int upper) {
    if (rowIndex == 0) return 0;  /* costRowIndex */
    if (rowIndex < 0 || rowIndex >= t->H) return 0;
    const int W = t->W;
    if (!var_is_integer(t, t->vrow[rowIndex])) return 0;  /* integerVar undefined or not integer */
    const double rhsValue = t->M[(size_t)rowIndex * W];
    const double fractionalPart = rhsValue - floor(rhsValue);
    if (fractionalPart < t->precision || fractionalPart > 1 - t->precision) return 0;
    const int height = t->H;
    ensure_rows(t, height + 1);
    double *mat = t->M;
    const double *src = mat + (size_t)rowIndex * W;
    double *nw = mat + (size_t)height * W;
    t->H += 1;
    t->nVars += 1;
    const int slackVarIndex = new_element_index(t);
    ensure_maps(t, slackVarIndex + 1);
    t->vrow[height] = slackVarIndex;
    t->rowOf[slackVarIndex] = height;
    t->colOf[slackVarIndex] = -1;
    if (!upper) {
        nw[0] = floor(rhsValue);
        for (int c = 1; c < W; c++) {
            const double coefficient = src[c];
            if (var_is_integer(t, t->vcol[c])) {
                const double fl = floor(coefficient);
                const double a = coefficient - fl;
                const double b = a - fractionalPart;
                nw[c] = fl + js_max0(b) / (1 - fractionalPart);
            } else {
                nw[c] = js_min0(coefficient / (1 - fractionalPart));
            }
        }
        for (int c = 0; c < W; c++) nw[c] -= src[c];
    } else {
        nw[0] = -fractionalPart;
        for (int c = 1; c < W; c++) {
            const double coefficient = src[c];
            const double termCoeff = coefficient - floor(coefficient);
            if (var_is_integer(t, t->vcol[c])) {
                nw[c] = termCoeff <= fractionalPart ? -termCoeff : (-(1 - termCoeff) * fractionalPart) / termCoeff;
            } else {
                nw[c] = coefficient >= 0 ? -coefficient : (coefficient * fractionalPart) / (1 - fractionalPart);
            }
        }
    }
    return 1;
}

/* cutting-strategies.ts:198-212; returns the number of cuts added */
int orc_apply_mir_cuts(orc_tab *t) {
    const int height = t->H;
    int cutsAdded = 0;
    const int maxCuts = 10;
    for (int r = 1; r < height && cutsAdded < maxCuts; r++)
        if (orc_add_mir_cut(t, r, 0)) cutsAdded++;
    return cutsAdded;
}

/* mip-utils.ts:67-98 */
double orc_fractional_volume(const orc_tab *t, int ignoreIntegerValues) {
    double volume = -1;
    for (int r = 1; r < t->H; r++) {
        if (!var_is_integer(t, t->vrow[r])) continue;
        const double value = t->M[(size_t)r * t->W];
        const double distance = fabs(value);
        const double a = distance - floor(distance), b = floor(distance + 1);
        if ((a < b ? a : b) < t->precision) {  /* Math.min of two non-NaN numbers */
            if (!ignoreIntegerValues) return 0;
        } else if (volume == -1) {
            volume = distance;
        } else {
            volume *= distance;
        }
    }
    return volume == -1 ? 0 : volume;
}

/* mip-utils.ts:43-61 */
int orc_is_integral(const orc_tab *t) {
    for (int v = 0; v < t->nInt; v++) {
        const int row = t->rowOf[t->intVars[v]];
        if (row != -1) {
            const double value = t->M[(size_t)row * t->W];
            if (fabs(value - js_round(value)) > t->precision) return 0;
        }
    }
    return 1;
}

/* mip-utils.ts:100-126; returns var index or -1, value through *val */
int orc_most_fractional(const orc_tab *t, double *val) {
    double biggest = 0;
    int sel = -1;
    double selVal = 0;
    for (int v = 0; v < t->nInt; v++) {
        const int varIndex = t->intVars[v];
        const int row = t->rowOf[varIndex];
        if (row != -1) {
            const double varValue = t->M[(size_t)row * t->W];
            const double fraction = fabs(varValue - js_round(varValue));
            if (fraction > biggest) { biggest = fraction; sel = varIndex; selVal = varValue; }
        }
    }
    *val = selVal;
    return sel;
}

/* ---- dynamic-modification.ts ---- */
/* :16-34; returns the row, or -2 when no pivot element exists (the reference would call pivot(-1, c)) */
int orc_dm_put_in_base(orc_tab *t, int varIndex) {
    ensure_maps(t, varIndex + 1);
    int r = t->rowOf[varIndex];
    if (r == -1) {
        const int c = t->colOf[varIndex];
        for (int r1 = 1; r1 < t->H; r1++) {
            const double coefficient = t->M[(size_t)r1 * t->W + c];
            if (coefficient < -t->precision || t->precision < coefficient) { r = r1; break; }
        }
        if (r == -1) return -2;
        orc_pivot(t, r, c);
    }
    return r;
}

/* :36-55 -- the scan bound is `this.height` in the reference (not the width); kept, reading the flat matrix */
int orc_dm_take_out_of_base(orc_tab *t, int varIndex) {
    ensure_maps(t, varIndex + 1);
    int c = t->colOf[varIndex];
    if (c == -1) {
        const int r = t->rowOf[varIndex];
        const size_t pivotRowOffset = (size_t)r * t->W, total = (size_t)t->H * t->W;
        for (int c1 = 1; c1 < t->H; c1++) {
            if (pivotRowOffset + c1 >= total) break;  /* undefined in JS: both comparisons false */
            const double coefficient = t->M[pivotRowOffset + c1];
            if (coefficient < -t->precision || t->precision < coefficient) { c = c1; break; }
        }
        if (c == -1 || c >= t->W) return -2;
        orc_pivot(t, r, c);
    }
    return c;
}

/* :78-106 */
void orc_dm_update_rhs(orc_tab *t, int constraintIndex, double difference) {
    const int W = t->W, lastRow = t->H - 1;
    const int constraintRow = t->rowOf[constraintIndex];
    if (constraintRow == -1) {
        const int slackColumn = t->colOf[constraintIndex];
        for (int r = 0; r <= lastRow; r++) {
            double *row = t->M + (size_t)r * W;
            const double prod = difference * row[slackColumn];
            row[0] -= prod;
        }
        for (int o = 0; o < t->nOpt; o++) {
            double *rc = t->optRC + (size_t)o * W;
            const double prod = difference * rc[slackColumn];
            rc[0] -= prod;
        }
    } else {
        t->M[(size_t)constraintRow * W] -= difference;
    }
}

/* :108-135; returns 0, -1 for the reference's thrown Error, -2 when putInBase finds no pivot */
int orc_dm_update_coefficient(orc_tab *t, int constraintIndex, int varIndex, double difference) {
    if (constraintIndex == varIndex) return -1;
    const int r = orc_dm_put_in_base(t, constraintIndex);
    if (r < 0) return -2;
    const int W = t->W;
    double *row = t->M + (size_t)r * W;
    const int colVar = t->colOf[varIndex];
    if (colVar == -1) {
        const double *vr = t->M + (size_t)t->rowOf[varIndex] * W;
        for (int c = 0; c < W; c++) { const double prod = difference * vr[c]; row[c] += prod; }
    } else {
        row[colVar] -= difference;
    }
    return 0;
}

/* :137-160; optSlot = -1 for priority 0 (cost row), else the optional objective's position */
void orc_dm_update_cost(orc_tab *t, int varIndex, int optSlot, double difference) {
    const int W = t->W;
    const int varColumn = t->colOf[varIndex];
    if (varColumn == -1) {
        const double *vr = t->M + (size_t)t->rowOf[varIndex] * W;
        double *dst = optSlot < 0 ? t->M : t->optRC + (size_t)optSlot * W;
        for (int c = 0; c < W; c++) { const double prod = difference * vr[c]; dst[c] += prod; }
    } else {
        t->M[varColumn] -= difference;
    }
}

/* :162-220 */
void orc_dm_add_constraint(orc_tab *t, int isUpperBound, double rhs, int slackIndex, const int *termVar,
                           const double *termCoef, int nTerms) {
    const double sign = isUpperBound ? 1 : -1;
    const int lastRow = t->H, W = t->W;
    ensure_rows(t, lastRow + 1);
    double *row = t->M + (size_t)lastRow * W;
    for (int c = 0; c < W; c++) row[c] = 0;
    row[0] = sign * rhs;
    for (int k = 0; k < nTerms; k++) {
        const double coefficient = termCoef[k];
        const int varIndex = termVar[k];
        const int varRowIndex = t->rowOf[varIndex];
        if (varRowIndex == -1) {
            row[t->colOf[varIndex]] += sign * coefficient;
        } else {
            const double *vr = t->M + (size_t)varRowIndex * W;
            const double sc = sign * coefficient;
            for (int c = 0; c < W; c++) { const double prod = sc * vr[c]; row[c] -= prod; }
        }
    }
    ensure_maps(t, slackIndex + 1);
    /* the caller's index came from Tableau.getNewElementIndex (model.ts:103-124), which advanced lastElementIndex:
       branching cuts added later must not reuse it */
    if (slackIndex + 1 > t->lastElementIndex) t->lastElementIndex = slackIndex + 1;
    t->vrow[lastRow] = slackIndex;
    t->rowOf[slackIndex] = lastRow;
    t->colOf[slackIndex] = -1;
    t->H += 1;
}

/* :222-251 (availableIndexes is host bookkeeping of the caller) */
int orc_dm_remove_constraint(orc_tab *t, int slackIndex) {
    const int lastRow = t->H - 1, W = t->W;
    const int r = orc_dm_put_in_base(t, slackIndex);
    if (r < 0) return -2;
    double *a = t->M + (size_t)r * W, *b = t->M + (size_t)lastRow * W;
    for (int c = 0; c < W; c++) { const double tmp = b[c]; b[c] = a[c]; a[c] = tmp; }
    t->vrow[r] = t->vrow[lastRow];
    t->vrow[lastRow] = -1;
    t->rowOf[slackIndex] = -1;
    /* the reference leaves rowByVarIndex of the moved row's variable stale here (dynamic-modification.ts:241-243);
       so does this restatement -- callers that go on must not rely on it, exactly as in the reference */
    t->H -= 1;
    return 0;
}

/* :253-302; costEntry = (isMinimization ? -cost : cost); optSlot = -1 for priority 0 */
void orc_dm_add_variable(orc_tab *t, int varIndex, double costEntry, int optSlot, int isInteger, int isUnrestricted) {
    const int oldW = t->W, newW = oldW + 1, H = t->H;
    double *nm = (double *)calloc((size_t)(t->capRows > H ? t->capRows : H) * newW, sizeof(double));
    for (int r = 0; r < H; r++) memcpy(nm + (size_t)r * newW, t->M + (size_t)r * oldW, sizeof(double) * oldW);
    free(t->M);
    t->M = nm;
    t->W = newW;
    t->vcol = (int *)realloc(t->vcol, sizeof(int) * newW);
    if (t->nOpt > 0) {
        double *no = (double *)calloc((size_t)t->nOpt * newW, sizeof(double));
        for (int o = 0; o < t->nOpt; o++) memcpy(no + (size_t)o * newW, t->optRC + (size_t)o * oldW, sizeof(double) * oldW);
        free(t->optRC);
        t->optRC = no;
    }
    free(t->nzc); t->nzc = 0;
    const int lastColumn = newW - 1;
    if (optSlot < 0) t->M[lastColumn] = costEntry;
    else { t->optRC[(size_t)optSlot * newW + lastColumn] = costEntry; t->M[lastColumn] = 0; }
    ensure_maps(t, varIndex + 1);
    if (varIndex + 1 > t->lastElementIndex) t->lastElementIndex = varIndex + 1;  /* getNewElementIndex (model.ts:163) */
    t->colOf[varIndex] = lastColumn;
    t->vcol[lastColumn] = varIndex;
    /* Model.addVariable (model.ts:169-187): integerVariables.push, unrestrictedVariables[varIndex] = true */
    if (isInteger) {
        t->intVars = (int *)realloc(t->intVars, sizeof(int) * (size_t)(t->nInt + 1));
        t->intVars[t->nInt++] = varIndex;
    }
    if (isUnrestricted) {
        if (varIndex >= t->unresN) {
            t->unres = (unsigned char *)realloc(t->unres, (size_t)varIndex + 1);
            memset(t->unres + t->unresN, 0, (size_t)(varIndex + 1 - t->unresN));
            t->unresN = varIndex + 1;
        }
        t->unres[varIndex] = 1;
    }
}

/* :304-316 (the stride stays width: the reference only decrements `width`, leaving the matrix layout at the old
   width -- every later access uses the NEW width as stride, i.e. the reference's tableau is scrambled after this
   call unless the removed column was the last one; restated literally).  The optional objectives are another
   matter: the reference keeps one reducedCosts array per objective, indexed by column alone, so a narrower width
   moves none of them.  Here they share one nOpt x W block, so each row is compacted to the new width to keep
   objective o at o * (W - 1), where separate arrays would leave its entries. */
int orc_dm_remove_variable(orc_tab *t, int varIndex) {
    const int W = t->W, lastColumn = W - 1;
    const int c = orc_dm_take_out_of_base(t, varIndex);
    if (c < 0) return -2;
    for (int r = 0; r < t->H; r++) t->M[(size_t)r * W + c] = t->M[(size_t)r * W + lastColumn];
    t->vcol[c] = t->vcol[lastColumn];
    t->rowOf[varIndex] = -1;
    t->colOf[varIndex] = -1;
    for (int o = 1; o < t->nOpt; o++)
        memmove(t->optRC + (size_t)o * (W - 1), t->optRC + (size_t)o * W, sizeof(double) * (size_t)(W - 1));
    t->W -= 1;
    return 0;
}

/* ---- min-heap.ts ---- */
typedef struct { heap_entry *h; long size, cap, seq; } minheap;

static int is_before(const heap_entry *a, const heap_entry *b) {
    if (a->branch->relaxedEvaluation != b->branch->relaxedEvaluation)
        return a->branch->relaxedEvaluation < b->branch->relaxedEvaluation;
    return a->seq > b->seq; /* LIFO ties */
}

static void heap_push(minheap *hp, orc_branch *br) {
    if (hp->size == hp->cap) {
        hp->cap = hp->cap ? hp->cap * 2 : 64;
        hp->h = (heap_entry *)realloc(hp->h, sizeof(heap_entry) * hp->cap);
    }
    long idx = hp->size++;
    heap_entry entry = {br, hp->seq++};
    while (idx > 0) {
        long parentIdx = (idx - 1) >> 1;
        if (!is_before(&entry, &hp->h[parentIdx])) break;
        hp->h[idx] = hp->h[parentIdx];
        idx = parentIdx;
    }
    hp->h[idx] = entry;
}

static orc_branch *heap_pop(minheap *hp) {
    if (hp->size == 0) return 0;
    orc_branch *result = hp->h[0].branch;
    hp->size--;
    if (hp->size == 0) return result;
    heap_entry last = hp->h[hp->size];
    long idx = 0;
    const long halfSize = hp->size >> 1;
    while (idx < halfSize) {
        long childIdx = (idx << 1) + 1;
        const long rightIdx = childIdx + 1;
        if (rightIdx < hp->size && is_before(&hp->h[rightIdx], &hp->h[childIdx])) childIdx = rightIdx;
        if (!is_before(&hp->h[childIdx], &last)) break;
        hp->h[idx] = hp->h[childIdx];
        idx = childIdx;
    }
    hp->h[idx] = last;
    return result;
}

static orc_branch *make_branch(double ev, int nCuts) {
    orc_branch *b = (orc_branch *)malloc(sizeof(orc_branch));
    b->relaxedEvaluation = ev; b->nCuts = 0;
    b->parentCheckpoint = 0; b->hasNewCut = 0;
    b->cuts = (orc_cut *)malloc(sizeof(orc_cut) * (nCuts > 0 ? nCuts : 1));
    return b;
}
static void checkpoint_release_v(void *c);
static void free_branch(orc_branch *b) { if (b) { if (b->parentCheckpoint) checkpoint_release_v(b->parentCheckpoint); free(b->cuts); free(b); } }

/* branch-and-cut.ts:33-52 */
static void apply_cuts(orc_tab *t, const orc_cut *cuts, int n) {
    orc_restore(t);
    orc_add_cuts(t, cuts, n);
    orc_simplex(t);
    if (t->useMIR) {
        int fractionalVolumeImproved = 1;
        while (fractionalVolumeImproved) {
            const double fractionalVolumeBefore = orc_fractional_volume(t, 1);
            orc_apply_mir_cuts(t);
            orc_simplex(t);
            const double fractionalVolumeAfter = orc_fractional_volume(t, 1);
            if (fractionalVolumeAfter >= 0.9 * fractionalVolumeBefore) fractionalVolumeImproved = 0;
        }
    }
}

void orc_apply_cuts(orc_tab *t, const orc_cut *cuts, int n) { apply_cuts(t, cuts, n); }

/* branch-and-cut.ts:54-199; timeout (Date.now) is not restated: parity runs disable it */
void orc_branch_and_cut(orc_tab *t) {
    minheap hp = {0, 0, 0, 0};
    int iterations = 0;
    const double tolerance = t->tolerance;
    int toleranceFlag = 1;
    double bestEvaluation = INFINITY;
    orc_branch *bestBranch = 0;
    const int nOpt = t->nOpt;
    double *bestOpt = (double *)malloc(sizeof(double) * (nOpt > 0 ? nOpt : 1));
    for (int o = 0; o < nOpt; o++) bestOpt[o] = INFINITY;

    heap_push(&hp, make_branch(-INFINITY, 0));
    while (hp.size > 0 && toleranceFlag) {
        if (t->maxNodes > 0 && iterations >= t->maxNodes) break;
        double acceptableThreshold;
        if (t->isMin) acceptableThreshold = t->bestPossibleEval * (1 + tolerance);
        else acceptableThreshold = t->bestPossibleEval * (1 - tolerance);
        if (tolerance > 0) {
            if (bestEvaluation < acceptableThreshold) toleranceFlag = 0;
        }

        orc_branch *active = heap_pop(&hp);
        if (active->relaxedEvaluation > bestEvaluation) { free_branch(active); continue; }

        const long pivBefore = t->totalPivots;
        apply_cuts(t, active->cuts, active->nCuts);
        iterations++;

        double *nl = 0;
        if (t->nlog && t->nlogN < t->nlogCap) {
            nl = t->nlog + 8 * t->nlogN++;
            nl[0] = iterations; nl[1] = active->nCuts; nl[2] = t->feasible;
            nl[3] = t->evaluation; nl[4] = -1; nl[5] = -1; nl[6] = 0;
            nl[7] = (double)(t->totalPivots - pivBefore);
        }

        if (!t->feasible) { free_branch(active); continue; }
        const double evaluation = t->evaluation;
        if (evaluation > bestEvaluation) { free_branch(active); continue; }

        if (evaluation == bestEvaluation) {
            int worse = 1;
            for (int o = 0; o < nOpt; o++) {
                const double v = t->optRC[(size_t)o * t->W];
                if (v > bestOpt[o]) break;
                else if (v < bestOpt[o]) { worse = 0; break; }
            }
            if (worse) { free_branch(active); continue; }
        }

        if (orc_is_integral(t)) {
            if (nl) nl[4] = 1;
            t->isIntegralFlag = 1;
            if (iterations == 1) {
                t->bncIterations = iterations;
                free_branch(active);
                goto done;
            }
            if (bestBranch) free_branch(bestBranch);
            bestBranch = active;
            bestEvaluation = evaluation;
            for (int o = 0; o < nOpt; o++) bestOpt[o] = t->optRC[(size_t)o * t->W];
        } else {
            if (nl) nl[4] = 0;
            if (iterations == 1) orc_save(t);
            double value;
            const int varIndex = orc_most_fractional(t, &value);
            if (nl) { nl[5] = varIndex; nl[6] = value; }
            orc_branch *high = make_branch(evaluation, active->nCuts + 1);
            orc_branch *low = make_branch(evaluation, active->nCuts + 1);
            for (int c = 0; c < active->nCuts; c++) {
                const orc_cut cut = active->cuts[c];
                if (cut.varIndex == varIndex) {
                    if (cut.type == 0) low->cuts[low->nCuts++] = cut;
                    else high->cuts[high->nCuts++] = cut;
                } else {
                    high->cuts[high->nCuts++] = cut;
                    low->cuts[low->nCuts++] = cut;
                }
            }
            orc_cut ch = {0, varIndex, ceil(value)};
            orc_cut cl = {1, varIndex, floor(value)};
            high->cuts[high->nCuts++] = ch;
            low->cuts[low->nCuts++] = cl;
            heap_push(&hp, high);
            heap_push(&hp, low);
            free_branch(active);
        }
    }

    if (bestBranch) {
        apply_cuts(t, bestBranch->cuts, bestBranch->nCuts);
        free(t->bestCuts);
        t->bestCuts = (orc_cut *)malloc(sizeof(orc_cut) * (bestBranch->nCuts > 0 ? bestBranch->nCuts : 1));
        memcpy(t->bestCuts, bestBranch->cuts, sizeof(orc_cut) * bestBranch->nCuts);
        t->nBestCuts = bestBranch->nCuts;
        free_branch(bestBranch);
    }
    t->bncIterations = iterations;
done:
    for (long i = 0; i < hp.size; i++) free_branch(hp.h[i].branch);
    free(hp.h);
    free(bestOpt);
}

/* ---- incremental-branch-and-cut.ts:28-107: StateCheckpoint / createCheckpoint / restoreCheckpoint ---- */
typedef struct {
    int W, H, nVars, lastElementIndex, feasible, refs, mapLen;
    double evaluation;
    double *M;
    int *vrow, *vcol, *rowOf, *colOf;
} orc_checkpoint;

static orc_checkpoint *checkpoint_create(const orc_tab *t) {
    orc_checkpoint *c = (orc_checkpoint *)calloc(1, sizeof(orc_checkpoint));
    c->W = t->W; c->H = t->H; c->nVars = t->nVars; c->lastElementIndex = t->lastElementIndex;
    c->feasible = t->feasible; c->evaluation = t->evaluation; c->refs = 0;
    c->M = (double *)malloc(sizeof(double) * (size_t)t->H * t->W);
    memcpy(c->M, t->M, sizeof(double) * (size_t)t->H * t->W);
    c->vrow = (int *)malloc(sizeof(int) * t->H);
    memcpy(c->vrow, t->vrow, sizeof(int) * t->H);
    c->vcol = (int *)malloc(sizeof(int) * t->W);
    memcpy(c->vcol, t->vcol, sizeof(int) * t->W);
    c->mapLen = t->mapCap;
    c->rowOf = (int *)malloc(sizeof(int) * t->mapCap);
    c->colOf = (int *)malloc(sizeof(int) * t->mapCap);
    memcpy(c->rowOf, t->rowOf, sizeof(int) * t->mapCap);
    memcpy(c->colOf, t->colOf, sizeof(int) * t->mapCap);
    return c;
}
static void checkpoint_release(orc_checkpoint *c) {
    if (!c || --c->refs > 0) return;
    free(c->M); free(c->vrow); free(c->vcol); free(c->rowOf); free(c->colOf); free(c);
}
/* :73-107: the index maps are restored for indices < checkpoint.nVars only; later entries keep what they hold */
static void checkpoint_restore(orc_tab *t, const orc_checkpoint *c) {
    ensure_rows(t, c->H);
    memcpy(t->M, c->M, sizeof(double) * (size_t)c->H * c->W);
    t->W = c->W; t->H = c->H; t->nVars = c->nVars;
    memcpy(t->vrow, c->vrow, sizeof(int) * c->H);
    memcpy(t->vcol, c->vcol, sizeof(int) * c->W);
    ensure_maps(t, c->nVars);
    for (int i = 0; i < c->nVars && i < c->mapLen; i++) { t->rowOf[i] = c->rowOf[i]; t->colOf[i] = c->colOf[i]; }
    t->lastElementIndex = c->lastElementIndex;
    t->evaluation = c->evaluation;
    t->feasible = c->feasible;
}

static void checkpoint_release_v(void *c) { checkpoint_release((orc_checkpoint *)c); }

/* ---- enhanced-branch-and-cut.ts ---- */
typedef struct { double upSum, downSum; long upCount, downCount; } pseudo_cost;
typedef struct { int index; double value, fraction; } frac_cand;

/* :94-108 */
static double pc_score(const pseudo_cost *d, double fraction) {
    const double upPseudo = d->upCount > 0 ? d->upSum / d->upCount : 1;
    const double downPseudo = d->downCount > 0 ? d->downSum / d->downCount : 1;
    const double upEstimate = upPseudo * (1 - fraction);
    const double downEstimate = downPseudo * fraction;
    const double a = upEstimate > 1e-6 ? upEstimate : (upEstimate != upEstimate ? upEstimate : 1e-6);     /* Math.max(x, 1e-6) */
    const double b = downEstimate > 1e-6 ? downEstimate : (downEstimate != downEstimate ? downEstimate : 1e-6);
    return a * b;
}

/* stable insertion sort by fraction descending == Array.prototype.sort((a, b) => b.fraction - a.fraction) */
static void sort_by_fraction_desc(frac_cand *c, int n) {
    for (int i = 1; i < n; i++) {
        frac_cand x = c[i];
        int j = i - 1;
        while (j >= 0 && c[j].fraction < x.fraction) { c[j + 1] = c[j]; j--; }
        c[j + 1] = x;
    }
}

/* :110-195; branching: 1 = most-fractional, 2 = pseudocost, 3 = strong.  Returns var index or -1. */
static int enh_select_branching_variable(orc_tab *t, pseudo_cost *pc, int branching, int strongCandidates, double *val) {
    frac_cand *cand = (frac_cand *)malloc(sizeof(frac_cand) * (size_t)(t->nInt > 0 ? t->nInt : 1));
    int n = 0;
    for (int v = 0; v < t->nInt; v++) {
        const int varIndex = t->intVars[v];
        const int row = t->rowOf[varIndex];
        if (row != -1) {
            const double value = t->M[(size_t)row * t->W];
            const double fraction = fabs(value - js_round(value));
            if (fraction > t->precision) { cand[n].index = varIndex; cand[n].value = value; cand[n].fraction = fraction; n++; }
        }
    }
    int sel = -1;
    if (n > 0) {
        frac_cand best = cand[0];
        if (branching == 1) {
            sort_by_fraction_desc(cand, n);
            best = cand[0];
        } else if (branching == 2) {
            double bestScore = -INFINITY;
            for (int i = 0; i < n; i++) {
                const double score = pc_score(&pc[cand[i].index], cand[i].fraction);
                if (score > bestScore) { bestScore = score; best = cand[i]; }
            }
        } else if (branching == 3) {
            sort_by_fraction_desc(cand, n);
            if (n > strongCandidates) n = strongCandidates;
            double bestScore = -INFINITY;
            best = cand[0];
            for (int i = 0; i < n; i++) {
                const pseudo_cost *d = &pc[cand[i].index];
                double score;
                if (d->upCount >= 2 && d->downCount >= 2) score = pc_score(d, cand[i].fraction);
                else score = cand[i].fraction * (1 - cand[i].fraction);
                if (score > bestScore) { bestScore = score; best = cand[i]; }
            }
        }
        sel = best.index;
        *val = best.value;
    }
    free(cand);
    return sel;
}

/* :197-221 */
static void enh_apply_cuts(orc_tab *t, const orc_cut *cuts, int n) {
    orc_restore(t);
    orc_add_cuts(t, cuts, n);
    orc_simplex(t);
    if (t->useMIR && t->feasible) {
        int improved = 1, mirIterations = 0;
        const int maxMIRIterations = 3;
        while (improved && mirIterations < maxMIRIterations) {
            const double before = orc_fractional_volume(t, 1);
            orc_apply_mir_cuts(t);
            orc_simplex(t);
            const double after = orc_fractional_volume(t, 1);
            mirIterations++;
            if (after >= 0.9 * before) improved = 0;
        }
    }
}

/* :223-434.  nodeSelection: 1 = best-first, 2 = depth-first, 3 = hybrid; branching as above.  One service instance per
 * call (main.ts:62-83 creates a fresh one per Solve), so the pseudocosts start empty. */
void orc_enhanced_branch_and_cut2(orc_tab *t, int nodeSelection, int branching, int strongCandidates, int incremental, int maxCheckpoints);
void orc_enhanced_branch_and_cut(orc_tab *t, int nodeSelection, int branching, int strongCandidates) {
    orc_enhanced_branch_and_cut2(t, nodeSelection, branching, strongCandidates, 0, 0);
}
/* incremental != 0: createIncrementalBranchAndCutService (incremental-branch-and-cut.ts:128-499) -- the same loop with
 * parent checkpoints: a depth-first child restores its parent's solved tableau and adds only its new cut (at most
 * maxCheckpoints checkpoints per call, :435-438), pseudocosts are fed by `newCut` (:353-362), "strong" means pseudocost. */
void orc_enhanced_branch_and_cut2(orc_tab *t, int nodeSelection, int branching, int strongCandidates, int incremental, int maxCheckpoints) {
    int checkpointCount = 0;
    if (incremental && branching == 3) branching = 2;
    minheap hp = {0, 0, 0, 0};
    orc_branch **stack = 0;
    long sp = 0, scap = 0;
    int iterations = 0;
    const double tolerance = t->tolerance;
    int toleranceFlag = 1;
    double bestEvaluation = INFINITY;
    orc_branch *bestBranch = 0;
    const int nOpt = t->nOpt;
    double *bestOpt = (double *)malloc(sizeof(double) * (nOpt > 0 ? nOpt : 1));
    for (int o = 0; o < nOpt; o++) bestOpt[o] = INFINITY;
    const int pcN = t->mapCap + 64;
    pseudo_cost *pc = (pseudo_cost *)calloc((size_t)pcN, sizeof(pseudo_cost));
    const int switchToBestFirstAfterSolutions = 1;
    int solutionsFound = 0;
    int useDepthFirst = nodeSelection == 2 || nodeSelection == 3;
#define STACK_PUSH(b) do { if (sp == scap) { scap = scap ? scap * 2 : 64; stack = (orc_branch **)realloc(stack, sizeof(orc_branch *) * scap); } stack[sp++] = (b); } while (0)
    if (useDepthFirst) STACK_PUSH(make_branch(-INFINITY, 0)); else heap_push(&hp, make_branch(-INFINITY, 0));

    while ((useDepthFirst ? sp > 0 : hp.size > 0) && toleranceFlag) {
        if (t->maxNodes > 0 && iterations >= t->maxNodes) break;
        const double acceptableThreshold = t->isMin ? t->bestPossibleEval * (1 + tolerance) : t->bestPossibleEval * (1 - tolerance);
        if (tolerance > 0 && bestEvaluation < acceptableThreshold) toleranceFlag = 0;
        orc_branch *active;
        if (useDepthFirst && sp > 0) active = stack[--sp];
        else if (hp.size > 0) active = heap_pop(&hp);
        else break;
        if (active->relaxedEvaluation > bestEvaluation) { free_branch(active); continue; }
        const double parentEval = t->evaluation;
        const long pivBefore = t->totalPivots;
        if (incremental && active->parentCheckpoint && active->hasNewCut) {  /* applyIncrementalCuts :253-261 */
            checkpoint_restore(t, (const orc_checkpoint *)active->parentCheckpoint);
            orc_add_cuts(t, &active->newCut, 1);
            orc_simplex(t);
            if (t->useMIR && t->feasible) {
                int improved = 1, mirIterations = 0;
                while (improved && mirIterations < 3) {
                    const double before = orc_fractional_volume(t, 1);
                    orc_apply_mir_cuts(t);
                    orc_simplex(t);
                    const double after = orc_fractional_volume(t, 1);
                    mirIterations++;
                    if (after >= 0.9 * before) improved = 0;
                }
            }
        } else {
            enh_apply_cuts(t, active->cuts, active->nCuts);
        }
        iterations++;
        double *nl = 0;
        if (t->nlog && t->nlogN < t->nlogCap) {
            nl = t->nlog + 8 * t->nlogN++;
            nl[0] = iterations; nl[1] = active->nCuts; nl[2] = t->feasible;
            nl[3] = t->evaluation; nl[4] = -1; nl[5] = -1; nl[6] = 0;
            nl[7] = (double)(t->totalPivots - pivBefore);
        }
        if (!t->feasible) { free_branch(active); continue; }
        const double evaluation = t->evaluation;
        if (evaluation > bestEvaluation) { free_branch(active); continue; }
        if ((incremental ? active->hasNewCut : active->nCuts > 0) && parentEval != 0) {  /* :281-294 / incremental :353-362 */
            const orc_cut lastCut = incremental ? active->newCut : active->cuts[active->nCuts - 1];
            const double improvement = fabs(evaluation - parentEval);
            const double fraction = 0.5;
            if (lastCut.varIndex >= 0 && lastCut.varIndex < pcN) {
                pseudo_cost *d = &pc[lastCut.varIndex];
                const int up = lastCut.type == 0;
                const double normalizedImprovement = improvement / (up ? 1 - fraction : fraction);
                if (up) { d->upSum += normalizedImprovement; d->upCount++; }
                else { d->downSum += normalizedImprovement; d->downCount++; }
            }
        }
        if (evaluation == bestEvaluation) {
            int worse = 1;
            for (int o = 0; o < nOpt; o++) {
                const double v = t->optRC[(size_t)o * t->W];
                if (v > bestOpt[o]) break;
                else if (v < bestOpt[o]) { worse = 0; break; }
            }
            if (worse) { free_branch(active); continue; }
        }
        if (orc_is_integral(t)) {
            if (nl) nl[4] = 1;
            t->isIntegralFlag = 1;
            solutionsFound++;
            if (iterations == 1) { t->bncIterations = iterations; free_branch(active); goto done; }
            if (bestBranch) free_branch(bestBranch);
            bestBranch = active;
            bestEvaluation = evaluation;
            for (int o = 0; o < nOpt; o++) bestOpt[o] = t->optRC[(size_t)o * t->W];
            if (nodeSelection == 3 && solutionsFound >= switchToBestFirstAfterSolutions) {
                useDepthFirst = 0;
                while (sp > 0) heap_push(&hp, stack[--sp]);
            }
        } else {
            if (nl) nl[4] = 0;
            if (iterations == 1) orc_save(t);
            double varValue = 0;
            const int varIndex = enh_select_branching_variable(t, pc, branching, strongCandidates, &varValue);
            if (varIndex < 0) { free_branch(active); continue; }
            if (nl) { nl[5] = varIndex; nl[6] = varValue; }
            orc_branch *high = make_branch(evaluation, active->nCuts + 1);
            orc_branch *low = make_branch(evaluation, active->nCuts + 1);
            for (int c = 0; c < active->nCuts; c++) {
                const orc_cut cut = active->cuts[c];
                if (cut.varIndex == varIndex) {
                    if (cut.type == 0) low->cuts[low->nCuts++] = cut;
                    else high->cuts[high->nCuts++] = cut;
                } else {
                    high->cuts[high->nCuts++] = cut;
                    low->cuts[low->nCuts++] = cut;
                }
            }
            orc_cut ch = {0, varIndex, ceil(varValue)};
            orc_cut cl = {1, varIndex, floor(varValue)};
            high->cuts[high->nCuts++] = ch;
            low->cuts[low->nCuts++] = cl;
            if (incremental && useDepthFirst) {  /* incremental :435-438,476-483 */
                orc_checkpoint *cp = 0;
                if (checkpointCount < maxCheckpoints) { cp = checkpoint_create(t); checkpointCount++; }
                low->parentCheckpoint = cp; low->newCut = cl; low->hasNewCut = 1;
                high->parentCheckpoint = cp; high->newCut = ch; high->hasNewCut = 1;
                if (cp) cp->refs = 2;
            }
            if (useDepthFirst) { STACK_PUSH(low); STACK_PUSH(high); }
            else { heap_push(&hp, high); heap_push(&hp, low); }
            free_branch(active);
        }
    }
    if (bestBranch) {
        enh_apply_cuts(t, bestBranch->cuts, bestBranch->nCuts);
        free(t->bestCuts);
        t->bestCuts = (orc_cut *)malloc(sizeof(orc_cut) * (bestBranch->nCuts > 0 ? bestBranch->nCuts : 1));
        memcpy(t->bestCuts, bestBranch->cuts, sizeof(orc_cut) * bestBranch->nCuts);
        t->nBestCuts = bestBranch->nCuts;
        free_branch(bestBranch);
    }
    t->bncIterations = iterations;
done:
    for (long i = 0; i < hp.size; i++) free_branch(hp.h[i].branch);
    for (long i = 0; i < sp; i++) free_branch(stack[i]);
    free(hp.h); free(stack); free(bestOpt); free(pc);
#undef STACK_PUSH
}

/* ---- read-back ---- */
typedef struct {
    int32_t width, height, nVars, lastElementIndex;
    int32_t feasible, bounded, simplexIters, unboundedVar;
    int32_t isIntegral, bncIterations, cyclePhase, cycleStart, cycleLen, nBestCuts;
    int64_t totalPivots, lastP1, lastP2, plogN, nlogN;
    double evaluation, bestPossibleEval;
} orc_state;

void orc_get_state(const orc_tab *t, orc_state *s) {
    s->width = t->W; s->height = t->H; s->nVars = t->nVars; s->lastElementIndex = t->lastElementIndex;
    s->feasible = t->feasible; s->bounded = t->bounded; s->simplexIters = t->simplexIters;
    s->unboundedVar = t->unboundedVar; s->isIntegral = t->isIntegralFlag;
    s->bncIterations = t->bncIterations; s->cyclePhase = t->cyclePhase;
    s->cycleStart = t->cycleStart; s->cycleLen = t->cycleLen; s->nBestCuts = t->nBestCuts;
    s->totalPivots = t->totalPivots; s->lastP1 = t->lastP1; s->lastP2 = t->lastP2;
    s->plogN = t->plogN; s->nlogN = t->nlogN;
    s->evaluation = t->evaluation; s->bestPossibleEval = t->bestPossibleEval;
}

void orc_get_matrix(const orc_tab *t, double *out) { memcpy(out, t->M, sizeof(double) * (size_t)t->H * t->W); }
void orc_get_flat(const orc_tab *t, double *out, long n) { memcpy(out, t->M, sizeof(double) * (size_t)n); }
void orc_get_maps(const orc_tab *t, int *vrow, int *vcol) {
    memcpy(vrow, t->vrow, sizeof(int) * t->H);
    memcpy(vcol, t->vcol, sizeof(int) * t->W);
}
int orc_row_of(const orc_tab *t, int varIndex) { return varIndex < t->mapCap ? t->rowOf[varIndex] : -1; }
void orc_get_optional(const orc_tab *t, double *out) {
    if (t->nOpt > 0) memcpy(out, t->optRC, sizeof(double) * (size_t)t->nOpt * t->W);
}
void orc_get_pivot_log(const orc_tab *t, int *out) { memcpy(out, t->plog, sizeof(int) * 4 * (size_t)t->plogN); }
void orc_get_node_log(const orc_tab *t, double *out) { memcpy(out, t->nlog, sizeof(double) * 8 * (size_t)t->nlogN); }
void orc_get_best_cuts(const orc_tab *t, orc_cut *out) { memcpy(out, t->bestCuts, sizeof(orc_cut) * t->nBestCuts); }
void orc_set_pivot_limit(orc_tab *t, long limit) { t->pivotLimit = limit; t->truncated = 0; }
int orc_truncated(const orc_tab *t) { return t->truncated; }
void orc_set_flags(orc_tab *t, int feasible, int bounded) { t->feasible = feasible; t->bounded = bounded; }
