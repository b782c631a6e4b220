/*
 * include/jslp_b200.h -- C ABI of libjslp_b200.so, the H100-native (sm_90a) drop-in for
 * jsLPSolver's dense-tableau simplex + branch-and-cut hot path.
 *
 * The reference (JWally/jsLPSolver, TypeScript) has no FFI of its own: its plug-in seam is the
 * `Tableau` method table plus the injected `BranchAndCutService` (SURVEY.md 8b).  Every entry
 * point below replaces exactly one member of that seam; an N-API addon (INTEGRATION.md) binds
 * them 1:1 from a `GpuTableau extends Tableau` subclass.  Plain pointers and sizes only.
 *
 * Conventions (mirroring the reference, SURVEY.md 8b "Conventions"):
 *   - every function returns 0 on success, a negative JSLP_E_* on misuse/driver failure;
 *     solver outcomes (infeasible / unbounded / cycle) are FLAGS in the status structs, never
 *     error codes (the reference never throws for them);
 *   - not thread-safe per handle, thread-safe across handles; one context per GPU;
 *   - all matrices are row-major fp64, stride == width, row 0 = cost row, column 0 = RHS
 *     (tableau.ts:49-54,304); index maps are int32 with -1 = "not there" (tableau.ts:306-316);
 *   - there is NO CPU fallback: without a CUDA device every call fails with JSLP_E_CUDA.
 */
#ifndef JSLP_B200_H
#define JSLP_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define JSLP_OK 0
#define JSLP_E_INVALID (-1)   /* bad argument / bad handle state            */
#define JSLP_E_CUDA (-2)      /* CUDA driver/runtime failure (see last_error) */
#define JSLP_E_CAPACITY (-3)  /* row capacity / shared-memory capacity exceeded */
#define JSLP_E_UNSUPPORTED (-4) /* feature outside the hot-path scope (e.g. useMIRCuts) */

typedef struct jslp_ctx jslp_ctx;
typedef struct jslp_tab jslp_tab;

/* Thread-local description of the last failure (never NULL). */
const char *jslp_last_error(void);
/* ABI version, bumped on any signature change. */
int jslp_abi_version(void);

/* One context per GPU.  `stream` is a cudaStream_t (as void*) the library launches on, or NULL
 * for a private non-blocking stream.  Replaces: nothing (the reference has no device). */
int jslp_ctx_create(int device, void *stream, jslp_ctx **out);
void jslp_ctx_destroy(jslp_ctx *ctx);
/* The stream all work of this context is enqueued on (cudaStream_t as void*). */
void *jslp_ctx_stream(jslp_ctx *ctx);
/* Number of kernel launches issued by this context so far (bench.py's gpu_launches). */
int64_t jslp_ctx_launches(jslp_ctx *ctx);
int jslp_ctx_sync(jslp_ctx *ctx);

/* Replaces Tableau.initialize (tableau.ts:292-317): allocates a device tableau of `width` x
 * `height` with room for `row_capacity` >= height rows (branching cuts append rows,
 * cutting-strategies.ts:24-34).  `precision` is Tableau.precision (default 1e-8, tableau.ts:96). */
int jslp_tab_create(jslp_ctx *ctx, int width, int height, int row_capacity, double precision,
                    jslp_tab **out);
void jslp_tab_destroy(jslp_tab *tab);

/* Replaces the result of Tableau._resetMatrix / setModel (tableau.ts:319-391): uploads the
 * initial tableau built by the (unchanged) host front end.
 *   matrix            height*width doubles, row-major, stride == width
 *   var_index_by_row  height int32 (entry 0 == -1)          (tableau.ts:63)
 *   var_index_by_col  width  int32 (entry 0 == -1)          (tableau.ts:64)
 *   unrestricted      n_index bytes, 1 = Tableau.unrestrictedVars[index] === true, or NULL
 *   n_index           width + height - 2 (= Tableau.nVars)
 *   int_var_indices   model.integerVariables[].index in model order (mip-utils.ts:47,108), or NULL
 *   n_opt, opt_obj    optionalObjectives sorted by priority; n_opt*width reducedCosts
 *                     (tableau.ts:278-290), or 0/NULL
 * All host pointers may be pageable or pinned; the copy is synchronous w.r.t. the host.  */
int jslp_tab_upload(jslp_tab *tab, const double *matrix, const int32_t *var_index_by_row,
                    const int32_t *var_index_by_col, const uint8_t *unrestricted, int n_index,
                    const int32_t *int_var_indices, int n_int, int n_opt, const double *opt_obj);

/* Solver options that the reference keeps on Model / Tableau. */
enum {
    JSLP_OPT_ENGINE = 1,       /* 0 = auto (resident when H*W <= 16384, else fused), 1 = two-kernel
                                  (select + update), 2 = fused step, 4 = single-CTA resident    */
    JSLP_OPT_BATCH = 2,        /* pivots enqueued per host poll (default 256)              */
    JSLP_OPT_PIVOT_LOG_CAP = 3, /* keep a host-side (row,col,leaving,entering) log, 0 = off */
    /* tuning / diagnostics of the fused pivot step (no effect on results) */
    JSLP_OPT_STEP_VARIANT = 4, /* kernel instantiation: threads, occupancy, rows per pass, prefetch; -1 = auto */
    JSLP_OPT_GRID_PER_SM = 5,  /* CTAs per SM of the fused step, 0 = the variant's default        */
    JSLP_OPT_LOOKAHEAD = 6,    /* 1 (default) = look-ahead ratio test, 0 = generic serial tail    */
    JSLP_OPT_TIMELINE = 7,     /* record a per-CTA timeline for the first N launches of a solve   */
    JSLP_OPT_PDL = 8,          /* 1 = chain the fused steps with programmatic dependent launch    */
    JSLP_OPT_PINGPONG = 9,     /* 1 (default) = ping-pong tableau + two selector CTAs, 0 = in place */
    /* branch-and-cut nodes too large for shared memory (no effect on results) */
    JSLP_OPT_NODE_SLOTS = 10,  /* node LPs in flight side by side in HBM: -1 = auto (default), 0 = one at a
                                  time (the reference's literal applyCuts sequence), n = at most n slots */
    JSLP_OPT_SLOT_STEPS = 11,  /* pivots per slot between host polls of the slot batch (default 32)   */
    JSLP_OPT_SLOT_VARIANT = 12, /* kernel instantiation used by the slot batch (JSLP_OPT_STEP_VARIANT values) */
    JSLP_OPT_NODE_LOG_CAP = 14, /* pivot-log entries per node LP of the shared-memory node kernel (default 512); a node
                                   that needs more is re-evaluated on the HBM path (tests lower it to hit that path) */
    JSLP_OPT_USE_MIR_CUTS = 13  /* model.useMIRCuts (model.ts:69,313): applyCuts / branchAndCut run the MIR loop of
                                   branch-and-cut.ts:38-51 after every node's simplex()                          */
};
int jslp_tab_set_option(jslp_tab *tab, int key, double value);
/* Diagnostics: per-CTA timeline (8 int64 per CTA per launch) recorded under JSLP_OPT_TIMELINE. */
int jslp_debug_timeline(jslp_tab *tab, int64_t *out, int64_t cap_values, int *launches, int *grid);
/* Diagnostics: bandwidth [GB/s, read + write] of the library's own 128-bit copy loop ping-ponging between two
 * buffers of `bytes` each, `iters` round trips -- with 2 * bytes below the L2 size this is the L2-resident roof
 * the in-solve streaming phase runs under, above it the HBM roof (bench.py reports both beside roofline.frac). */
int jslp_debug_copy_gbs(jslp_ctx *ctx, int64_t bytes, int iters, double *gbs);

/* Tableau state read by callers after simplex() (SURVEY.md 8b "State contract"). */
typedef struct {
    int32_t feasible;            /* Tableau.feasible                                     */
    int32_t bounded;             /* Tableau.bounded                                      */
    int32_t cycled;              /* 0, or the phase (1/2) in which checkForCycles fired  */
    int32_t cycle_start;         /* model.messages "Start :"                             */
    int32_t cycle_length;        /* model.messages "Length :"                            */
    int32_t phase1_pivots;       /* return value of Tableau.phase1()                     */
    int32_t phase2_pivots;       /* return value of Tableau.phase2()                     */
    int32_t unbounded_var_index; /* Tableau.unboundedVarIndex, -1 = null                 */
    int32_t simplex_iters;       /* Tableau.simplexIters                                 */
    int32_t width, height;       /* current logical size                                 */
    int32_t engine;              /* engine that actually ran (JSLP_OPT_ENGINE values)    */
    double evaluation_raw;       /* matrix[0] at exit                                    */
    double evaluation;           /* Tableau.evaluation (setEvaluation rounding, tableau.ts:420-430) */
    double best_possible_eval;   /* Tableau.bestPossibleEval                             */
    double gpu_ms;               /* CUDA-event time of the solve on the context stream   */
    int64_t kernel_launches;     /* launches issued for this call                        */
} jslp_lp_status;

/* == Tableau.simplex() (tableau.ts:103-111 -> simplex.ts:14-23): phase1, then phase2 if
 * feasible.  check_cycles == model.checkForCycles (model.ts:73,359-363).                 */
int jslp_simplex(jslp_tab *tab, int check_cycles, jslp_lp_status *out);
/* == Tableau.phase1() / phase2() (simplex.ts:25-98 / 100-325). */
int jslp_phase1(jslp_tab *tab, int check_cycles, jslp_lp_status *out);
int jslp_phase2(jslp_tab *tab, int check_cycles, jslp_lp_status *out);
/* == Tableau.pivot(row, col) (simplex.ts:330-413). */
int jslp_pivot(jslp_tab *tab, int row, int col);

/* == Tableau.save() / restore() (backup.ts:49-105): device-side snapshot, D2D restore. */
int jslp_save(jslp_tab *tab);
int jslp_restore(jslp_tab *tab);

/* BranchCut (types.ts:17-21). type: 0 = "min" (x >= value), 1 = "max" (x <= value). */
typedef struct {
    int32_t type;
    int32_t var_index;
    double value;
} jslp_cut;

/* == Tableau.addCutConstraints(cuts) (cutting-strategies.ts:16-72). */
int jslp_add_cuts(jslp_tab *tab, const jslp_cut *cuts, int n);
/* == Tableau.addLowerBoundMIRCut(row) (upper_bound = 0) / addUpperBoundMIRCut(row) (1), cutting-strategies.ts:
 * 74-196: *added = 1 when a cut row (and its slack) was appended.  == Tableau.applyMIRCuts() (198-212): lower-
 * bound cuts on the first (at most 10) eligible rows.  == Tableau.computeFractionalVolume (mip-utils.ts:67-98). */
int jslp_add_mir_cut(jslp_tab *tab, int row, int upper_bound, int *added);
int jslp_apply_mir_cuts(jslp_tab *tab, int *n_added);
int jslp_fractional_volume(jslp_tab *tab, int ignore_integer_values, double *volume);
/* == BranchAndCutService.applyCuts (branch-and-cut.ts:33-52): restore, add cuts, simplex [, MIR loop]. */
int jslp_apply_cuts(jslp_tab *tab, const jslp_cut *cuts, int n, int check_cycles, jslp_lp_status *out);
/* == Tableau.isIntegral() (mip-utils.ts:43-61) and getMostFractionalVar() (mip-utils.ts:100-126):
 * *var_index = -1 when no fractional integer variable exists.                             */
int jslp_is_integral(jslp_tab *tab, int *is_integral);
int jslp_most_fractional(jslp_tab *tab, int32_t *var_index, double *value);

/* The dynamic-modification API on the device-resident tableau (dynamic-modification.ts:16-55,78-316): edits after a
 * solve without rebuilding / re-uploading it.  Constraints and variables are named by their element index
 * (Constraint.index == its slack's index, Variable.index); availableIndexes and the Constraint / Variable objects stay
 * host bookkeeping.  opt_slot: -1 = priority 0 (cost row), k = the k-th uploaded optional objective.
 *   put_in_base / take_out_of_base   == Tableau.putInBase / takeOutOfBase (may pivot); *row / *col = where it ended
 *   update_rhs                       == updateRightHandSide(constraint, difference)
 *   update_coefficient               == updateConstraintCoefficient(constraint, variable, difference)
 *   update_cost                      == updateCost(variable, difference)
 *   add_constraint / remove_constraint == addConstraint(constraint) / removeConstraint(constraint); terms in order
 *   add_variable / remove_variable   == addVariable(variable) / removeVariable(variable); cost_entry is the signed
 *                                       cost-row entry (isMinimization ? -cost : cost)                            */
int jslp_put_in_base(jslp_tab *tab, int var_index, int *row);
int jslp_take_out_of_base(jslp_tab *tab, int var_index, int *col);
int jslp_update_rhs(jslp_tab *tab, int constraint_index, double difference);
int jslp_update_coefficient(jslp_tab *tab, int constraint_index, int var_index, double difference);
int jslp_update_cost(jslp_tab *tab, int var_index, int opt_slot, double difference);
int jslp_add_constraint(jslp_tab *tab, int is_upper_bound, double rhs, int slack_index, const int32_t *term_var,
                        const double *term_coef, int n_terms);
int jslp_remove_constraint(jslp_tab *tab, int slack_index);
int jslp_add_variable(jslp_tab *tab, int var_index, double cost_entry, int opt_slot, int is_integer, int is_unrestricted);
/* Tableau's scalar bookkeeping for the host mirror: {width, height, nVars, lastElementIndex, row stride, row capacity} */
int jslp_tab_info(jslp_tab *tab, int32_t *out6);
int jslp_remove_variable(jslp_tab *tab, int var_index);

/* Read-back for updateVariableValues / generateSolutionSet / getSolution
 * (dynamic-modification.ts:57-76, solution.ts:35-60).  Any pointer may be NULL.
 *   matrix     height*width doubles (stride == width)   rhs_col   height doubles
 *   cost_row   width doubles                             opt_obj   n_opt*width doubles   */
int jslp_download(jslp_tab *tab, double *matrix, double *rhs_col, double *cost_row,
                  int32_t *var_index_by_row, int32_t *var_index_by_col, double *opt_obj,
                  int32_t *width, int32_t *height);
/* Drains the host-side pivot log: 4 int32 per pivot (row, col, leaving var, entering var). */
int jslp_pivot_log(jslp_tab *tab, int32_t *entries, int cap, int *n);

/* Ratio-test bounds of the current tableau for the sensitivity report of a solved LP (no reference counterpart;
 * DESIGN.md section 2b).  One device pass over rows 1 .. height-1; the tableau, the index maps and the pivot record are
 * left unchanged.  With P = precision and only rows / columns as stated taking part:
 *   col_lo[c] / col_hi[c]  width doubles: max / min of -M[r,0] / M[r,c] over rows whose basic variable is restricted
 *                          and M[r,c] > P / M[r,c] < -P
 *   row_lo[r] / row_hi[r]  height doubles: max / min of M[0,c] / M[r,c] over restricted columns c >= 1 with
 *                          M[r,c] > P / M[r,c] < -P; an unrestricted column with |M[r,c]| > P contributes 0 to both
 * Quotients are normalised from -0 to +0 and NaN quotients are skipped; an empty set gives -inf (lo) / +inf (hi), as do row 0 and column 0.
 * Duals and reduced costs are the cost row itself (jslp_download's cost_row). */
int jslp_sensitivity(jslp_tab *tab, double *col_lo, double *col_hi, double *row_lo, double *row_hi);

/* Phase-1 feasibility of row subsets of the tableau's saved snapshot (jslp_save); no reference counterpart,
 * DESIGN.md section 2c.  keep: n_sets * height bytes, keep[s*height + r] = 1 keeps row r in set s (row 0 is
 * always kept).  verdict[s]: 0 = feasible, 1 = infeasible, 2 = undecided (cycle).  pivots[s] (may be NULL):
 * phase-1 pivots.  The cycle check is always on.  On return the tableau equals its snapshot. */
int jslp_feasibility_batch(jslp_tab *tab, const uint8_t *keep, int n_sets, int32_t *verdict, int32_t *pivots);

/* Parametric path of the current (optimal) tableau: one right-hand side (kind 0) or one cost (kind 1) moves from
 * theta0 to target, with one pivot per basis change (no reference counterpart; DESIGN.md section 2d).
 *   labels / signs  n_labels entries: the moved slack labels (1 or 2, in tableau row order) with sign g * s_i, or the
 *                   moved variable's label (1) with sign g * sigma; g = +1 when target >= theta0, s_i = +1 for a
 *                   `max` row and -1 for a `min` row, sigma = +1 for maximisation and -1 for minimisation
 *   max_breaks      at most this many pieces (>= 1); the output arrays hold max_breaks entries
 *   per piece k < *n_breaks:  theta[k] where it ends, obj_raw[k] = M[0,0] there, dobj[k] = the direction's objective
 *                   entry it moved along, rc_lbl[4k .. 4k+3] = pivot row, pivot column, leaving and entering label of
 *                   the basis change that ends it (-1 where there is none)
 *   stop            1 reached target, 2 infeasible beyond theta, 3 unbounded beyond theta, 4 max_breaks pieces
 *   end_rhs / end_vrow  height entries: column 0 and the row labels at the end of the path
 * The tableau, its labels, the staged pivot and the pivot record are restored before the call returns. */
int jslp_parametric(jslp_tab *tab, int kind, const int32_t *labels, const double *signs, int n_labels,
                    double theta0, double target, int max_breaks, double *theta, double *obj_raw, double *dobj,
                    int32_t *rc_lbl, int *n_breaks, int *stop, double *end_rhs, int32_t *end_vrow);

/* One edit of a what-if scenario: kind 0 = Tableau.updateRightHandSide(index, difference) of the constraint row with
 * slack index `index`, kind 1 = Tableau.updateCost(index, difference) of the priority-0 variable `index`
 * (dynamic-modification.ts:78-106,137-160).  `difference` is what setRightHandSide / setCost pass.                 */
typedef struct {
    int32_t kind;
    int32_t index;
    double difference;
} jslp_scenario_edit;

/* What-if scenarios on the current (solved) tableau, DESIGN.md section 2e.  Scenario s is edits[offsets[s] ..
 * offsets[s+1]) (every kind-0 edit before every kind-1 edit) applied in order to the current tableau, then simplex()
 * with check_cycles; each scenario starts from the current tableau.  Per scenario:
 *   status[s]     0 optimal, 1 infeasible, 2 unbounded, 3 cycled (the cycle check fired)
 *   eval_raw[s]   matrix[0][0] as simplex() left it (Tableau.evaluation before rounding, when optimal)
 *   p1[s], p2[s]  phase-1 / phase-2 pivots
 *   rhs, vrow     height entries each at s * height: the final right-hand-side column and varIndexByRow
 * The tableau, its labels, the staged pivot, the pivot record, the scalar Tableau state, the pivot log and the
 * jslp_save snapshot are as they were when the call returns.  No optional objectives. */
int jslp_scenario_batch(jslp_tab *tab, const jslp_scenario_edit *edits, const int32_t *offsets, int n_scenarios,
                        int check_cycles, int32_t *status, double *eval_raw, int32_t *p1, int32_t *p2, double *rhs,
                        int32_t *vrow);

/* The recourse LPs of one iteration of a two-stage stochastic LP, DESIGN.md section 2u.  Scenario s is
 * edits[offsets[s] .. offsets[s+1]) as jslp_scenario_batch runs it, with the cycle check on; status .. vrow are that
 * call's outputs, bit for bit, and so is the state on return.  Beyond them, per scenario:
 *   cert_rhs[s]  column 0 of the certificate row: row 0 when the scenario is optimal; when it is infeasible, the row
 *                phase 1 stopped at (column 0 below -precision, no entering column: a Farkas row); NaN otherwise
 *   alpha        n_first entries at s * n_first: alpha[j] = sum over i in increasing order of u[i] * tech[(ts * n_rows
 *                + i) * n_first + j] (unfused), ts = s when tech_per_case, else 0.  u[i] is the certificate row's
 *                multiplier of the row whose slack label is rows[i]: its entry when the label is non-basic, 1 or 0 when
 *                it is basic in or off the row; all 0 without a certificate.  tech holds each row's coefficients of the
 *                first-stage variables with the row's tableau sign (negated for a lower-bound row), so that column 0
 *                of the certificate row moves by -alpha . dx when the first stage moves by dx.
 * rows are distinct labels of the tableau, n_rows >= 0, n_first >= 0 (JSLP_E_INVALID otherwise).  No optional
 * objectives (JSLP_E_UNSUPPORTED). */
int jslp_recourse_batch(jslp_tab *tab, const jslp_scenario_edit *edits, const int32_t *offsets, int n_scenarios,
                        const int32_t *rows, int n_rows, const double *tech, int n_first, int tech_per_case,
                        int32_t *status, double *eval_raw, int32_t *p1, int32_t *p2, double *rhs, int32_t *vrow,
                        double *cert_rhs, double *alpha);

/* Warm-start crash, DESIGN.md section 2f: for each label enter[k] in order, pivot it into the basis on the row with the
 * largest |M[r,c]| among the rows r >= 1 whose basic label l has leave[l] != 0 and M[r,c] < -P || P < M[r,c] (lowest
 * row on ties); leave has one byte per label (n_index, see jslp_tab_info).  out[4k .. 4k+3] = (label, row, column,
 * leaving label) of a pivot, (label, row, -1, -2) when the label is already basic, (label, -1, column, -1) when no row
 * is eligible.  n_pivots = pivots done.  The tableau, labels and pivot record are left as the same jslp_pivot calls
 * would leave them; the crash pivots are not added to the pivot log.  No optional objectives. */
int jslp_crash(jslp_tab *tab, const int32_t *enter, int n_enter, const uint8_t *leave, int32_t *out, int *n_pivots);

/* Pareto frontier of two objectives from the current (optimal) tableau of the first, DESIGN.md section 2g: the second
 * objective's row is priced against the basis, then the weight theta of (1 - theta) * first + theta * second moves from
 * 0 to 1 with one pivot per basis change (the cost path of section 2d along the carried direction E = R2 - row 0).
 *   cost2_by_label  n_index entries (see jslp_tab_info): sigma2 * c2_j at each structural label, 0 elsewhere
 *   r2 / dir        width entries: the priced second objective R2 and the direction E at theta = 0
 *   theta .. rc_lbl, n_breaks, stop   the breakpoint records and the stop code as jslp_parametric writes them
 *                   (max_breaks entries; stop 1 reached theta = 1, 3 unbounded beyond theta, 4 max_breaks pieces)
 *   pt_rhs / pt_vrow / pt_break   per point k < min(n_points, max_points): column 0 and the row labels (height
 *                   entries each at k * height) and the number of records before it (0 = the start); a point is
 *                   appended after every pivot that changes column 0 (M[r*,0] != 0), and the last one is the end
 *   n_points        points on the whole path (may exceed max_points: call again with more room)
 *   end_rhs / end_vrow  height entries: column 0 and the row labels at the end of the path
 * The tableau, its labels, the staged pivot, the pivot record and the descriptor (no optional objectives) are restored
 * before the call returns.  No optional objectives. */
int jslp_frontier(jslp_tab *tab, const double *cost2_by_label, int max_breaks, int max_points, double *r2, double *dir,
                  double *theta, double *obj_raw, double *dobj, int32_t *rc_lbl, int *n_breaks, int *stop,
                  double *pt_rhs, int32_t *pt_vrow, int32_t *pt_break, int *n_points, double *end_rhs,
                  int32_t *end_vrow);

/* The optimal face of the current (optimal) tableau as a sibling tab in the same context, DESIGN.md section 2h: column
 * 0 and every column c >= 1 whose cost entry lies within the precision (M[0,c] >= -P && M[0,c] <= P) are kept, in
 * order; the face holds rows 1.. of those columns bit for bit under a cost row of +0, the row labels, the kept column
 * labels, and the parent's precision, unrestricted / integer tables, element indices and options.  Every vertex of the
 * face is an optimum of the parent, so any objective set on it with jslp_update_cost / jslp_scenario_batch is
 * optimised over the parent's optimal solutions.
 *   face       the new tab (free it with jslp_tab_destroy); NULL when only column 0 is kept (n_keep = 1)
 *   n_keep     kept columns W', column 0 included
 *   kept_cols  NULL, or room for width entries: the first n_keep receive the kept columns of the parent
 * The copy runs device to device; the parent is only read.  No optional objectives (JSLP_E_UNSUPPORTED). */
int jslp_face_create(jslp_tab *tab, jslp_tab **face, int32_t *n_keep, int32_t *kept_cols);

/* The current (optimal) tableau with its objective turned into a bound row, as a sibling tab in the same context,
 * DESIGN.md section 2i: with M the tableau (H x W) and l* = max(n_index, lastElementIndex), the new tab B is (H+1) x W
 * with the same stride; rows 1..H-1 are M's rows bit for bit, row 0 is +0 everywhere, and row H is B[H,0] = allowance,
 * B[H,c] = -M[0,c] (a sign flip) for c >= 1.  Its row labels are M's followed by l*, its column labels M's; precision,
 * unrestricted / integer tables (l* restricted, not integer), element indices and options are the parent's, with
 * lastElementIndex = l* + 1.  Every feasible point of B is a point of the parent at most `allowance` worse than the
 * optimum, so any objective set on it with jslp_update_cost / jslp_scenario_batch is optimised over those points.
 *   allowance  finite and >= 0 (JSLP_E_INVALID otherwise)
 *   bound      the new tab (free it with jslp_tab_destroy)
 * The copy runs device to device; the parent is only read.  No optional objectives (JSLP_E_UNSUPPORTED). */
int jslp_bound_create(jslp_tab *tab, double allowance, jslp_tab **bound);

/* One step of a lexicographic objective chain, DESIGN.md section 2j: the starting tableau of the next level from the
 * current (optimal) tableau, as a sibling tab in the same context.  With allowance == 0 it is jslp_face_create's face,
 * with allowance > 0 jslp_bound_create's bound tableau; in both, row 0 is the next objective priced against the
 * current basis instead of +0 -- R[c] = delta(c) + the section 2g block sums of -C[vrow[r]] * M[r,c] (jslp_frontier's
 * r2), taken at the kept columns of a face and at every column of a bound tableau, padding +0.  Every other element,
 * label, table and option is the face's or the bound tableau's.  Column 0 is the parent's (plus the allowance), so
 * the new tab starts primal feasible and jslp_simplex runs phase 2 only.
 *   cost_by_label  the next objective's row-0 entries by label (sigma * c_j at structural labels, 0 elsewhere), one
 *                  per label of tab (nVars of jslp_tab_info)
 *   allowance      finite and >= 0 (JSLP_E_INVALID otherwise)
 *   next           the new tab (free it with jslp_tab_destroy); NULL when a face keeps only column 0
 *   n_keep         W' (the tab's width for a bound tableau);  kept_cols (optional, W entries) the kept columns
 * The copy and row 0 stay on the device; the parent is only read.  No optional objectives (JSLP_E_UNSUPPORTED). */
int jslp_lex_next(jslp_tab *tab, const double *cost_by_label, double allowance, jslp_tab **next, int32_t *n_keep,
                  int32_t *kept_cols);

/* The elastic tableau of a possibly infeasible LP, DESIGN.md section 2k: a sibling tab in the same context in which
 * the relaxable rows r_1 < ... < r_k each get a violation column e_j (>= 0, in the constraint's own units) and row 0
 * is the weighted total violation sum_j w_j e_j.  With M the tab (H x W), P its precision and l* = max(n_index,
 * lastElementIndex), the new tab E is H x (W + k): column W+j enters row r_j as -1 (s.a.x <= s.rhs + e_j); a row with
 * M[r_j,0] < -P is crashed onto e_j (its entries sign-flipped, column 0 included; vrow[r_j] = l*+j and the slack's
 * label moves to column W+j); every other element of rows 1..H-1 is M's bit for bit, elastic entries of other rows
 * +0; row 0 is sum over crashed j of w_j * E[r_j,c] in the fixed order of section 2k, and -w_j at the elastic column
 * of a row that is not crashed.  The new labels are restricted and not integer; tables and options are the parent's.
 * Rows that start below -P may all be relaxed => E starts primal feasible and jslp_simplex runs phase 2 only.
 *   rows, weights  k increasing rows in 1..H-1 whose basic label is still the one they were uploaded with (the tab
 *                  as jslp_tab_upload left it), weights finite and > 0 (JSLP_E_INVALID otherwise)
 *   elastic        the new tab (free it with jslp_tab_destroy); JSLP_E_CAPACITY when W + k is beyond the width cap
 *   n_crashed      the number of crashed rows
 * The parent is only read; nothing but the crash count leaves the device.  No optional objectives (JSLP_E_INVALID). */
int jslp_elastic_create(jslp_tab *tab, const int32_t *rows, const double *weights, int n_rows, jslp_tab **elastic,
                        int32_t *n_crashed);

/* The recession cone of an LP, DESIGN.md section 2l: a sibling tab in the same context.  With M the tab (H x W, as
 * jslp_tab_upload left it) and l* = max(n_index, lastElementIndex), the new tab K is (H+1) x W: rows 0..H-1 are M's
 * rows bit for bit except column 0, which is +0 in every one of them; row H is 1.0 at column 0 and at every column
 * 1..W-1 (the normalisation sum_j d_j <= 1), +0 padding.  Its row labels are M's followed by l*, its column labels
 * M's; precision, unrestricted / integer tables (l* restricted, not integer), element indices and options are the
 * parent's, with lastElementIndex = l* + 1.  K's slack basis is primal feasible, and its optimum is non-zero exactly
 * when M has an improving direction d >= 0 (every row's activity rate at most 0 towards its bound).
 *   cone   the new tab (free it with jslp_tab_destroy)
 * The copy runs device to device; the parent is only read.  No optional objectives (JSLP_E_UNSUPPORTED). */
int jslp_cone_create(jslp_tab *tab, jslp_tab **cone);

/* simplex() (cycle check on) of column subsets of the saved snapshot, DESIGN.md section 2l: set i writes +0 over every
 * column c in 1..W-1 with keep_cols[i * W + c] == 0, in every row, row 0 included, and solves.  Sets whose tableau
 * fits shared memory run one CTA each in one launch; the others, and any set whose pivot log shows a cycle or that hits
 * the in-kernel pivot or log cap, run one after another on the single-tableau path (restore, zero, simplex).
 *   keep_cols      n_sets x W bytes, nonzero = keep (column 0 is always kept)
 *   status         per set: 0 optimal, 1 unbounded, 2 cycled (stopped before the pivot that completes the repeat),
 *                  3 infeasible (only when the snapshot does not start primal feasible)
 *   eval_raw       per set: the final M[0,0];  pivots: per set, phase-1 plus phase-2 pivots
 *   rhs, vrow      n_sets x H: the final column 0 and row labels of each set
 * Needs a snapshot (jslp_save); on return the tableau equals it, and the scalar Tableau state and executed-pivot log
 * are as they were.  No optional objectives (JSLP_E_UNSUPPORTED). */
int jslp_column_batch(jslp_tab *tab, const uint8_t *keep_cols, int n_sets, int32_t *status, double *eval_raw,
                      int32_t *pivots, double *rhs, int32_t *vrow);

/* One fixing of a solution-pool region: the non-basic column `column` (1..W-1) of the snapshot held at `value`. */
typedef struct {
    int32_t column;
    double value;
} jslp_fix;

/* The region LPs of a MIP solution-pool search, DESIGN.md section 2m.  Region i is the saved snapshot (the model's
 * initial tableau) with fixes[fix_offsets[i] .. fix_offsets[i+1]) applied in order -- M[r,0] = M[r,0] - value *
 * M[r,column], then M[r,column] = +0, for every row r, row 0 included -- then the cut rows cuts[cut_offsets[i] ..
 * cut_offsets[i+1]) appended as jslp_add_cuts appends them (labels from the snapshot's lastElementIndex), then
 * simplex() with check_cycles and the isIntegral / getMostFractionalVar scan.  Regions whose rows fit shared memory
 * run one CTA each in one launch; the others, and any region whose pivot log shows a cycle or that hits the in-kernel
 * pivot or log cap, run one after another on the single-tableau path.  Per region:
 *   status         0 optimal, 1 infeasible, 2 unbounded, 3 cycled (the cycle check fired)
 *   evaluation     Tableau.evaluation when optimal (M[0,0] rounded to the precision), -inf when unbounded, else 0
 *   is_integral    1 when optimal and every basic integer variable is integral
 *   branch_var / branch_value   getMostFractionalVar when optimal and not integral, else -1 / 0
 *   pivots         phase-1 plus phase-2 pivots
 *   rhs, vrow      row_stride entries each at i * row_stride; for an integral region the first H + n_cuts(i) hold the
 *                  final column 0 and row labels, otherwise they are not written
 * row_stride must be at least the snapshot's height plus every region's cut count.  Needs a snapshot (jslp_save); on
 * return the tableau equals it, and the scalar Tableau state and executed-pivot log are as they were.  No optional
 * objectives (JSLP_E_UNSUPPORTED). */
int jslp_pool_batch(jslp_tab *tab, const jslp_fix *fixes, const int32_t *fix_offsets, const jslp_cut *cuts,
                    const int32_t *cut_offsets, int n_nodes, int check_cycles, int row_stride, int32_t *status,
                    double *evaluation, int32_t *is_integral, int32_t *branch_var, double *branch_value,
                    int32_t *pivots, double *rhs, int32_t *vrow);

/* The node LPs of the bounding searches behind the near-optimal variability of a MIP, DESIGN.md section 2o.  Node i is
 * the saved snapshot (a bound tableau, jslp_bound_create) with the cost edits edits[edit_offsets[i] ..
 * edit_offsets[i+1]) applied in order as jslp_scenario_batch applies them (kind 1 = updateCost of the label `index`,
 * resolved against the snapshot's labels; every other kind is JSLP_E_INVALID), then the cut rows cuts[cut_offsets[i] ..
 * cut_offsets[i+1]) appended as jslp_add_cuts appends them (labels from the snapshot's lastElementIndex), then
 * simplex() with check_cycles and the isIntegral / getMostFractionalVar scan.  Nodes whose rows fit shared memory run
 * one CTA each in one launch; the others, and any node whose pivot log shows a cycle or that hits the in-kernel pivot
 * or log cap, run one after another on the single-tableau path.  The outputs are jslp_pool_batch's, per node:
 *   status         0 optimal, 1 infeasible, 2 unbounded, 3 cycled (the cycle check fired)
 *   evaluation     Tableau.evaluation when optimal (M[0,0] rounded to the precision), -inf when unbounded, else 0
 *   is_integral    1 when optimal and every basic integer variable is integral
 *   branch_var / branch_value   getMostFractionalVar when optimal and not integral, else -1 / 0
 *   pivots         phase-1 plus phase-2 pivots
 *   rhs, vrow      row_stride entries each at i * row_stride; for an integral node the first H + n_cuts(i) hold the
 *                  final column 0 and row labels, otherwise they are not written
 * row_stride must be at least the snapshot's height plus every node's cut count.  Needs a snapshot (jslp_save); on
 * return the tableau equals it, and the scalar Tableau state and executed-pivot log are as they were.  No optional
 * objectives (JSLP_E_UNSUPPORTED). */
int jslp_target_batch(jslp_tab *tab, const jslp_scenario_edit *edits, const int32_t *edit_offsets, const jslp_cut *cuts,
                      const int32_t *cut_offsets, int n_nodes, int check_cycles, int row_stride, int32_t *status,
                      double *evaluation, int32_t *is_integral, int32_t *branch_var, double *branch_value,
                      int32_t *pivots, double *rhs, int32_t *vrow);

/* The node LPs of the box searches behind the Pareto frontier of a two-objective MIP, DESIGN.md section 2s.  Node i is
 * the saved snapshot (the model's initial tableau with one bound row per objective) with the edits
 * edits[edit_offsets[i] .. edit_offsets[i+1]) applied in order as jslp_scenario_batch applies them (kind 0 =
 * updateRightHandSide of the slack label `index`, kind 1 = updateCost of the label `index`, both resolved against the
 * snapshot's labels; a node's kind-0 edits come before its kind-1 edits; any other kind is JSLP_E_INVALID), then the
 * cut rows cuts[cut_offsets[i] .. cut_offsets[i+1]) appended as jslp_add_cuts appends them (labels from the snapshot's
 * lastElementIndex), then simplex() with check_cycles and the isIntegral / getMostFractionalVar scan.  Routing, outputs,
 * row_stride and the state on return are jslp_target_batch's.  No optional objectives (JSLP_E_UNSUPPORTED). */
int jslp_box_batch(jslp_tab *tab, const jslp_scenario_edit *edits, const int32_t *edit_offsets, const jslp_cut *cuts,
                   const int32_t *cut_offsets, int n_nodes, int check_cycles, int row_stride, int32_t *status,
                   double *evaluation, int32_t *is_integral, int32_t *branch_var, double *branch_value,
                   int32_t *pivots, double *rhs, int32_t *vrow);

/* The node LPs of the feasibility searches behind a MIP conflict, DESIGN.md section 2n.  Node i is cost row 0 plus the
 * rows r >= 1 of the saved snapshot with keep[i * H + r] != 0 (H = the snapshot's height; row 0 is always kept), in
 * their original order, followed by the cut rows cuts[cut_offsets[i] .. cut_offsets[i+1]) appended as jslp_add_cuts
 * appends them (labels from the snapshot's lastElementIndex), then the reference's phase 1 with the cycle check on,
 * then the isIntegral / getMostFractionalVar scan over the integer variables whose position p in the model's integer
 * list has int_keep[i * n_int + p] != 0 (n_int = the number of integer variables; int_keep may be NULL when it is 0).
 * Nodes whose rows fit shared memory run one CTA each in one launch; the others, and any node that hits the in-kernel
 * pivot or log cap, run one after another on the single-tableau path.  Per node:
 *   status         0 feasible (phase 1 ended with no leaving row), 1 infeasible, 2 cycled (stopped before the pivot
 *                  that completes the repeat)
 *   is_integral    1 when feasible and every basic integer variable of the mask is integral
 *   branch_var / branch_value   the most fractional integer variable of the mask when feasible and not integral
 *                  (lowest position on ties), else -1 / 0
 *   pivots         phase-1 pivots
 *   rhs, vrow      row_stride entries each at i * row_stride; unless the node cycled, the first 1 + kept rows + cuts
 *                  hold the final column 0 and row labels, otherwise they are not written
 * row_stride must be at least every node's height (1 + kept rows + cuts).  Needs a snapshot (jslp_save); on return the
 * tableau equals it, and the scalar Tableau state and executed-pivot log are as they were.  No optional objectives
 * (JSLP_E_UNSUPPORTED). */
int jslp_conflict_batch(jslp_tab *tab, const uint8_t *keep, const uint8_t *int_keep, const jslp_cut *cuts,
                        const int32_t *cut_offsets, int n_nodes, int row_stride, int32_t *status, int32_t *is_integral,
                        int32_t *branch_var, double *branch_value, int32_t *pivots, double *rhs, int32_t *vrow);

/* Column `col` (0..W-1) of the current tableau, H doubles, into out: one strided device-to-host copy, so a single
 * column of a large tableau is read without downloading the whole of it. */
int jslp_column(jslp_tab *tab, int col, double *out);

/* Multi-GPU communicator of the branch-and-cut frontier (one process per GPU).  NCCL is loaded at run time;
 * without libnccl these calls fail with JSLP_E_UNSUPPORTED and single-GPU use is unaffected.  Rank 0 obtains a
 * 128-byte unique id and hands it to the other ranks through whatever bootstrap the host has (the N-API host:
 * its own IPC; the Python mirror: torch.distributed); every rank then creates its communicator.  Replaces
 * nothing in the reference (it is single-process); carries the two collectives of SURVEY.md 8e.  */
typedef struct jslp_comm jslp_comm;
int jslp_comm_unique_id(uint8_t *id128);
int jslp_comm_create(jslp_ctx *ctx, const uint8_t *id128, int rank, int n_ranks, jslp_comm **out);
void jslp_comm_destroy(jslp_comm *comm);
/* The collectives themselves (host buffers in and out, staged through device memory on the context stream):
 * in-place rank-major all-gather of bytes_per_rank bytes, element-wise all-reduce(min) of n doubles.       */
int jslp_comm_all_gather(jslp_comm *comm, void *buf, int64_t bytes_per_rank);
int jslp_comm_all_reduce_min(jslp_comm *comm, double *vals, int n);

/* == BranchAndCutService.branchAndCut (branch-and-cut.ts:54-199). */
typedef struct {
    double tolerance;        /* model.tolerance                                            */
    int32_t is_minimization; /* model.isMinimization                                       */
    int32_t check_cycles;    /* model.checkForCycles                                       */
    int32_t max_spec_batch;  /* nodes evaluated speculatively per round (1 = reference order,
                                one node at a time); results are committed in exact pop order */
    int32_t rank, n_ranks;   /* node sharding across GPUs; 0/1 = single GPU                */
    int64_t max_nodes;       /* safety cap on evaluated nodes, 0 = none                    */
    /* Multi-GPU exchange hook: all-gather `bytes` per rank (in-place, rank-major).  The host
     * layer implements it with torch.distributed/NCCL.  NULL when n_ranks <= 1.            */
    int (*all_gather)(void *user, void *buf, int64_t bytes_per_rank);
    void *user;
    jslp_comm *comm;        /* NCCL communicator: when set it carries the all-gather of node summaries and the
                               all-reduce(min) of the incumbent bound, and the hook above is ignored          */
    int32_t shard_policy;   /* 0 = auto: shard a round over the ranks only when its node LPs run in HBM (nodes
                               that fit shared memory cost less than a collective: every rank evaluates them
                               itself); 1 = shard every round                                                */
    int32_t keep_solutions; /* model.keep_solutions (branch-and-cut.ts:143-153): every incumbent is stored   */
    double timeout_ms;      /* model.timeout (branch-and-cut.ts:61-63,76), wall clock, 0 = none              */
    /* Which BranchAndCutService main.ts:62-83 would have injected: 0 = createBranchAndCutService (default;
     * speculative frontier, node slots, multi-GPU), 1 = createEnhancedBranchAndCutService (options.nodeSelection /
     * options.branching; pseudocosts make it sequential: one node LP at a time, one GPU), 2 =
     * createIncrementalBranchAndCutService (options.useIncremental: the enhanced loop with parent checkpoints).  */
    int32_t service;
    int32_t node_selection;    /* enhanced: 1 = "best-first", 2 = "depth-first", 3 = "hybrid" (0 = its default, hybrid) */
    int32_t branching;         /* enhanced: 1 = "most-fractional", 2 = "pseudocost", 3 = "strong" (0 = pseudocost)      */
    int32_t strong_candidates; /* enhanced: strongBranchingCandidates (0 = 5)                                          */
} jslp_bnb_opts;

typedef struct {
    int32_t feasible, bounded, is_integral; /* Tableau.feasible/bounded/__isIntegral        */
    int32_t iterations;                     /* Tableau.branchAndCutIterations               */
    int32_t n_best_cuts;                    /* cuts of the winning branch (left appended)   */
    int32_t rounds;                         /* speculative rounds                           */
    int64_t nodes_evaluated;                /* node LPs solved, including discarded speculation */
    int64_t pivots;                         /* pivots over all node LPs                     */
    double evaluation;                      /* Tableau.evaluation of the final tableau      */
    double best_possible_eval;
    double gpu_ms;
    int64_t kernel_launches;
    double host_eval_ms;   /* wall time spent evaluating node batches (launch + read-back + sync) */
    double host_commit_ms; /* wall time spent in the sequential commit loop                     */
    double host_root_ms;   /* part of host_eval_ms spent on the root relaxation                 */
    double host_final_ms;  /* wall time of the final re-solve of the winning branch             */
    double node_kernel_ms; /* sum over rounds of the slowest node CTA's lifetime (%globaltimer) */
    int32_t timed_out;     /* the loop ended because Date.now() >= terminalTime (branch-and-cut.ts:76)   */
    int32_t n_solutions;   /* incumbents stored under keep_solutions (jslp_bnb_solution)                 */
    int64_t nodes_pruned;  /* speculative node LPs dropped or aborted by the incumbent bound of the round */
    int64_t collectives;   /* all-gathers + all-reduces issued (n_ranks > 1)                             */
    int64_t slot_pivots;   /* pivots executed in HBM node slots (jslp_slots.cuh), this rank             */
    double slot_ms;        /* wall time of the slot-batch graphs, this rank                              */
    double slot_bytes;     /* algorithmic bytes of those pivots: 16 * H_node * stride each               */
    /* Node LPs whose pivot log repeated a block of (leaving, entering) pairs and that were solved again one after
     * another on the single tableau, where the reference's stop-before-the-repeat rule is exact; this rank.  */
    int64_t cycle_redos_kernel; /* cycles seen in the shared-memory node kernel's logs                       */
    int64_t cycle_redos_slots;  /* cycles seen in the node slots' logs, re-solved                            */
    int64_t cycle_redos_pruned; /* cycles seen in the node slots' logs, dropped unsolved: by the end of the
                                   round an incumbent below the node's relaxed evaluation was known           */
} jslp_bnb_status;

int jslp_branch_and_cut(jslp_tab *root, const jslp_bnb_opts *opts, jslp_bnb_status *out,
                        jslp_cut *best_cuts, int best_cuts_cap);
/* MIP starts, DESIGN.md section 2t: jslp_branch_and_cut (default service) seeded with known integer plans.  Start i is
 * the cut list start_cuts[start_offsets[i] .. start_offsets[i + 1]) on integer labels.  Right after the root is
 * committed fractional (where the snapshot is taken), each start's node is evaluated from the snapshot as every node
 * is; a feasible fractional node begins a depth-first dive (most fractional variable, nearer child first) of at most
 * start_nodes node LPs, all live dives advancing together, one node batch per wave.  The integral node with the
 * smallest evaluation (lowest index on a tie) becomes the incumbent before the next pop, without an iteration or a
 * node-log entry; the loop then runs unchanged.  iterations, nodes_evaluated, pivots, max_nodes and the node log count
 * tree nodes only; kernel_launches counts the whole call.  The tableau and its scalar state leave the seed stage as
 * the root left them.  n_starts = 0 is jslp_branch_and_cut.  With n_starts > 0, opts->service != 0, n_ranks > 1 and
 * optional objectives are JSLP_E_UNSUPPORTED.                                                                        */
enum { JSLP_START_SEED = 0, JSLP_START_FEASIBLE = 1, JSLP_START_INFEASIBLE = 2, JSLP_START_INCOMPLETE = 3,
       JSLP_START_SKIPPED = 4 };
typedef struct {
    int32_t status;    /* JSLP_START_*: skipped when the root was integral, infeasible or unbounded        */
    int32_t n_cuts;    /* cuts of its integral node (0 when none)                                          */
    int64_t nodes;     /* node LPs of its dive                                                             */
    int64_t pivots;    /* pivots of those node LPs                                                         */
    double evaluation; /* of its integral node (Tableau.evaluation, minimisation sense); NaN when none    */
} jslp_start_status;
int jslp_branch_and_cut_start(jslp_tab *root, const jslp_bnb_opts *opts, const jslp_cut *start_cuts,
                              const int32_t *start_offsets, int n_starts, int64_t start_nodes,
                              jslp_start_status *starts, jslp_bnb_status *out, jslp_cut *best_cuts, int best_cuts_cap);
/* What-if scenarios of a MIP, DESIGN.md section 2p: scenario s is jslp_branch_and_cut's default service (service 0)
 * over the tab's current tableau with rows 1.. of column 0 replaced by col0[s * H + r] and row 0 by row0[s * W + c]
 * (H x W = the tab's size), every tree committed in its own best-first order.  Each round evaluates the next
 * opts->max_spec_batch (0 = 16) open nodes of every live tree together, in k_node_batch launches that carry the nodes
 * of all trees.  A tableau beyond shared memory runs its scenarios one after another through jslp_branch_and_cut.
 * Without integer variables each scenario is its root LP, as jslp_simplex solves it.  Per scenario:
 *   status         feasible, bounded, is_integral, iterations, n_best_cuts, pivots, evaluation and best_possible_eval
 *                  as jslp_branch_and_cut reports them for that scenario; rounds, nodes_evaluated and nodes_pruned
 *                  count this call's own rounds and node LPs (jslp_branch_and_cut's HBM paths also prune inside a
 *                  round); status[0].kernel_launches counts the launches of the whole call
 *   rhs, vrow      row_stride entries each at s * row_stride: the final column 0 and row labels, height[s] of them
 * row_stride must be at least H plus two cuts per integer variable.  opts->service, keep_solutions, timeout_ms and
 * n_ranks > 1, useMIRCuts and optional objectives are JSLP_E_UNSUPPORTED.  On return the tab's tableau and labels,
 * snapshot, scalar Tableau state, node log and stored solutions are as they were. */
int jslp_bnb_batch(jslp_tab *tab, const double *col0, const double *row0, int n_scenarios, const jslp_bnb_opts *opts,
                   int row_stride, jslp_bnb_status *status, double *rhs, int32_t *vrow, int32_t *height);
/* Per-node trace of the last branch_and_cut: 8 doubles per committed node
 * (iteration, nCuts, feasible, evaluation, integral(-1/0/1), branchVar, branchValue, pivots). */
int jslp_bnb_node_log(jslp_tab *root, double *entries, int64_t cap, int64_t *n);
/* model.solutions under keep_solutions (branch-and-cut.ts:143-153): incumbent i of the last branch_and_cut as
 * the state generateSolutionSet reads (solution.ts:35-60): Tableau.evaluation, height, varIndexByRow[height],
 * right-hand-side column[height].  `cap` = entries the two arrays can hold.                                */
int jslp_bnb_solution(jslp_tab *root, int i, double *evaluation, int32_t *height, int32_t *var_index_by_row,
                      double *rhs_col, int cap);

#ifdef __cplusplus
}
#endif
#endif /* JSLP_B200_H */
