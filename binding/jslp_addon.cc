// binding/jslp_addon.cc -- N-API addon over include/jslp_b200.h (the thin shim BASELINE.json's north_star asks
// for: "host code stays TypeScript on Node.js calling hand-written CUDA through a thin N-API C-ABI shim").
//
// Written against the C N-API (node_api.h, ABI-stable since Node 8) rather than node-addon-api, so that it
// builds with nothing but Node's own headers: `node-gyp rebuild` in this directory (binding.gyp) links it against
// libjslp_b200.so.  One JS class, `Tab`, wraps one jslp_tab; each method is ONE call of the C ABI and replaces one
// member of the reference's Tableau seam (src/tableau/tableau.ts:103-258, SURVEY.md 8b); binding/gpu-tableau.ts
// is the `GpuTableau extends Tableau` that calls it.
//
// Node.js is not in the build image: tests/test_host_cpu.py::test_napi_addon_compiles compiles this file against
// tests/stubs/node_api.h (prototypes of exactly the N-API functions used here) and the real include/jslp_b200.h,
// which keeps the shim in step with the ABI; it has not been run under a Node runtime.
#include <node_api.h>

#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "jslp_b200.h"

namespace {

jslp_ctx *g_ctx[16] = {nullptr};
napi_ref g_tab_ctor = nullptr;

struct TabBox {
    jslp_tab *tab = nullptr;
    jslp_ctx *ctx = nullptr;
    jslp_comm *comm = nullptr;  // multi-GPU: created by Tab.prototype.createComm
    int rank = 0, n_ranks = 1;
};

// ---- small helpers -----------------------------------------------------------------------------------
#define NAPI_OK(env, call)                                                        \
    do {                                                                          \
        if ((call) != napi_ok) {                                                  \
            napi_throw_error((env), nullptr, "jslp_b200 addon: " #call " failed"); \
            return nullptr;                                                       \
        }                                                                         \
    } while (0)

bool throw_if(napi_env env, int rc) {  // solver outcomes are flags, never errors; this is misuse / driver failure
    if (rc == JSLP_OK) return false;
    std::string msg = std::string("jslp_b200: ") + jslp_last_error();
    napi_throw_error(env, nullptr, msg.c_str());
    return true;
}

napi_value undefined(napi_env env) {
    napi_value v;
    napi_get_undefined(env, &v);
    return v;
}

bool is_nullish(napi_env env, napi_value v) {
    napi_valuetype t;
    if (napi_typeof(env, v, &t) != napi_ok) return true;
    return t == napi_undefined || t == napi_null;
}

double num(napi_env env, napi_value v, double dflt = 0.0) {
    double d = dflt;
    if (!is_nullish(env, v)) napi_get_value_double(env, v, &d);
    return d;
}

bool truthy(napi_env env, napi_value v) {
    if (is_nullish(env, v)) return false;
    napi_value b;
    bool out = false;
    if (napi_coerce_to_bool(env, v, &b) == napi_ok) napi_get_value_bool(env, b, &out);
    return out;
}

void set_num(napi_env env, napi_value obj, const char *key, double v) {
    napi_value n;
    napi_create_double(env, v, &n);
    napi_set_named_property(env, obj, key, n);
}

void set_bool(napi_env env, napi_value obj, const char *key, bool v) {
    napi_value b;
    napi_get_boolean(env, v, &b);
    napi_set_named_property(env, obj, key, b);
}

napi_value prop(napi_env env, napi_value obj, const char *key) {
    napi_value v = nullptr;
    bool has = false;
    if (is_nullish(env, obj) || napi_has_named_property(env, obj, key, &has) != napi_ok || !has) return undefined(env);
    napi_get_named_property(env, obj, key, &v);
    return v;
}

// Typed-array view (data pointer + element count), or {nullptr, 0} for null / undefined.
template <typename T>
struct View {
    T *data = nullptr;
    size_t n = 0;
};
template <typename T>
bool view(napi_env env, napi_value v, napi_typedarray_type want, View<T> *out) {
    *out = View<T>();
    if (is_nullish(env, v)) return true;
    bool is_ta = false;
    if (napi_is_typedarray(env, v, &is_ta) != napi_ok || !is_ta) {
        napi_throw_type_error(env, nullptr, "jslp_b200 addon: typed array expected");
        return false;
    }
    napi_typedarray_type type;
    size_t length = 0, offset = 0;
    void *data = nullptr;
    napi_value buf;
    if (napi_get_typedarray_info(env, v, &type, &length, &data, &buf, &offset) != napi_ok || type != want) {
        napi_throw_type_error(env, nullptr, "jslp_b200 addon: wrong typed-array element type");
        return false;
    }
    out->data = static_cast<T *>(data);
    out->n = length;
    return true;
}

template <typename T>
napi_value new_typed(napi_env env, napi_typedarray_type type, size_t n, T **data) {
    napi_value buf, arr;
    void *p = nullptr;
    if (napi_create_arraybuffer(env, n * sizeof(T), &p, &buf) != napi_ok) return nullptr;
    if (napi_create_typedarray(env, type, n, buf, 0, &arr) != napi_ok) return nullptr;
    *data = static_cast<T *>(p);
    return arr;
}

TabBox *unwrap(napi_env env, napi_callback_info info, size_t *argc, napi_value *argv) {
    napi_value self;
    if (napi_get_cb_info(env, info, argc, argv, &self, nullptr) != napi_ok) return nullptr;
    TabBox *box = nullptr;
    if (napi_unwrap(env, self, reinterpret_cast<void **>(&box)) != napi_ok || !box || !box->tab) {
        napi_throw_error(env, nullptr, "jslp_b200 addon: Tab is destroyed or not a Tab");
        return nullptr;
    }
    return box;
}

// BranchCut[] {type: "min" | "max", varIndex, value} (types.ts:17-21) -> jslp_cut[]
bool read_cuts(napi_env env, napi_value arr, std::vector<jslp_cut> *out) {
    out->clear();
    if (is_nullish(env, arr)) return true;
    uint32_t n = 0;
    if (napi_get_array_length(env, arr, &n) != napi_ok) {
        napi_throw_type_error(env, nullptr, "jslp_b200 addon: BranchCut[] expected");
        return false;
    }
    out->resize(n);
    for (uint32_t i = 0; i < n; i++) {
        napi_value c;
        napi_get_element(env, arr, i, &c);
        char type[8] = {0};
        size_t len = 0;
        napi_get_value_string_utf8(env, prop(env, c, "type"), type, sizeof(type), &len);
        (*out)[i].type = std::strcmp(type, "min") == 0 ? 0 : 1;
        (*out)[i].var_index = (int32_t)num(env, prop(env, c, "varIndex"));
        (*out)[i].value = num(env, prop(env, c, "value"));
    }
    return true;
}

napi_value lp_status(napi_env env, const jslp_lp_status &s) {
    napi_value o;
    napi_create_object(env, &o);
    set_bool(env, o, "feasible", s.feasible != 0);
    set_bool(env, o, "bounded", s.bounded != 0);
    set_num(env, o, "cycled", s.cycled);
    set_num(env, o, "cycleStart", s.cycle_start);
    set_num(env, o, "cycleLength", s.cycle_length);
    set_num(env, o, "phase1Pivots", s.phase1_pivots);
    set_num(env, o, "phase2Pivots", s.phase2_pivots);
    set_num(env, o, "unboundedVarIndex", s.unbounded_var_index);
    set_num(env, o, "simplexIters", s.simplex_iters);
    set_num(env, o, "width", s.width);
    set_num(env, o, "height", s.height);
    set_num(env, o, "evaluation", s.evaluation);
    set_num(env, o, "bestPossibleEval", s.best_possible_eval);
    set_num(env, o, "gpuMs", s.gpu_ms);
    return o;
}

void tab_finalize(napi_env, void *data, void *) {
    TabBox *box = static_cast<TabBox *>(data);
    if (box->comm) jslp_comm_destroy(box->comm);
    if (box->tab) jslp_tab_destroy(box->tab);
    delete box;
}

// ---- new Tab(width, height, rowCapacity, precision, device = 0)  == Tableau.initialize (tableau.ts:292-317)
napi_value tab_new(napi_env env, napi_callback_info info) {
    size_t argc = 5;
    napi_value argv[5], self;
    NAPI_OK(env, napi_get_cb_info(env, info, &argc, argv, &self, nullptr));
    if (argc < 4) {
        napi_throw_type_error(env, nullptr, "Tab(width, height, rowCapacity, precision[, device])");
        return nullptr;
    }
    const int device = argc > 4 ? (int)num(env, argv[4]) : 0;
    if (device < 0 || device >= 16) {
        napi_throw_range_error(env, nullptr, "device ordinal out of range");
        return nullptr;
    }
    if (!g_ctx[device] && throw_if(env, jslp_ctx_create(device, nullptr, &g_ctx[device]))) return nullptr;
    TabBox *box = new TabBox();
    box->ctx = g_ctx[device];
    if (throw_if(env, jslp_tab_create(box->ctx, (int)num(env, argv[0]), (int)num(env, argv[1]), (int)num(env, argv[2]),
                                      num(env, argv[3], 1e-8), &box->tab))) {
        delete box;
        return nullptr;
    }
    NAPI_OK(env, napi_wrap(env, self, box, tab_finalize, nullptr, nullptr));
    return self;
}

// upload(matrix: Float64Array, varIndexByRow: Int32Array, varIndexByCol: Int32Array, unrestricted: Uint8Array | null,
//        intVarIndices: Int32Array | null, optCosts: Float64Array | null, nOpt: number)
// == the result of Tableau._resetMatrix / setModel (tableau.ts:319-391)
napi_value tab_upload(napi_env env, napi_callback_info info) {
    size_t argc = 7;
    napi_value argv[7];
    TabBox *box = unwrap(env, info, &argc, argv);
    if (!box) return nullptr;
    View<double> m, opt;
    View<int32_t> vr, vc, iv;
    View<uint8_t> un;
    if (!view(env, argv[0], napi_float64_array, &m) || !view(env, argv[1], napi_int32_array, &vr) ||
        !view(env, argv[2], napi_int32_array, &vc) || !view(env, argv[3], napi_uint8_array, &un) ||
        !view(env, argv[4], napi_int32_array, &iv) || !view(env, argv[5], napi_float64_array, &opt))
        return nullptr;
    const int n_opt = (int)num(env, argv[6]);
    if (!m.data || !vr.data || !vc.data || m.n != vr.n * vc.n) {
        napi_throw_range_error(env, nullptr, "upload: matrix must hold height * width doubles");
        return nullptr;
    }
    const int n_index = (int)(vr.n + vc.n - 2);
    if ((un.data && un.n < (size_t)n_index) || (opt.data && opt.n < (size_t)n_opt * vc.n)) {
        napi_throw_range_error(env, nullptr, "upload: unrestricted / optCosts too short");
        return nullptr;
    }
    if (throw_if(env, jslp_tab_upload(box->tab, m.data, vr.data, vc.data, un.data, n_index, iv.data, (int)iv.n, n_opt, opt.data)))
        return nullptr;
    return undefined(env);
}

napi_value tab_set_option(napi_env env, napi_callback_info info) {
    size_t argc = 2;
    napi_value argv[2];
    TabBox *box = unwrap(env, info, &argc, argv);
    if (!box) return nullptr;
    if (throw_if(env, jslp_tab_set_option(box->tab, (int)num(env, argv[0]), num(env, argv[1])))) return nullptr;
    return undefined(env);
}

// simplex(checkCycles) / phase1(checkCycles) / phase2(checkCycles) == Tableau.simplex / phase1 / phase2
template <int (*FN)(jslp_tab *, int, jslp_lp_status *)>
napi_value tab_lp(napi_env env, napi_callback_info info) {
    size_t argc = 1;
    napi_value argv[1];
    TabBox *box = unwrap(env, info, &argc, argv);
    if (!box) return nullptr;
    jslp_lp_status s;
    if (throw_if(env, FN(box->tab, argc > 0 ? truthy(env, argv[0]) : 1, &s))) return nullptr;
    return lp_status(env, s);
}

napi_value tab_pivot(napi_env env, napi_callback_info info) {  // == Tableau.pivot(r, c) (simplex.ts:330-413)
    size_t argc = 2;
    napi_value argv[2];
    TabBox *box = unwrap(env, info, &argc, argv);
    if (!box) return nullptr;
    if (throw_if(env, jslp_pivot(box->tab, (int)num(env, argv[0]), (int)num(env, argv[1])))) return nullptr;
    return undefined(env);
}

napi_value tab_save(napi_env env, napi_callback_info info) {  // backup.ts:49-51
    size_t argc = 0;
    TabBox *box = unwrap(env, info, &argc, nullptr);
    if (!box || throw_if(env, jslp_save(box->tab))) return nullptr;
    return undefined(env);
}

napi_value tab_restore(napi_env env, napi_callback_info info) {  // backup.ts:53-105
    size_t argc = 0;
    TabBox *box = unwrap(env, info, &argc, nullptr);
    if (!box || throw_if(env, jslp_restore(box->tab))) return nullptr;
    return undefined(env);
}

napi_value tab_add_cuts(napi_env env, napi_callback_info info) {  // cutting-strategies.ts:16-72
    size_t argc = 1;
    napi_value argv[1];
    TabBox *box = unwrap(env, info, &argc, argv);
    std::vector<jslp_cut> cuts;
    if (!box || !read_cuts(env, argv[0], &cuts)) return nullptr;
    if (throw_if(env, jslp_add_cuts(box->tab, cuts.data(), (int)cuts.size()))) return nullptr;
    return undefined(env);
}

napi_value tab_apply_cuts(napi_env env, napi_callback_info info) {  // branch-and-cut.ts:33-52
    size_t argc = 2;
    napi_value argv[2];
    TabBox *box = unwrap(env, info, &argc, argv);
    std::vector<jslp_cut> cuts;
    if (!box || !read_cuts(env, argv[0], &cuts)) return nullptr;
    jslp_lp_status s;
    if (throw_if(env, jslp_apply_cuts(box->tab, cuts.data(), (int)cuts.size(), argc > 1 ? truthy(env, argv[1]) : 1, &s)))
        return nullptr;
    return lp_status(env, s);
}

napi_value tab_is_integral(napi_env env, napi_callback_info info) {  // mip-utils.ts:43-61
    size_t argc = 0;
    TabBox *box = unwrap(env, info, &argc, nullptr);
    int v = 0;
    if (!box || throw_if(env, jslp_is_integral(box->tab, &v))) return nullptr;
    napi_value b;
    napi_get_boolean(env, v != 0, &b);
    return b;
}

napi_value tab_most_fractional(napi_env env, napi_callback_info info) {  // mip-utils.ts:100-126 -> {index, value}
    size_t argc = 0;
    TabBox *box = unwrap(env, info, &argc, nullptr);
    int32_t idx = -1;
    double val = 0;
    if (!box || throw_if(env, jslp_most_fractional(box->tab, &idx, &val))) return nullptr;
    napi_value o, n;
    napi_create_object(env, &o);
    if (idx < 0) {
        napi_get_null(env, &n);
        napi_set_named_property(env, o, "index", n);
        napi_set_named_property(env, o, "value", n);
    } else {
        set_num(env, o, "index", idx);
        set_num(env, o, "value", val);
    }
    return o;
}

// download({matrix?, rhs?, cost?, maps?, opt?: nOpt}) -> {width, height, matrix?, rhs?, cost?, varIndexByRow?, varIndexByCol?, opt?}
// what updateVariableValues / generateSolutionSet / getSolution read (dynamic-modification.ts:57-76, solution.ts:35-60)
napi_value tab_download(napi_env env, napi_callback_info info) {
    size_t argc = 1;
    napi_value argv[1];
    TabBox *box = unwrap(env, info, &argc, argv);
    if (!box) return nullptr;
    int32_t W = 0, H = 0;
    if (throw_if(env, jslp_download(box->tab, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, &W, &H))) return nullptr;
    napi_value what = argc > 0 ? argv[0] : undefined(env);
    const bool want_m = truthy(env, prop(env, what, "matrix")), want_rhs = truthy(env, prop(env, what, "rhs"));
    const bool want_cost = truthy(env, prop(env, what, "cost")), want_maps = truthy(env, prop(env, what, "maps"));
    const int n_opt = (int)num(env, prop(env, what, "opt"));
    napi_value o;
    napi_create_object(env, &o);
    set_num(env, o, "width", W);
    set_num(env, o, "height", H);
    double *m = nullptr, *rhs = nullptr, *cost = nullptr, *opt = nullptr;
    int32_t *vr = nullptr, *vc = nullptr;
    if (want_m) napi_set_named_property(env, o, "matrix", new_typed(env, napi_float64_array, (size_t)W * H, &m));
    if (want_rhs) napi_set_named_property(env, o, "rhs", new_typed(env, napi_float64_array, (size_t)H, &rhs));
    if (want_cost) napi_set_named_property(env, o, "cost", new_typed(env, napi_float64_array, (size_t)W, &cost));
    if (want_maps) {
        napi_set_named_property(env, o, "varIndexByRow", new_typed(env, napi_int32_array, (size_t)H, &vr));
        napi_set_named_property(env, o, "varIndexByCol", new_typed(env, napi_int32_array, (size_t)W, &vc));
    }
    if (n_opt > 0) napi_set_named_property(env, o, "opt", new_typed(env, napi_float64_array, (size_t)n_opt * W, &opt));
    if (throw_if(env, jslp_download(box->tab, m, rhs, cost, vr, vc, opt, nullptr, nullptr))) return nullptr;
    return o;
}

napi_value tab_pivot_log(napi_env env, napi_callback_info info) {  // Int32Array of (row, col, leaving, entering)
    size_t argc = 0;
    TabBox *box = unwrap(env, info, &argc, nullptr);
    if (!box) return nullptr;
    int n = 0;
    std::vector<int32_t> buf((size_t)4 << 20);
    if (throw_if(env, jslp_pivot_log(box->tab, buf.data(), (int)(buf.size() / 4), &n))) return nullptr;
    const size_t m = (size_t)4 * (size_t)std::min<int64_t>(n, (int64_t)buf.size() / 4);
    int32_t *out = nullptr;
    napi_value arr = new_typed(env, napi_int32_array, m, &out);
    if (arr && m) std::memcpy(out, buf.data(), m * sizeof(int32_t));
    return arr;
}

// Multi-GPU (one Node process per GPU): Tab.uniqueId() on rank 0 -> Uint8Array(128), shipped to the other ranks over
// the host's own IPC; tab.createComm(id, rank, nRanks) on every rank; branchAndCut then shards each round's nodes.
napi_value tab_unique_id(napi_env env, napi_callback_info) {
    uint8_t *out = nullptr;
    napi_value arr = new_typed(env, napi_uint8_array, 128, &out);
    if (!arr || throw_if(env, jslp_comm_unique_id(out))) return nullptr;
    return arr;
}

napi_value tab_create_comm(napi_env env, napi_callback_info info) {
    size_t argc = 3;
    napi_value argv[3];
    TabBox *box = unwrap(env, info, &argc, argv);
    View<uint8_t> id;
    if (!box || !view(env, argv[0], napi_uint8_array, &id)) return nullptr;
    if (!id.data || id.n != 128) {
        napi_throw_range_error(env, nullptr, "createComm: the unique id is 128 bytes");
        return nullptr;
    }
    if (box->comm) jslp_comm_destroy(box->comm);
    box->comm = nullptr;
    box->rank = (int)num(env, argv[1]);
    box->n_ranks = (int)num(env, argv[2], 1);
    if (throw_if(env, jslp_comm_create(box->ctx, id.data, box->rank, box->n_ranks, &box->comm))) return nullptr;
    return undefined(env);
}

// branchAndCut({tolerance, isMinimization, checkCycles, maxSpecBatch?, keepSolutions?, timeout?, maxNodes?, shardPolicy?,
//               nodeSelection?, branching?, strongBranchingCandidates?})
//   == BranchAndCutService.branchAndCut (branch-and-cut.ts:54-199)
// -> {feasible, bounded, isIntegral, iterations, evaluation, bestPossibleEval, timedOut, bestCuts: BranchCut[],
//     solutions: [{evaluation, varIndexByRow: Int32Array, rhs: Float64Array}], nodeLps, rounds, pivots, gpuMs}
napi_value tab_branch_and_cut(napi_env env, napi_callback_info info) {
    size_t argc = 1;
    napi_value argv[1];
    TabBox *box = unwrap(env, info, &argc, argv);
    if (!box) return nullptr;
    napi_value o = argc > 0 ? argv[0] : undefined(env);
    jslp_bnb_opts opts;
    std::memset(&opts, 0, sizeof(opts));
    opts.tolerance = num(env, prop(env, o, "tolerance"));
    opts.is_minimization = truthy(env, prop(env, o, "isMinimization"));
    opts.check_cycles = is_nullish(env, prop(env, o, "checkCycles")) ? 1 : truthy(env, prop(env, o, "checkCycles"));
    opts.max_spec_batch = (int32_t)num(env, prop(env, o, "maxSpecBatch"));
    opts.keep_solutions = truthy(env, prop(env, o, "keepSolutions"));
    opts.timeout_ms = num(env, prop(env, o, "timeout"));
    opts.max_nodes = (int64_t)num(env, prop(env, o, "maxNodes"));
    opts.shard_policy = (int32_t)num(env, prop(env, o, "shardPolicy"));
    {   // options.nodeSelection / options.branching select the enhanced service (main.ts:62-83)
        char ns[16] = {0}, br[20] = {0};
        size_t len = 0;
        if (!is_nullish(env, prop(env, o, "nodeSelection"))) napi_get_value_string_utf8(env, prop(env, o, "nodeSelection"), ns, sizeof(ns), &len);
        if (!is_nullish(env, prop(env, o, "branching"))) napi_get_value_string_utf8(env, prop(env, o, "branching"), br, sizeof(br), &len);
        const bool incremental = truthy(env, prop(env, o, "useIncremental"));
        if (ns[0] || br[0] || incremental || truthy(env, prop(env, o, "enhanced"))) {
            opts.service = incremental ? 2 : 1;  // main.ts:62-83: useIncremental wins over nodeSelection / branching
            opts.node_selection = !std::strcmp(ns, "best-first") ? 1 : !std::strcmp(ns, "depth-first") ? 2 : 3;
            opts.branching = !std::strcmp(br, "most-fractional") ? 1 : !std::strcmp(br, "strong") ? 3 : 2;
            opts.strong_candidates = (int32_t)num(env, prop(env, o, "strongBranchingCandidates"));
        }
    }
    opts.rank = box->rank;
    opts.n_ranks = box->comm ? box->n_ranks : 1;
    opts.comm = box->comm;
    jslp_bnb_status st;
    std::vector<jslp_cut> best(4096);
    if (throw_if(env, jslp_branch_and_cut(box->tab, &opts, &st, best.data(), (int)best.size()))) return nullptr;
    napi_value r;
    napi_create_object(env, &r);
    set_bool(env, r, "feasible", st.feasible != 0);
    set_bool(env, r, "bounded", st.bounded != 0);
    set_bool(env, r, "isIntegral", st.is_integral != 0);
    set_bool(env, r, "timedOut", st.timed_out != 0);
    set_num(env, r, "iterations", st.iterations);
    set_num(env, r, "evaluation", st.evaluation);
    set_num(env, r, "bestPossibleEval", st.best_possible_eval);
    set_num(env, r, "rounds", st.rounds);
    set_num(env, r, "nodeLps", (double)st.nodes_evaluated);
    set_num(env, r, "pivots", (double)st.pivots);
    set_num(env, r, "gpuMs", st.gpu_ms);
    napi_value cuts;
    const int nb = std::min<int>(st.n_best_cuts, (int)best.size());
    napi_create_array_with_length(env, (size_t)nb, &cuts);
    for (int i = 0; i < nb; i++) {
        napi_value c, ty;
        napi_create_object(env, &c);
        napi_create_string_utf8(env, best[i].type == 0 ? "min" : "max", NAPI_AUTO_LENGTH, &ty);
        napi_set_named_property(env, c, "type", ty);
        set_num(env, c, "varIndex", best[i].var_index);
        set_num(env, c, "value", best[i].value);
        napi_set_element(env, cuts, (uint32_t)i, c);
    }
    napi_set_named_property(env, r, "bestCuts", cuts);
    napi_value sols;
    napi_create_array_with_length(env, (size_t)st.n_solutions, &sols);
    for (int i = 0; i < st.n_solutions; i++) {
        double ev = 0;
        int32_t h = 0;
        if (throw_if(env, jslp_bnb_solution(box->tab, i, &ev, &h, nullptr, nullptr, 0))) return nullptr;
        int32_t *vr = nullptr;
        double *rhs = nullptr;
        napi_value s, a_vr = new_typed(env, napi_int32_array, (size_t)h, &vr), a_rhs = new_typed(env, napi_float64_array, (size_t)h, &rhs);
        if (throw_if(env, jslp_bnb_solution(box->tab, i, nullptr, nullptr, vr, rhs, h))) return nullptr;
        napi_create_object(env, &s);
        set_num(env, s, "evaluation", ev);
        napi_set_named_property(env, s, "varIndexByRow", a_vr);
        napi_set_named_property(env, s, "rhs", a_rhs);
        napi_set_element(env, sols, (uint32_t)i, s);
    }
    napi_set_named_property(env, r, "solutions", sols);
    set_num(env, r, "cycleRedosKernel", (double)st.cycle_redos_kernel);
    set_num(env, r, "cycleRedosSlots", (double)st.cycle_redos_slots);
    set_num(env, r, "cycleRedosPruned", (double)st.cycle_redos_pruned);
    return r;
}

// ---- dynamic-modification.ts on the device tableau: constraints / variables named by their element index
napi_value tab_put_in_base(napi_env env, napi_callback_info info) {       // putInBase(varIndex) -> row
    size_t argc = 1;
    napi_value argv[1];
    TabBox *box = unwrap(env, info, &argc, argv);
    int r = -1;
    if (!box || throw_if(env, jslp_put_in_base(box->tab, (int)num(env, argv[0]), &r))) return nullptr;
    napi_value v;
    napi_create_int32(env, r, &v);
    return v;
}
napi_value tab_take_out_of_base(napi_env env, napi_callback_info info) {  // takeOutOfBase(varIndex) -> column
    size_t argc = 1;
    napi_value argv[1];
    TabBox *box = unwrap(env, info, &argc, argv);
    int c = -1;
    if (!box || throw_if(env, jslp_take_out_of_base(box->tab, (int)num(env, argv[0]), &c))) return nullptr;
    napi_value v;
    napi_create_int32(env, c, &v);
    return v;
}
napi_value tab_update_rhs(napi_env env, napi_callback_info info) {        // updateRightHandSide(constraintIndex, difference)
    size_t argc = 2;
    napi_value argv[2];
    TabBox *box = unwrap(env, info, &argc, argv);
    if (!box || throw_if(env, jslp_update_rhs(box->tab, (int)num(env, argv[0]), num(env, argv[1])))) return nullptr;
    return undefined(env);
}
napi_value tab_update_coefficient(napi_env env, napi_callback_info info) {  // (constraintIndex, varIndex, difference)
    size_t argc = 3;
    napi_value argv[3];
    TabBox *box = unwrap(env, info, &argc, argv);
    if (!box || throw_if(env, jslp_update_coefficient(box->tab, (int)num(env, argv[0]), (int)num(env, argv[1]), num(env, argv[2])))) return nullptr;
    return undefined(env);
}
napi_value tab_update_cost(napi_env env, napi_callback_info info) {       // (varIndex, optSlot, difference)
    size_t argc = 3;
    napi_value argv[3];
    TabBox *box = unwrap(env, info, &argc, argv);
    if (!box || throw_if(env, jslp_update_cost(box->tab, (int)num(env, argv[0]), (int)num(env, argv[1], -1), num(env, argv[2])))) return nullptr;
    return undefined(env);
}
napi_value tab_add_constraint(napi_env env, napi_callback_info info) {    // (isUpperBound, rhs, slackIndex, termVars: Int32Array, termCoefs: Float64Array)
    size_t argc = 5;
    napi_value argv[5];
    TabBox *box = unwrap(env, info, &argc, argv);
    View<int32_t> tv;
    View<double> tc;
    if (!box || !view(env, argv[3], napi_int32_array, &tv) || !view(env, argv[4], napi_float64_array, &tc)) return nullptr;
    if (tv.n != tc.n) {
        napi_throw_range_error(env, nullptr, "addConstraint: termVars and termCoefs differ in length");
        return nullptr;
    }
    if (throw_if(env, jslp_add_constraint(box->tab, truthy(env, argv[0]), num(env, argv[1]), (int)num(env, argv[2]), tv.data, tc.data, (int)tv.n)))
        return nullptr;
    return undefined(env);
}
napi_value tab_remove_constraint(napi_env env, napi_callback_info info) {
    size_t argc = 1;
    napi_value argv[1];
    TabBox *box = unwrap(env, info, &argc, argv);
    if (!box || throw_if(env, jslp_remove_constraint(box->tab, (int)num(env, argv[0])))) return nullptr;
    return undefined(env);
}
napi_value tab_add_variable(napi_env env, napi_callback_info info) {      // (varIndex, costEntry, optSlot, isInteger, isUnrestricted)
    size_t argc = 5;
    napi_value argv[5];
    TabBox *box = unwrap(env, info, &argc, argv);
    if (!box || throw_if(env, jslp_add_variable(box->tab, (int)num(env, argv[0]), num(env, argv[1]), (int)num(env, argv[2], -1),
                                                truthy(env, argv[3]), truthy(env, argv[4]))))
        return nullptr;
    return undefined(env);
}
napi_value tab_remove_variable(napi_env env, napi_callback_info info) {
    size_t argc = 1;
    napi_value argv[1];
    TabBox *box = unwrap(env, info, &argc, argv);
    if (!box || throw_if(env, jslp_remove_variable(box->tab, (int)num(env, argv[0])))) return nullptr;
    return undefined(env);
}
napi_value tab_info(napi_env env, napi_callback_info info) {  // {width, height, nVars, lastElementIndex}
    size_t argc = 0;
    TabBox *box = unwrap(env, info, &argc, nullptr);
    int32_t v[6];
    if (!box || throw_if(env, jslp_tab_info(box->tab, v))) return nullptr;
    napi_value o;
    napi_create_object(env, &o);
    set_num(env, o, "width", v[0]);
    set_num(env, o, "height", v[1]);
    set_num(env, o, "nVars", v[2]);
    set_num(env, o, "lastElementIndex", v[3]);
    return o;
}

napi_value tab_destroy(napi_env env, napi_callback_info info) {
    napi_value self;
    size_t argc = 0;
    NAPI_OK(env, napi_get_cb_info(env, info, &argc, nullptr, &self, nullptr));
    TabBox *box = nullptr;
    if (napi_unwrap(env, self, reinterpret_cast<void **>(&box)) == napi_ok && box) {
        if (box->comm) jslp_comm_destroy(box->comm);
        if (box->tab) jslp_tab_destroy(box->tab);
        box->comm = nullptr;
        box->tab = nullptr;
    }
    return undefined(env);
}

napi_value abi_version(napi_env env, napi_callback_info) {
    napi_value v;
    napi_create_int32(env, jslp_abi_version(), &v);
    return v;
}

napi_value init(napi_env env, napi_value exports) {
    const napi_property_descriptor methods[] = {
        {"upload", nullptr, tab_upload, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"setOption", nullptr, tab_set_option, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"simplex", nullptr, tab_lp<jslp_simplex>, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"phase1", nullptr, tab_lp<jslp_phase1>, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"phase2", nullptr, tab_lp<jslp_phase2>, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"pivot", nullptr, tab_pivot, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"save", nullptr, tab_save, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"restore", nullptr, tab_restore, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"addCuts", nullptr, tab_add_cuts, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"applyCuts", nullptr, tab_apply_cuts, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"isIntegral", nullptr, tab_is_integral, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"mostFractional", nullptr, tab_most_fractional, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"download", nullptr, tab_download, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"pivotLog", nullptr, tab_pivot_log, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"createComm", nullptr, tab_create_comm, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"branchAndCut", nullptr, tab_branch_and_cut, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"putInBase", nullptr, tab_put_in_base, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"takeOutOfBase", nullptr, tab_take_out_of_base, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"updateRhs", nullptr, tab_update_rhs, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"updateCoefficient", nullptr, tab_update_coefficient, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"updateCost", nullptr, tab_update_cost, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"addConstraint", nullptr, tab_add_constraint, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"removeConstraint", nullptr, tab_remove_constraint, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"addVariable", nullptr, tab_add_variable, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"removeVariable", nullptr, tab_remove_variable, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"info", nullptr, tab_info, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"destroy", nullptr, tab_destroy, nullptr, nullptr, nullptr, napi_default, nullptr},
        {"uniqueId", nullptr, tab_unique_id, nullptr, nullptr, nullptr, napi_static, nullptr},
    };
    napi_value ctor, fn;
    NAPI_OK(env, napi_define_class(env, "Tab", NAPI_AUTO_LENGTH, tab_new, nullptr, sizeof(methods) / sizeof(methods[0]), methods, &ctor));
    NAPI_OK(env, napi_create_reference(env, ctor, 1, &g_tab_ctor));
    NAPI_OK(env, napi_set_named_property(env, exports, "Tab", ctor));
    NAPI_OK(env, napi_create_function(env, "abiVersion", NAPI_AUTO_LENGTH, abi_version, nullptr, &fn));
    NAPI_OK(env, napi_set_named_property(env, exports, "abiVersion", fn));
    return exports;
}

}  // namespace

NAPI_MODULE(jslp_b200, init)
