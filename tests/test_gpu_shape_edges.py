"""The pivot step at the edges of its launch geometry, bit for bit against the oracle.

How the fused step splits a tableau depends on the device and the shape: rows per row CTA (the ping-pong step runs
while every row CTA has at most 32 rows, its look-ahead warp owning one row per lane), the row stride against the
CTA's threads, the phase-1 selector's register path (stride <= 8 x threads), whether two ping-pong CTAs with a long
staged pivot row are co-resident, the automatic flat-8 choice once the ping-pong pair outgrows L2, and whether a
tableau fits the shared-memory node kernel.  A small planner restates those rules from the device's properties, every
shape is derived from it, and every case reads the step's timeline to check that it ran the regime it claims.

Two value families run at those geometries too: exact ties across row CTAs, lanes and pricing batches, and entries
sitting on the fixed thresholds (1e-16, the 1e-8 precision), signed zeros, subnormals and values near 1e+-300 whose
products overflow during pivoting."""
import ctypes as C
import functools
from collections import namedtuple

import numpy as np
import pytest

from test_gpu_lp_parity import assert_lp_parity, gpu_lp, oracle_lp, same_bits

pytestmark = pytest.mark.gpu

# ------------------------------------------------------------------ geometry planner
# STEP_VARIANTS of jslp_api.cu: (threads, CTAs per SM, rows per pass; negative = flat loop of that many pairs)
STEP_VARIANTS = [(256, 2, 8), (256, 2, 4), (256, 4, 4), (512, 1, 8), (256, 3, 4), (128, 8, 4), (256, 2, 4),
                 (256, 2, 2), (256, 1, 8), (512, 1, 4), (256, 2, -4), (256, 2, -8), (256, 3, -4), (256, 4, -2)]
PP_MAX_ROWS = 32         # rows per row CTA the ping-pong look-ahead warp covers (one per lane)
STATIC_SMEM_MAX = 8192   # generous bound on the step kernel's static shared memory + the per-CTA reservation
Dev = namedtuple("Dev", "sms l2 smem_optin smem_per_sm")
Plan = namedtuple("Plan", "variant threads grid G rows pp coresident rows_fit stride")
H100_SXM = Dev(132, 50 << 20, 232448, 233472)


def device():
    import torch
    p = torch.cuda.get_device_properties(0)
    return Dev(p.multi_processor_count, p.L2_cache_size, p.shared_memory_per_block_optin,
               p.shared_memory_per_multiprocessor)


def stride_of(W):
    return (W + 15) & ~15


def plan(dev, H, W, variant=-1, grid_per_sm=0, rowcap=None, pingpong=True):
    """step_grid / use_pp / variant_index of jslp_api.cu restated.  coresident is None when the shared-memory estimate
    cannot decide whether the ping-pong grid fits on the device at once."""
    rowcap = rowcap or H + 64
    stride = stride_of(W)
    v = variant if variant >= 0 else (11 if 16.0 * rowcap * stride > 0.95 * dev.l2 else 10)
    nt, occ, _ = STEP_VARIANTS[v]
    grid = max(1, min(dev.sms * (grid_per_sm or occ), rowcap))
    dyn = stride * 8
    per_sm = [min(dev.smem_per_sm // (dyn + s), 2048 // nt) for s in (1024, STATIC_SMEM_MAX)]
    fit = [k * dev.sms >= grid for k in per_sm]
    coresident = fit[0] if fit[0] == fit[1] else None
    pp = bool(pingpong and grid >= 3 and H // (grid - 2) + 1 <= PP_MAX_ROWS and coresident)
    G = grid - 2 if pp else grid
    return Plan(v, nt, grid, G, -(-H // G), pp, coresident, H // G + 1 <= nt, stride)


def pp_rows(dev, variant, grid_per_sm=0):
    """Row CTAs of the ping-pong step at the variant's grid (a tableau tall enough not to shrink it)."""
    return dev.sms * (grid_per_sm or STEP_VARIANTS[variant][1]) - 2


def height_for(dev, variant, r, grid_per_sm=0):
    """Tableau height whose largest row CTA has r rows under the ping-pong split; r = 33 is the first height past it."""
    G = pp_rows(dev, variant, grid_per_sm)
    if r == 1:
        return G
    if r == PP_MAX_ROWS + 1:
        return PP_MAX_ROWS * G
    return r * G - 1


def node_smem_bytes(H, W):
    """node_smem_bytes of jslp_bnb.cuh: tableau, two staged rows, pivot column, cut records, index arrays."""
    Ws = (W + 1) & ~1
    return 8 * (H * Ws + 2 * Ws + H + 1) + 16 * H + 4 * (2 * H + W) + 16


def resident_rows(dev, W):
    """Largest tableau height the shared-memory node kernel takes at width W (resident_fits)."""
    limit = dev.smem_optin - 4096
    H = max(1, (limit - node_smem_bytes(0, W)) // max(1, node_smem_bytes(1, W) - node_smem_bytes(0, W)))
    while node_smem_bytes(H + 1, W) <= limit:
        H += 1
    while node_smem_bytes(H, W) > limit:
        H -= 1
    return H


def flat8_height(dev, W):
    """Smallest height whose ping-pong pair (16 rowcap stride bytes) crosses 0.95 x L2 at width W."""
    stride = stride_of(W)
    H = max(1, int(0.95 * dev.l2 / (16.0 * stride)) - 64 - 2)
    while not 16.0 * (H + 64) * stride > 0.95 * dev.l2:
        H += 1
    return H


# ------------------------------------------------------------------ inputs
def mixed_arrays(n_rows, n_vars, seed, n_lower=4, profitable=None):
    """Dense LP, max c.x: packing rows a.x <= b and n_lower covering rows a.x >= b (phase 1), a ~ U{1..20}.  x = 0.5
    satisfies every row, so the LP is feasible, and the packing rows bound it.  profitable: only that many columns
    keep a positive cost and the others get a negative one (never priced in by phase 2, as the packing rows' duals are
    non-negative), so a wide or tall tableau is solved in few pivots."""
    rng = np.random.default_rng(seed)
    A = rng.integers(1, 21, size=(n_rows, n_vars)).astype(np.float64)
    b = rng.integers(100, 501, size=n_rows).astype(np.float64) + 10.0 * n_vars
    lower = np.zeros(n_rows, dtype=bool)
    lower[rng.choice(n_rows, size=min(n_lower, n_rows - 1), replace=False)] = True
    b[lower] = np.ceil(0.25 * A[lower].sum(axis=1))
    c = rng.integers(1, 51, size=n_vars).astype(np.float64)
    if profitable is not None and profitable < n_vars:
        c[rng.permutation(n_vars)[profitable:]] *= -1.0
    return A, b, c, lower


def tie_arrays(n_rows, n_vars, seed, G, nt, profitable=None, row_offsets=None, col_offsets=None):
    """mixed_arrays with exact ties where the device merges partial results.  Rows: lanes 2..9 of row CTA 1 are copied
    to the same lanes of three other row CTAs (equal ratio-test quotients merged across CTAs; after a pivot on one copy
    the others are degenerate in several CTAs).  Columns: the most profitable column is copied 50 columns on (the next
    partial-pricing batch) and 8 x threads columns on (another register slot of the selector).  Row CTA b of G owns
    tableau rows from b * (H // G) + min(b, H % G).  row_offsets / col_offsets replace those placements for a kernel
    that splits the tableau differently: tableau rows 2..9 are copied that many rows on, the column that many columns
    on."""
    A, b, c, lower = mixed_arrays(n_rows, n_vars, seed, n_lower=2, profitable=profitable)
    H = n_rows + 1
    base, rem = divmod(H, G)
    r0 = lambda k: k * base + min(k, rem)
    lanes = range(2, min(10, base))
    if row_offsets is None:
        pairs = [(r0(1) + lane - 1, r0(k) + lane - 1) for k in sorted({3 % G, G // 2, G - 1} - {1}) for lane in lanes]
    else:
        pairs = [(t - 1, t - 1 + off) for off in row_offsets for t in range(2, 10)]
    for src, dst in pairs:   # tableau row t is array row t - 1
        if 0 <= dst < n_rows and dst != src:
            A[dst], b[dst], lower[dst] = A[src], b[src], lower[src]
    j0 = 1
    c[j0] = c.max() + 1.0
    for off in (50, 8 * nt) if col_offsets is None else col_offsets:
        if j0 + off < n_vars:
            A[:, j0 + off], c[j0 + off] = A[:, j0], c[j0]
    return A, b, c, lower


_tiny = [1e-16, np.nextafter(1e-16, 1.0), 1e-8, np.nextafter(1e-8, 0.0), np.nextafter(1e-8, 1.0)]
THRESHOLDS = [0.0, -0.0] + [s * v for v in _tiny for s in (1.0, -1.0)]
SUBNORMALS = [5e-324, -2.5e-320, 1e-310, -4.9e-315]
HUGE = [1e300, -7e299, 3e-300, -1e-300]


def threshold_arrays(n_rows, n_vars, seed, extreme=True):
    """mixed_arrays with entries on the thresholds every element rule tests: costs, right-hand sides and whole columns
    set to +-0, +-1e-16 and +-1e-8 and their neighbours (precision 1e-8); with extreme, also a sprinkle of such entries,
    subnormals, and entries near 1e+-300 whose products overflow to +-inf / NaN during pivoting (an outside solver drops
    matrix entries that small, so its comparison runs without them).  The rows with a threshold
    right-hand side pin the solution near 0, which keeps the LP feasible."""
    A, b, c, lower = mixed_arrays(n_rows, n_vars, seed, n_lower=max(4, n_rows // 20))
    rng = np.random.default_rng(seed + 1000)
    T = np.array(THRESHOLDS)
    cols = rng.permutation(n_vars)
    k = min(len(T), n_vars // 3)
    c[cols[:k]] = T[:k]                                            # cost row entries
    rows = rng.permutation(n_rows)
    kr = min(len(T), n_rows // 3)
    lower[:] = False                                               # right-hand sides: every other one a covering row,
    lower[rows[:kr:2]] = True                                      # the packing rows' kept non-negative (x = 0 fits)
    # (without extreme, the packing rows keep their right-hand sides: an optimum pinned within 1e-8 of 0 is decided by
    # the precision rules, which an outside solver with its own tolerances does not share)
    b[rows[:kr]] = np.where(lower[rows[:kr]], T[:kr], np.abs(T[:kr]) if extreme else b[rows[:kr]])
    for j, v in zip(cols[k:k + 3], (1e-8, np.nextafter(1e-8, 0.0), -1e-16)):
        A[:, j], c[j] = v, -1.0                                    # whole columns on a threshold (a cost that
                                                                   # prices them in would make the LP unbounded)
    if extreme:
        m = rng.random(A.shape) < 0.02
        A[m] = rng.choice(T, size=int(m.sum()))
        pos = rng.integers(0, [n_rows, n_vars], size=(len(SUBNORMALS), 2))
        A[pos[:, 0], pos[:, 1]] = SUBNORMALS
        pos = rng.integers(0, [n_rows, n_vars], size=(len(HUGE), 2))
        A[pos[:, 0], pos[:, 1]] = HUGE
        A[rows[kr], cols[0]] = 1e300
        b[rows[kr + 1]] = 1e300
    # (extreme) rows that hold only the top-cost column, at exactly / just under / just over the precision, with a zero or 1e-16
    # right-hand side: untouched by phase 1 (which pivots elsewhere), they decide phase 2's first ratio test -- an entry
    # of exactly 1e-8 takes part (|col| >= prec) and wins with a zero quotient
    if extreme:
        jp = int(np.argmax(c[:50]))
        c[jp] = c.max() + 1.0
        for r, v, rhs in zip(rows[kr + 2:kr + 6], (1e-8, np.nextafter(1e-8, 0.0), 1e-8, np.nextafter(1e-8, 1.0)),
                             (1e-16, 0.0, 0.0, 0.0)):
            A[r], lower[r], b[r] = 0.0, False, rhs
            A[r, jp] = v
    return A, b, c, lower


FAMILIES = {"mixed": mixed_arrays, "ties": tie_arrays, "thresholds": threshold_arrays}


@functools.lru_cache(maxsize=None)
def solved(family, n_rows, n_vars, seed, extra=()):
    """(initial tableau, oracle solved from it); each shape is solved by the oracle once for every variant."""
    from jslpsolver_b200 import problems
    A, b, c, lower = FAMILIES[family](n_rows, n_vars, seed, *extra)
    it = problems.lp_tableau(A, b, c, lower)
    o = oracle_lp(it)
    o.simplex()
    return it, o


# ------------------------------------------------------------------ regime checks
def timeline(g):
    """Per-CTA records of the first pivot steps (jslp_debug_timeline): (launches, grid, 8)."""
    from jslpsolver_b200 import _lib
    L = g.context.lib
    n, grid = C.c_int(), C.c_int()
    _lib.check(L.jslp_debug_timeline(g.handle, None, 0, C.byref(n), C.byref(grid)))
    buf = np.zeros((n.value, grid.value, 8), dtype=np.int64)
    if buf.size:
        _lib.check(L.jslp_debug_timeline(g.handle, buf.ctypes.data, buf.size, C.byref(n), C.byref(grid)))
    return grid.value, buf


def assert_regime(g, p, what):
    """The step ran the planned geometry: grid, rows of the largest row CTA (d[7]), and the ping-pong step exactly when
    planned (its staging selector writes d[6] = 2; the in-place step writes only 0 / 1 there)."""
    st = g.lastStatus
    grid, tl = timeline(g)
    ran_pp = bool((tl[:, :, 6] == 2).any())
    rows = int(tl[:, :, 7].max()) if tl.size else 0
    print(f"{what}: variant {p.variant} grid {grid} rows/CTA {rows} {'ping-pong' if ran_pp else 'in-place'} "
          f"engine {st.engine} pivots {st.phase1_pivots}+{st.phase2_pivots}")
    assert st.engine == 2, (what, st.engine)
    assert tl.size and tl[:, :, 7].any(), f"{what}: no pivot step recorded"
    assert grid == p.grid, (what, grid, p)
    assert rows == p.rows, (what, rows, p)
    assert ran_pp == p.pp, (what, ran_pp, p)


def run(family, n_rows, n_vars, seed, p, what, extra=(), variant=None, grid_per_sm=0, pingpong=True, engine=2):
    it, o = solved(family, n_rows, n_vars, seed, extra)
    assert it.matrix.shape == (n_rows + 1, n_vars + 1)
    v = p.variant if variant is None else variant
    g = gpu_lp(it, (engine, 1, v, 0, int(pingpong)), grid_per_sm=grid_per_sm, timeline=64)
    g.simplex()
    assert_lp_parity(g, o, what)
    assert_regime(g, p, what)
    st = g.lastStatus
    g.close()
    return st


# ------------------------------------------------------------------ rows per row CTA, every variant
ROW_CASES = [(1, 17), ("rc+1", 32), (17, 31), (32, 41), (33, 17)]   # (rows per CTA, W): W = 1, 0, 15, 9 mod 16


@pytest.mark.parametrize("r,W", ROW_CASES, ids=[f"r{r}-W{w}" for r, w in ROW_CASES])
@pytest.mark.parametrize("variant", range(len(STEP_VARIANTS)))
def test_rows_per_cta_every_variant(variant, r, W):
    """1, rows-per-pass + 1, 17 and 32 rows per row CTA run the ping-pong step; 33 (H = 32 G) the in-place step.
    Every LP has covering rows (phase-1 pivots); the 1- and 33-row cases pivot in phase 2 as well."""
    dev = device()
    if r == "rc+1":
        r = abs(STEP_VARIANTS[variant][2]) + 1
    H = height_for(dev, variant, r)
    p = plan(dev, H, W, variant)
    assert p.pp == (r <= PP_MAX_ROWS)
    st = run("mixed", H - 1, W - 1, 1000 + r, p, f"variant {variant} {H}x{W}")
    assert st.phase1_pivots > 0 and (st.phase2_pivots > 0 or r not in (1, PP_MAX_ROWS + 1))


@pytest.mark.parametrize("W", [3, 17])
@pytest.mark.parametrize("edge", ["fits", "past"])
def test_in_place_lookahead_tail_edge(edge, W):
    """In-place step, 128 threads, one CTA per SM: base + 1 = threads rows per CTA keeps the look-ahead tail (one row per
    thread); one row more and the last CTA selects with cta_select."""
    dev = device()
    nt = STEP_VARIANTS[5][0]
    H = nt * dev.sms - (1 if edge == "fits" else 0)
    p = plan(dev, H, W, 5, grid_per_sm=1)
    assert not p.pp and p.rows_fit == (edge == "fits")
    st = run("mixed", H - 1, W - 1, 2000 + W, p, f"in-place tail {edge} {H}x{W}", grid_per_sm=1)
    assert st.phase2_pivots > 0


@pytest.mark.parametrize("W", [41, 600])
@pytest.mark.parametrize("variant", [10, 11, 12, 13, 0, 5])
def test_row_length_against_cta(variant, W):
    """17 rows per row CTA, one CTA per SM: 24 column pairs per row (fewer than the threads: the flat loop wraps rows
    inside one thread's walk) and 304 (more than the threads, not a multiple of them)."""
    dev = device()
    H = height_for(dev, variant, 17, grid_per_sm=1)
    p = plan(dev, H, W, variant, grid_per_sm=1)
    assert p.pp and p.rows == 17
    pairs = p.stride // 2
    assert (pairs < p.threads) if W == 41 else (pairs > p.threads and pairs % p.threads)
    run("mixed", H - 1, W - 1, 3000 + variant, p, f"row length variant {variant} {H}x{W}", extra=(1, 24),
        grid_per_sm=1)


# (variant, W, seed): the reference's phase-1 rule runs very long on some random instances; these seeds solve quickly
SELECTOR_EDGES = [(10, 2048, 4200), (10, 2049, 4010), (5, 1024, 4005), (5, 1025, 4005), (3, 4096, 4003), (3, 4097, 4003)]


@pytest.mark.parametrize("variant,W,seed", SELECTOR_EDGES, ids=[f"v{v}-W{w}" for v, w, _ in SELECTOR_EDGES])
def test_phase1_selector_width_edge(variant, W, seed):
    """The phase-1 selector keeps the derived row in registers while stride <= 8 x threads and reloads past that."""
    dev = device()
    H = 40
    p = plan(dev, H, W, variant)
    assert p.pp and (p.stride <= 8 * p.threads) == (W % 2 == 0)
    st = run("mixed", H - 1, W - 1, seed, p, f"selector edge variant {variant} {H}x{W}", extra=(12, 40))
    assert st.phase1_pivots > 0


CORESIDENCY = [(12000, "wave", 17000), (16000, "wave", 21000), (25600, "short", 30600), (25600, "wave", 5200)]


@pytest.mark.parametrize("W,rows,seed", CORESIDENCY, ids=[f"W{w}-{r}" for w, r, _ in CORESIDENCY])
def test_coresidency_cut_over(W, rows, seed):
    """A long staged pivot row: two ping-pong CTAs per SM fit at 12 000 columns, one at 16 000 and at the 25 600-column
    cap.  A grid wider than one CTA per SM ('wave', rowcap = H + 64 > SMs) cannot be co-resident there and runs the
    in-place step; a short tableau ('short') keeps the grid within one wave and runs the ping-pong step."""
    dev = device()
    H = dev.sms - 24 if rows == "wave" else 20
    if stride_of(W) * 8 + 1024 > dev.smem_optin:
        pytest.skip(f"{W} columns do not fit this device's shared memory per block")
    p = plan(dev, H, W)
    if p.coresident is None:
        pytest.skip(f"co-residency of {W} columns on this device is too close to call")
    assert p.grid > dev.sms or rows == "short"
    run("mixed", H - 1, W - 1, seed, p, f"co-residency {H}x{W}", extra=(0, 6), variant=-1)


@pytest.mark.parametrize("side", ["below", "above"])
def test_automatic_flat8_choice(side):
    """Automatic variant: the ping-pong pair (16 rowcap stride bytes) just below / above 0.95 x L2 picks flat-4
    (variant 10) / flat-8 (variant 11), both on the ping-pong step."""
    dev = device()
    W = 400
    H = flat8_height(dev, W) - (1 if side == "below" else 0)
    p = plan(dev, H, W)
    if not p.pp:
        pytest.skip(f"{H} rows exceed the ping-pong step on this device before the L2 threshold")
    assert p.variant == (11 if side == "above" else 10)
    run("mixed", H - 1, W - 1, 6000, p, f"auto variant {side} {H}x{W}", extra=(1, 8), variant=-1, engine=0)


# ------------------------------------------------------------------ the shared-memory node kernel
def _resident(it, engine):
    g = gpu_lp(it, engine)
    g.simplex()
    return g


@pytest.mark.parametrize("W", [17, 60])
@pytest.mark.parametrize("edge", ["fits", "past"])
def test_resident_engine_cut_over(edge, W):
    """Engine 4 at the largest height the node kernel's shared memory takes runs there; one row more falls back to the
    fused step, and both match the oracle."""
    dev = device()
    H = resident_rows(dev, W) + (1 if edge == "past" else 0)
    it, o = solved("mixed", H - 1, W - 1, 7000 + W)
    g = _resident(it, 4)
    assert_lp_parity(g, o, f"resident {edge} {H}x{W}")
    print(f"resident {edge} {H}x{W}: engine {g.lastStatus.engine}")
    assert g.lastStatus.engine == (4 if edge == "fits" else 2)
    g.close()


@pytest.mark.parametrize("H,W,engine,seed", [(256, 64, 4, 7164), (145, 113, 2, 7300)])
def test_auto_engine_area_cut_over(H, W, engine, seed):
    """The automatic engine takes the node kernel up to H x W = 16 384 entries and the fused step past that (both
    shapes fit the node kernel's shared memory)."""
    dev = device()
    assert H * W in (16384, 16385) and H <= resident_rows(dev, W)
    it, o = solved("mixed", H - 1, W - 1, seed)
    g = _resident(it, 0)
    assert_lp_parity(g, o, f"auto {H}x{W}")
    assert g.lastStatus.engine == engine
    g.close()


def test_resident_solve_past_the_log_head():
    """A resident solve of more than 64 pivots (NODE_LOG_HEAD): the log is read back from the device buffer."""
    it, o = solved("mixed", 120, 150, 7200, (10,))
    g = _resident(it, 4)
    assert_lp_parity(g, o, "resident 121x151")
    st = g.lastStatus
    assert st.engine == 4 and st.phase1_pivots + st.phase2_pivots > 64, (st.engine, st.phase1_pivots, st.phase2_pivots)
    g.close()


def test_branch_and_cut_across_the_shared_memory_limit():
    """Knapsack whose root tableau sits two rows under the node kernel's limit: shallow nodes run in shared memory,
    deeper ones (more cut rows) in node slots or on the HBM path; the node log, the final tableau and the index arrays
    match the oracle's."""
    import jslpsolver_b200 as J
    from jslpsolver_b200 import problems
    from oracle import ref_model
    dev = device()
    n_items = 30
    n_cons = resident_rows(dev, n_items + 1) - 2 - n_items - 1
    jm = problems.knapsack_mip_model(n_items, n_cons, seed=8)
    max_nodes = 300
    osol = ref_model.solve_full(jm, fast_cycles=True, node_log=1 << 20, max_nodes=max_nodes)
    inst = J.Model().loadJson(jm)
    inst.max_nodes = max_nodes
    inst.tableau.max_spec_batch = 8
    inst.solve()
    gt = inst.tableau
    assert gt.height >= n_cons + n_items + 1
    onl, gnl = osol.tableau.node_log(), gt.node_log()
    assert gnl.shape == onl.shape, (gnl.shape, onl.shape)
    for i in range(len(onl)):
        a, b = gnl[i], onl[i]
        ok = all(a[k] == b[k] for k in (0, 1, 2, 4, 5, 7)) and same_bits(a[6], b[6]) and (not b[2] or same_bits(a[3], b[3]))
        assert ok, f"node {i}: gpu={a.tolist()} oracle={b.tolist()}"
    st = osol.state
    assert gt.branchAndCutIterations == st.bncIterations
    assert (gt.feasible, gt.bounded) == (bool(st.feasible), bool(st.bounded))
    assert same_bits(gt.matrix2d(), osol.tableau.matrix())
    assert np.array_equal(gt.varIndexByRow, osol.tableau.maps()[0])
    assert np.array_equal(gt.varIndexByCol, osol.tableau.maps()[1])
    b = gt.lastBnbStatus
    print(f"knapsack {n_items}x{n_cons}: nodes {len(onl)} node kernel {b.node_kernel_ms:.3f} ms slot pivots {b.slot_pivots}")
    assert b.node_kernel_ms > 0 and b.slot_pivots > 0, (b.node_kernel_ms, b.slot_pivots)
    gt.close()


# ------------------------------------------------------------------ value edges at those geometries
# (variant, ping-pong): the default flat variant, a per-row variant, the in-place step; one CTA per SM, 17 rows per CTA
VALUE_STEPS = {"flat4": (10, True), "t128": (5, True), "in_place": (10, False)}


@pytest.mark.parametrize("step", list(VALUE_STEPS))
@pytest.mark.parametrize("family", ["ties", "thresholds"])
def test_value_edges(family, step):
    dev = device()
    variant, pingpong = VALUE_STEPS[step]
    nt = STEP_VARIANTS[variant][0]
    G = dev.sms - (2 if pingpong else 0)
    H = 17 * G
    if family == "ties":
        W = 8 * nt + 60
        extra = (G, nt, 20)
    else:
        W, extra = 120, ()
    p = plan(dev, H, W, variant, grid_per_sm=1, pingpong=pingpong)
    assert p.pp == pingpong and p.rows == 17 and p.G == G
    st = run(family, H - 1, W - 1, 8000 + variant, p, f"{family} {step} {H}x{W}", extra=extra, grid_per_sm=1,
             pingpong=pingpong)
    assert st.phase1_pivots + st.phase2_pivots > 0
