// jslpsolver_b200/csrc/jslp_step.cuh -- the fused pivot step (included by jslp_kernels.cuh).
//
// One launch == one simplex iteration on a tableau that lives in HBM / L2.  Two instantiations of
// k_pivot_step<threads, occupancy, rows per pass, prefetch, PP>:
//
// PP = true, the ping-pong step (every step of a solve without optional objectives and with at most 32
// rows per row CTA).  The tableau is read from T.M and written to T.M2, then the two pointers are swapped
// in the device descriptor, so old values stay readable for the whole launch and the NEXT pivot is chosen
// beside the streaming, not after it.  Grid = G row CTAs + 2 selector CTAs.
//   head   TMA (cp.async.bulk + mbarrier) pulls the pivot row -- staged already normalised by the previous
//          launch (simplex.ts:352-364, lazy flush 380-382) -- into shared memory; it is issued before
//          anything else because it needs only kernel parameters.  The pivot record (one 128-byte line) and
//          the descriptor are requested together: the head is one L2 round trip deep.
//   row CTA  last warp = look-ahead of the next pivot on this CTA's rows, computed from OLD values with
//          new_entry(): ratio-test partial (phase 2, simplex.ts:271-296) or most negative right-hand side
//          (phase 1, 38-54), published as one self-validating 16-byte message.  All warps then stream the
//          row block: M2[r][c] = M[r][c] - coef_r * prow[c] (two roundings, simplex.ts:379), pivot column
//          entry -coef_r / q (385), pivot row rewrite.
//   selector S1  polls the G messages and reduces them (redux.sync on order-preserving keys) to the next
//          leaving row; phase 2: derives that row and the cost row from the old tableau, prices the pivot
//          AFTER next (140-219), writes the record, swaps labels, flips the descriptor
//          (cta_selector_decide).  Phase 1, and phase-2 pivots without a priced successor: also picks the
//          entering column (56-76) or runs pricing + ratio test on derived values, and stages the next
//          pivot row itself (cta_selector_decide_full).
//   selector S2  (phase 2) stages the normalised next pivot row into the prow side buffer.
//
// PP = false, the in-place step (two-kernel engine, optional objectives 393-412, very tall tableaux):
// rank-1 update in place; with do_select the last CTA to finish (atomic ticket) reduces look-ahead partials
// (cta_tail_lookahead) or runs the generic selection (cta_select).
//
// Code layout matters as much as instruction count here (DESIGN.md section 6): hot paths are inlined and
// contiguous, rarely taken ones are __noinline__.
#pragma once
// (included inside namespace jslp)

// ---- pricing of the pivot AFTER the staged one (phase 2, no optional objectives) -------------
// cta_price_scan<true> (jslp_kernels.cuh) prices the cost row as the staged pivot will leave
// it, with the very expression update_rows evaluates for row 0, so the decision is bit-identical
// to pricing afterwards; one L2 round trip whatever the number of pricing batches.

// Generic entry: the pivot is already staged (prow side buffer, labels swapped, rec filled).
__device__ __noinline__ void cta_price_next(const TabDev &T, Rec *rec, SelSmem &s) {
    const int cstar = rec->c;
    const double q = rec->q;
    const double coef0 = ldg_cg(T.M + cstar);
    int found, neg;
    cta_price_scan<true>(T, s, T.M, T.prow, q, coef0, cstar, T.vcol[cstar], &found, &neg);
    if (threadIdx.x == 0) { rec->next_c = found; rec->next_neg = neg; }
}

// upd_entry on a column pair of a row with a non-zero pivot-column entry; pc = the pair holds the pivot column (the
// odd half when codd), whose entry is divided once.
__device__ __forceinline__ double2 upd2(double2 old, double2 f, double coef, bool pc, int codd, double q) {
    double2 nv = make_double2(upd_entry(old.x, coef, f.x, false, q), upd_entry(old.y, coef, f.y, false, q));
    if (pc) {
        const double pv = upd_entry(0.0, coef, 0.0, true, q);
        if (codd) nv.y = pv; else nv.x = pv;
    }
    return nv;
}

// ---- body: rank-1 update of rows [r0, r0+nr) ---------------------------------------------------
// RC rows are processed together (RC independent 128-bit loads in flight per thread); PF adds a
// software prefetch of the next column pair's RC loads before the current pair is stored.
template <int RC, bool PF>
__device__ __noinline__ void update_rows(const TabDev &T, const double *frow, int r0, int nr, int rstar,
                                            int cstar, double q, bool do_opt) {
    const int tid = threadIdx.x, NT = blockDim.x;
    const size_t stride = (size_t)T.stride;
    const int npair = T.stride >> 1;
    double *const Mb = T.M;
    const double *const pcol = T.pcol;
    const double2 *frow2 = reinterpret_cast<const double2 *>(frow);
    const int cpair = cstar >> 1, codd = cstar & 1;
    for (int rb = r0; rb < r0 + nr; rb += RC) {
        double coef[RC];
        bool act[RC];
        bool any = false;
#pragma unroll
        for (int j = 0; j < RC; j++) {
            const int r = rb + j;
            const bool valid = (r < r0 + nr) && (r != rstar);
            coef[j] = valid ? pcol[r] : 0.0;
            act[j] = valid && nz16(coef[j]);
            any |= act[j];
            // simplex.ts:389-391 is dead code in the reference (same predicate as :371): a pivot-column
            // entry with |x| <= 1e-16 is left untouched.
        }
        double *const base = Mb + (size_t)rb * stride;
        if (any && !PF) {
            for (int c2 = tid; c2 < npair; c2 += NT) {
                const double2 f = frow2[c2];
                const bool z0 = nz16(f.x), z1 = nz16(f.y);
                const bool pc = (c2 == cpair);
                if (!z0 && !z1 && !pc) continue;  // zero pivot-row entries touch nothing (nonZeroColumns)
                double2 old[RC];
#pragma unroll
                for (int j = 0; j < RC; j++)
                    if (act[j]) old[j] = ld_v2(base + j * stride + 2 * c2);
#pragma unroll
                for (int j = 0; j < RC; j++)
                    if (act[j]) st_v2(base + j * stride + 2 * c2, upd2(old[j], f, coef[j], pc, codd, q));
            }
        } else if (any) {
            int c2 = tid;
            double2 f = make_double2(0.0, 0.0), old[RC];
            if (c2 < npair) {
                f = frow2[c2];
#pragma unroll
                for (int j = 0; j < RC; j++)
                    if (act[j]) old[j] = ld_v2(base + j * stride + 2 * c2);
            }
            while (c2 < npair) {
                const int n2 = c2 + NT;
                double2 fn = make_double2(0.0, 0.0), oldn[RC];
                if (n2 < npair) {
                    fn = frow2[n2];
#pragma unroll
                    for (int j = 0; j < RC; j++)
                        if (act[j]) oldn[j] = ld_v2(base + j * stride + 2 * n2);
                }
                const bool z0 = nz16(f.x), z1 = nz16(f.y);
                const bool pc = (c2 == cpair);
                if (z0 || z1 || pc) {
#pragma unroll
                    for (int j = 0; j < RC; j++)
                        if (act[j]) st_v2(base + j * stride + 2 * c2, upd2(old[j], f, coef[j], pc, codd, q));
                }
                c2 = n2;
                f = fn;
#pragma unroll
                for (int j = 0; j < RC; j++) old[j] = oldn[j];
            }
        }
        if (rstar >= rb && rstar < rb + RC && rstar < r0 + nr) {
            double *dst = Mb + rstar * stride;
            for (int c = tid; c < T.stride; c += NT) dst[c] = frow[c];
        }
    }
    if (do_opt) {  // simplex.ts:393-412 (exact-zero predicates)
        for (int o = 0; o < T.nOpt; o++) {
            const double coefficient = T.optcoef[o];
            if (coefficient == 0.0) continue;
            double *rc = T.opt + (size_t)o * stride;
            for (int c = tid; c < T.W; c += NT) {
                const double v0 = frow[c];
                double v = rc[c];
                bool wr = false;
                if (v0 != 0.0) { v = __dsub_rn(v, __dmul_rn(coefficient, v0)); wr = true; }
                if (c == cstar) { v = ddiv(-coefficient, q); wr = true; }
                if (wr) rc[c] = v;
            }
        }
    }
}


// ---- look-ahead: ratio-test partial of this CTA's rows against the next entering column ---------
// One row per thread (nr <= blockDim.x); col/rhs are the UPDATED entries of that row.
__device__ __forceinline__ void cta_ratio_partial(const TabDev &T, SelSmem &s, int r0, int nr, bool have, double col,
                                                  double rhs, int isneg) {
    const int tid = threadIdx.x;
    VI m = {INFINITY, INT_MAX};
    int dmin = INT_MAX, cnt = 0;
    if (have) {
        const int r = r0 + tid;
        T.pcol[r] = col;  // pivot column of the next pivot (this CTA is the only reader of these entries)
        ratio_step(r, col, rhs, isneg, T.prec, dmin, m, cnt);
    }
    block_reduce_ratio(dmin, m, cnt, s.red);
    const int dall = dmin;
    const VI mall = m;
    Part *p = T.part + blockIdx.x;
    if (tid == 0) { p->minq = mall.v; p->minr = mall.i; p->dmin = dall; p->cnt = cnt; }
    (void)nr;
}

// ---- tail (look-ahead): reduce the partials, stage the next pivot, price the one after it -------
// Two dependent L2 round trips: (1) the partials, (2) everything that depends on the leaving row.
__device__ __noinline__ void cta_tail_lookahead(const TabDev &T, Rec *rec, SelSmem &s, int G, int cn, int isneg, int log_n) {
    const int tid = threadIdx.x, NT = blockDim.x;
    if (cn == 0) {  // nothing prices in: optimal (simplex.ts:265-269); setEvaluation is done on the host
        if (tid == 0) { rec->status = ST_OPTIMAL; rec->phase = 2; rec->has_pivot = 0; rec->eval_raw = ldg_cg(T.M); }
        return;
    }
    const VI init = {INFINITY, INT_MAX};
    VI m = init;
    int dmin = INT_MAX, cnt = 0;
    const Part *parts = T.part;
    for (int b0 = 0; b0 < G; b0 += 4 * NT) {  // all loads of a pass first: one L2 round trip
        double pq[4];
        int4 iv[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int b = b0 + tid + k * NT;
            if (b < G) {
                pq[k] = __ldcg(&parts[b].minq);
                iv[k] = __ldcg(reinterpret_cast<const int4 *>(&parts[b].minr));
            }
        }
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int b = b0 + tid + k * NT;
            if (b >= G) continue;
            const int pr = iv[k].x, pd = iv[k].y;
            cnt += iv[k].z;
            if (pd < dmin) dmin = pd;
            if (pr != INT_MAX && (pq[k] < m.v || (pq[k] == m.v && pr < m.i))) { m.v = pq[k]; m.i = pr; }
        }
    }
    block_reduce_ratio(dmin, m, cnt, s.red);
    const int dall = dmin;
    const VI mall = m;
    int rstar;
    if (dall != INT_MAX) rstar = dall;
    else if (mall.i != INT_MAX) rstar = mall.i;
    else {  // unbounded (simplex.ts:298-303)
        if (tid == 0) {
            rec->status = ST_UNBOUNDED; rec->phase = 2; rec->has_pivot = 0;
            rec->unbounded_var = T.vcol[cn];
            rec->eval_raw = ldg_cg(T.M);
        }
        return;
    }
    // round trip 2: pivot element, cost-row entry, labels, raw pivot row, first pricing batch
    const double *rowp = T.M + (size_t)rstar * T.stride;
    const double q = ldg_cg(rowp + cn);
    const double coef0 = ldg_cg(T.M + cn);
    const int leaving = T.vrow[rstar];
    const int entering = T.vcol[cn];
    cta_copy_row(T.prow, rowp, T.W, T.stride);
    int found, neg;
    cta_price_scan<true>(T, s, T.M, rowp, q, coef0, cn, leaving, &found, &neg);
    if (tid == 0) {
        stage_pivot(T, rec, log_n, 2, rstar, cn, leaving, entering, q, isneg, flush_flag(cnt, q), found, 0);
        rec->next_neg = neg;
    }
}

// =================================== ping-pong step ===================================================
// The tableau is read from T.M and the updated tableau written to T.M2 (same traffic as in place:
// every element is read once and written once), then the two pointers are swapped in the device
// descriptor.  Because the old values stay readable for the whole launch there is no in-place
// hazard left, and the serial work of choosing the next pivot moves OFF the critical path:
//   * every row CTA publishes its look-ahead ratio-test partial BEFORE it starts streaming;
//   * one extra CTA (the selector) waits for those G partials, reduces them to the next leaving
//     row, derives that row and the cost row as this pivot will leave them from the OLD tableau
//     (new_entry), stages the next pivot, prices the pivot after it and flips the descriptor --
//     all while the row CTAs are still streaming.  The launch ends when the streaming ends.

// dst rows [r0, r0+nr) = pivot applied to src rows (simplex.ts:352-391); every pair is written.
template <int RC, bool PF>
__device__ __forceinline__ void update_rows_pp(const double *src, double *dst, int stride_i, const double *frow,
                                               const double *s_coef, int r0, int nr, int rstar, int cstar, double q) {
    const int tid = threadIdx.x, NT = blockDim.x;
    const size_t stride = (size_t)stride_i;
    const int npair = stride_i >> 1;
    const double2 *frow2 = reinterpret_cast<const double2 *>(frow);
    const int cpair = cstar >> 1, codd = cstar & 1;
    for (int rb = r0; rb < r0 + nr; rb += RC) {
        double coef[RC];
        bool valid[RC], act[RC], isp[RC];
#pragma unroll
        for (int j = 0; j < RC; j++) {
            const int r = rb + j;
            valid[j] = r < r0 + nr;
            isp[j] = valid[j] && r == rstar;
            coef[j] = (valid[j] && !isp[j]) ? s_coef[r - r0] : 0.0;
            act[j] = valid[j] && !isp[j] && nz16(coef[j]);
        }
        const double *sb = src + (size_t)rb * stride;
        double *db = dst + (size_t)rb * stride;
        auto emit = [&](int c2, const double2 f, const double2 *old) {
            const bool pc = (c2 == cpair);
#pragma unroll
            for (int j = 0; j < RC; j++) {
                if (!valid[j]) continue;
                double2 nv;
                if (isp[j]) nv = f;                                                   // normalised pivot row
                else if (act[j]) nv = upd2(old[j], f, coef[j], pc, codd, q);  // rank-1 update
                else nv = old[j];  // untouched row, tiny pivot-column entry included (simplex.ts:371; :389-391 is dead)
                st_v2(db + j * stride + 2 * c2, nv);
            }
        };
        if (!PF) {
            for (int c2 = tid; c2 < npair; c2 += NT) {
                double2 old[RC];
#pragma unroll
                for (int j = 0; j < RC; j++)
                    if (valid[j] && !isp[j]) old[j] = ld_v2_dead(sb + j * stride + 2 * c2);
                emit(c2, frow2[c2], old);
            }
        } else {  // software prefetch: the next pair's RC loads are in flight while this pair is stored
            int c2 = tid;
            double2 old[RC];
            if (c2 < npair) {
#pragma unroll
                for (int j = 0; j < RC; j++)
                    if (valid[j] && !isp[j]) old[j] = ld_v2_dead(sb + j * stride + 2 * c2);
            }
            while (c2 < npair) {
                const int n2 = c2 + NT;
                double2 oldn[RC];
                if (n2 < npair) {
#pragma unroll
                    for (int j = 0; j < RC; j++)
                        if (valid[j] && !isp[j]) oldn[j] = ld_v2_dead(sb + j * stride + 2 * n2);
                }
                emit(c2, frow2[c2], old);
                c2 = n2;
#pragma unroll
                for (int j = 0; j < RC; j++) old[j] = oldn[j];
            }
        }
    }
}

// Flat form of update_rows_pp for tableaux whose rows are short next to the CTA (config 5: 520 column pairs
// against 256 threads -- the per-row loop above runs three dependent load->store rounds per pass, the third
// with 8 active threads).  Rows are padded to the stride, so the CTA's row block is ONE contiguous run of
// nr * stride/2 column pairs: thread t owns pairs t, t+NT, t+2NT, ... of that run, K of them in flight plus
// the next K prefetched, whatever the row length.  (row, pair-in-row) is only needed to pick the pivot-row
// entry and the row's coefficient from shared memory and advances incrementally.
template <int K>
__device__ __forceinline__ void update_rows_pp_flat(const double *src, double *dst, int stride_i, const double *frow,
                                                    const double *s_coef, int r0, int nr, int rstar, int cstar, double q) {
    const int tid = threadIdx.x, NT = blockDim.x;
    const int npair = stride_i >> 1;
    const double2 *frow2 = reinterpret_cast<const double2 *>(frow);
    const int cpair = cstar >> 1, codd = cstar & 1;
    const int total = nr * npair;
    const double *sb = src + (size_t)r0 * stride_i;
    double *db = dst + (size_t)r0 * stride_i;
    const int prel = rstar - r0;  // pivot row relative to the block (outside [0, nr) when it is not ours)
    int row = 0, c2 = tid;
    while (c2 >= npair) { c2 -= npair; row++; }
    double2 cur[K], nxt[K];
#pragma unroll
    for (int j = 0; j < K; j++) {
        const int idx = tid + j * NT;
        if (idx < total) cur[j] = ld_v2_dead(sb + 2 * (size_t)idx);
    }
    for (int i0 = tid; i0 < total; i0 += K * NT) {
#pragma unroll
        for (int j = 0; j < K; j++) {
            const int idx = i0 + (K + j) * NT;
            if (idx < total) nxt[j] = ld_v2_dead(sb + 2 * (size_t)idx);
        }
#pragma unroll
        for (int j = 0; j < K; j++) {
            const int idx = i0 + j * NT;
            if (idx < total) {
                const double2 f = frow2[c2];
                double2 nv;
                if (row == prel) nv = f;  // normalised pivot row
                else {
                    const double coef = s_coef[row];
                    nv = nz16(coef) ? upd2(cur[j], f, coef, c2 == cpair, codd, q) : cur[j];
                }
                st_v2(db + 2 * (size_t)idx, nv);
            }
            c2 += NT;
            while (c2 >= npair) { c2 -= npair; row++; }
        }
#pragma unroll
        for (int j = 0; j < K; j++) cur[j] = nxt[j];
    }
}

// ---- look-ahead partials as self-validating 16-byte messages -------------------------------------
// A row CTA publishes the ratio-test partial of its rows with ONE 128-bit store; selectors poll the
// slots.  Word B carries a 24-bit sequence tag (launch + 1) and a 16-bit checksum of word A, so a
// reader accepts a slot only when both halves belong to the same publication: no fence, no atomic,
// no barrier on the publishing side.  Rows are encoded relative to the CTA's first row (<= 254 rows).
__device__ __forceinline__ unsigned int part_chk(unsigned long long a, unsigned int seq) {
    const unsigned long long x = a ^ (a >> 16) ^ (a >> 32) ^ (a >> 48);
    return (unsigned int)((x ^ seq ^ (seq >> 16)) & 0xffffull);
}
__device__ __forceinline__ void part_publish(Part *slot, double minq, int minr_rel, int dmin_rel, int cnt, unsigned int seq) {
    const unsigned long long a = (unsigned long long)__double_as_longlong(minq);
    const unsigned long long b = (unsigned long long)(seq & 0xffffffu) | ((unsigned long long)(cnt & 0xff) << 24) |
                                 ((unsigned long long)(minr_rel & 0xff) << 32) | ((unsigned long long)(dmin_rel & 0xff) << 40) |
                                 ((unsigned long long)part_chk(a, seq & 0xffffffu) << 48);
    asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(slot), "l"(a), "l"(b) : "memory");
}
// raw 16-byte probe of a slot / validation of a probe against the publication tagged `seq`
__device__ __forceinline__ void part_probe(const Part *slot, unsigned long long *a, unsigned long long *b) {
    asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(*a), "=l"(*b) : "l"(slot) : "memory");
}
__device__ __forceinline__ bool part_decode(unsigned long long a, unsigned long long b, unsigned int seq, double *minq,
                                            int *minr_rel, int *dmin_rel, int *cnt) {
    if ((unsigned int)(b & 0xffffffull) != (seq & 0xffffffu)) return false;
    if ((unsigned int)(b >> 48) != part_chk(a, seq & 0xffffffu)) return false;
    *minq = __longlong_as_double((long long)a);
    *cnt = (int)((b >> 24) & 0xff);
    *minr_rel = (int)((b >> 32) & 0xff);
    *dmin_rel = (int)((b >> 40) & 0xff);
    return true;
}
__device__ __forceinline__ bool part_try_read(const Part *slot, unsigned int seq, double *minq, int *minr_rel,
                                              int *dmin_rel, int *cnt) {
    unsigned long long a, b;
    part_probe(slot, &a, &b);
    return part_decode(a, b, seq, minq, minr_rel, dmin_rel, cnt);
}

// Selector side: wait for all G partials of this launch and reduce them (simplex.ts:271-296 over the
// whole column).  Returns false on a watchdog timeout (a lost publication must not hang the GPU).
__device__ __forceinline__ bool cta_collect_partials(const TabDev &T, SelSmem &s, int G, unsigned int seq, int *rnext, int *cnt_out) {
    const int tid = threadIdx.x, NT = blockDim.x;
    const int base = T.H / G, rem = T.H % G;
    VI m = {INFINITY, INT_MAX};
    int dmin = INT_MAX, cnt = 0, ok = 1;
    const long long tstart = clock64();
    for (int b0 = 0; b0 < G && ok; b0 += 4 * NT) {  // up to four slots per thread are polled together
        unsigned int pending = 0;
#pragma unroll
        for (int k = 0; k < 4; k++)
            if (b0 + tid + k * NT < G) pending |= 1u << k;
        while (pending) {
            double pq[4];
            int mr[4], dr[4], pc[4];
            bool got[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                got[k] = false;
                if (pending & (1u << k)) got[k] = part_try_read(T.part + b0 + tid + k * NT, seq, &pq[k], &mr[k], &dr[k], &pc[k]);
            }
#pragma unroll
            for (int k = 0; k < 4; k++) {
                if (!got[k]) continue;
                pending &= ~(1u << k);
                const int b = b0 + tid + k * NT;
                const int r0 = b * base + min(b, rem);
                cnt += pc[k];
                if (dr[k] != 255 && r0 + dr[k] < dmin) dmin = r0 + dr[k];
                if (mr[k] != 255) {
                    const int pr = r0 + mr[k];
                    if (pq[k] < m.v || (pq[k] == m.v && pr < m.i)) { m.v = pq[k]; m.i = pr; }
                }
            }
            if (pending) {
                __nanosleep(20);
                if (clock64() - tstart > 4000000000LL) { ok = 0; break; }
            }
        }
    }
    block_reduce_ratio_rx(dmin, m, cnt, ok, s.red);
    if (!ok) return false;
    *rnext = dmin != INT_MAX ? dmin : (m.i != INT_MAX ? m.i : -1);
    *cnt_out = cnt;
    return true;
}

// Selector S1 of a ping-pong step: decides the next pivot, prices the one after it, writes the
// record, swaps the labels and flips the descriptor.  frow = normalised row of the executing pivot.
__device__ __forceinline__ void cta_selector_decide(TabDev *Tp, const TabDev &T, Rec *rec, SelSmem &s, const double *frow, int G,
                                    int rstar, int cstar, double q, int cn, int isneg, int launch, int p2, int log_n,
                                    bool stop_after, long long *ts) {
    const int tid = threadIdx.x, NT = blockDim.x;
    const double *src = T.M;
    const double coef0 = ldg_cg(src + cstar);  // cost-row entry of the executing pivot's column
    auto flip = [&]() {  // the updated tableau becomes the current one
        Tp->M = T.M2;
        Tp->M2 = T.M;
    };
    if (cn == 0 || stop_after) {  // optimal after this pivot (simplex.ts:265-269), or a replay stop
        if (tid == 0) {
            rec->done = launch + 1; rec->p2 = p2 + 1; rec->has_pivot = 0;
            if (!stop_after) {
                rec->status = ST_OPTIMAL; rec->phase = 2;
                rec->eval_raw = new_entry(ldg_cg(src), false, coef0, frow[0], false, q);
            }
            flip();
        }
        return;
    }
    int rnext, cnt;
    if (!cta_collect_partials(T, s, G, (unsigned int)(launch + 1), &rnext, &cnt)) {
        if (tid == 0) { rec->status = ST_ERROR; rec->has_pivot = 0; }
        return;
    }
    if (tid == 0) ts[0] = ts[1] = clock64();
    if (rnext < 0) {  // unbounded (simplex.ts:298-303)
        if (tid == 0) {
            rec->done = launch + 1; rec->p2 = p2 + 1; rec->has_pivot = 0;
            rec->status = ST_UNBOUNDED; rec->phase = 2;
            rec->unbounded_var = T.vcol[cn];
            rec->eval_raw = new_entry(ldg_cg(src), false, coef0, frow[0], false, q);
            flip();
        }
        return;
    }
    // Entries of the next pivot row / the cost row as the executing pivot leaves them, derived from
    // the OLD tableau.  First pass: only the leading columns (one per thread) -- the reference's
    // partial pricing almost always stops in the first batches.
    const double *rowp = src + (size_t)rnext * T.stride;
    const bool is_prow = rnext == rstar;
    const double coef_r = is_prow ? 0.0 : ldg_cg(rowp + cstar);
    const int leaving = T.vrow[rnext];
    const int entering = T.vcol[cn];
    const double rv_cn = ldg_cg(rowp + cn), cv_cn = ldg_cg(src + cn);
    constexpr int K1 = 4;  // columns per thread in the first pass (c = tid + k*NT)
    double rv1[K1], cv1[K1];
#pragma unroll
    for (int k = 0; k < K1; k++) {
        const int c = tid + k * NT;
        rv1[k] = (c >= 1 && c < T.W) ? ldg_cg(rowp + c) : 0.0;
        cv1[k] = (c >= 1 && c < T.W) ? ldg_cg(src + c) : 0.0;
    }
    const double qn = new_entry(rv_cn, is_prow, coef_r, frow[cn], cn == cstar, q);      // next pivot element
    const double coef0n = new_entry(cv_cn, false, coef0, frow[cn], cn == cstar, q);     // its cost-row entry
    const int bsz = T.use_partial ? T.batch_size : max(1, T.W - 1);
    // batches that lie entirely inside the first pass (columns 1 .. K1*NT-1)
    const int covered = min(T.W - 1, K1 * NT - 1);
    const int nfull = (covered == T.W - 1) ? INT_MAX : covered / bsz;
    int found = 0, neg = 0;
    {
        PriceAcc acc;
        price_init(acc, T.prec);
#pragma unroll
        for (int k = 0; k < K1; k++) {
            const int c1 = tid + k * NT;
            if (c1 >= 1 && c1 < T.W && (c1 - 1) / bsz < nfull) {
                const double ur = new_entry(rv1[k], is_prow, coef_r, frow[c1], c1 == cstar, q);
                const double uc = new_entry(cv1[k], false, coef0, frow[c1], c1 == cstar, q);
                const double nc = priced_cost(uc, ur, coef0n, c1 == cn, qn);
                int label = -1;
                if (T.unres != nullptr && nc < 0) label = (c1 == cn) ? leaving : T.vcol[c1];
                price_consider(T, acc, c1, nc, label, bsz);
            }
        }
        price_finish_rx(T, s, acc, &found, &neg);
    }
    if (tid == 0) ts[2] = clock64();
    if (found == 0 && nfull != INT_MAX) {  // nothing in the leading batches: price the whole row
        PriceAcc acc;
        price_init(acc, T.prec);
        for (int c0 = 1; c0 < T.W; c0 += 8 * NT) {
            double rv[8], cv[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int c = c0 + tid + k * NT;
                rv[k] = c < T.W ? ldg_cg(rowp + c) : 0.0;
                cv[k] = c < T.W ? ldg_cg(src + c) : 0.0;
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int c = c0 + tid + k * NT;
                if (c >= T.W) continue;
                const double ur = new_entry(rv[k], is_prow, coef_r, frow[c], c == cstar, q);
                const double uc = new_entry(cv[k], false, coef0, frow[c], c == cstar, q);
                const double nc = priced_cost(uc, ur, coef0n, c == cn, qn);
                int label = -1;
                if (T.unres != nullptr && nc < 0) label = (c == cn) ? leaving : T.vcol[c];
                price_consider(T, acc, c, nc, label, bsz);
            }
        }
        price_finish_rx(T, s, acc, &found, &neg);
    }
    if (tid == 0) {
        // the staging selector writes the normalised row
        stage_pivot(T, rec, log_n, 2, rnext, cn, leaving, entering, qn, isneg, flush_flag(cnt, qn), found, 1);
        rec->next_neg = neg;
        rec->done = launch + 1; rec->p2 = p2 + 1;
        flip();
    }
}

// Waits for the message tagged `seq` in `slot` (handshakes between the two selector CTAs).
__device__ __forceinline__ void part_wait(const Part *slot, unsigned int seq) {
    double dq;
    int d1, d2, d3;
    const long long tstart = clock64();
    while (!part_try_read(slot, seq, &dq, &d1, &d2, &d3)) {
        __nanosleep(20);
        if (clock64() - tstart > 4000000000LL) break;
    }
}

// Stages the NEXT pivot (rnext, cn) for the launch after this one: its row as the executing pivot (rstar, cstar, q,
// normalised row frow) leaves it, derived from the old tableau (new_entry) and already normalised (norm_entry), so
// that no CTA of the next launch divides it again, goes into the prow side buffer, zero padded.  cnt = non-zero
// entries of the next pivot column.  Returns the next pivot element.
__device__ __forceinline__ double stage_next_row(const TabDev &T, const double *frow, int rstar, int cstar, double q,
                                                 int rnext, int cn, int cnt) {
    const int tid = threadIdx.x, NT = blockDim.x;
    const double *rowp = T.M + (size_t)rnext * T.stride;
    const bool is_prow = rnext == rstar;
    const double coef_r = is_prow ? 0.0 : ldg_cg(rowp + cstar);
    const double qn = new_entry(ldg_cg(rowp + cn), is_prow, coef_r, frow[cn], cn == cstar, q);
    const bool flushn = flush_flag(cnt, qn);
    for (int c0 = 0; c0 < T.stride; c0 += 8 * NT) {
        double rv[8];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = c0 + tid + k * NT;
            rv[k] = c < T.W ? ldg_cg(rowp + c) : 0.0;
        }
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = c0 + tid + k * NT;
            if (c >= T.stride) continue;
            T.prow[c] = c < T.W ? norm_entry(new_entry(rv[k], is_prow, coef_r, frow[c], c == cstar, q), c == cn, qn, flushn) : 0.0;
        }
    }
    return qn;
}

// Selector of a ping-pong step that executes a PHASE-1 pivot (rstar, cstar, q), or a phase-2 pivot whose
// successor has not been priced.  In phase 1 the row CTAs publish,
// before they stream, the most negative right-hand side their rows will have after this pivot; this
// CTA reduces those to the next leaving row (simplex.ts:38-54), derives that row and the cost row as
// this pivot leaves them from the OLD tableau (new_entry), picks the entering column (56-76), counts
// the non-zero entries of the next pivot column (lazy-flush flag), stages the next pivot row already
// normalised and flips the descriptor -- all while the row CTAs stream.  When no infeasible row is
// left it opens phase 2 itself (pricing 129-269, ratio test 271-296), again from derived values.
__device__ __noinline__ void cta_selector_decide_full(TabDev *Tp, const TabDev &T, Rec *rec, SelSmem &s, const double *frow, int G,
                                         int rstar, int cstar, double q, int launch, int phase_exec, int pcount,
                                         int log_n, bool stop_after, int only_phase) {
    const int tid = threadIdx.x, NT = blockDim.x;
    const double *src = T.M;
    const size_t stride = (size_t)T.stride;
    const int W = T.W, H = T.H;
    const double prec = T.prec;
    const double coef0 = ldg_cg(src + cstar);  // cost-row entry of the executing pivot's column
    const unsigned int seq = (unsigned int)(launch + 1);
    auto flip = [&]() {  // the updated tableau becomes the current one
        Tp->M = T.M2;
        Tp->M2 = T.M;
    };
    auto finish = [&](int status, int phase, int unb) {  // no further pivot: final record (tid 0 only)
        rec->done = launch + 1; rec->has_pivot = 0;
        if (phase_exec == 1) rec->p1 = pcount + 1; else rec->p2 = pcount + 1;
        if (status != ST_RUNNING) {
            rec->status = status;
            if (phase) rec->phase = phase;
            if (unb >= 0) rec->unbounded_var = unb;
            rec->eval_raw = new_entry(ldg_cg(src), false, coef0, frow[0], false, q);
        }
        flip();
    };
    if (stop_after) {  // replay stop: execute this pivot and select nothing
        if (tid == 0) finish(ST_RUNNING, 0, -1);
        return;
    }
    if (tid == 0) part_wait(T.part + G + 1, seq);  // the other selector's TMA read of prow has landed (it is
                                                   // published within the first microsecond: no wait later)
    // A phase-2 pivot without a priced successor (the first phase-2 pivot of a solve) has no partials:
    // the next pivot is derived below exactly as when phase 1 ends.
    int rnext = -1, cnt_unused;
    if (phase_exec == 1 && !cta_collect_partials(T, s, G, seq, &rnext, &cnt_unused)) {
        if (tid == 0) { rec->status = ST_ERROR; rec->has_pivot = 0; }
        return;
    }
    int phase_next = 1, cn = 0, isneg = 0, cnt = 0;
    const bool has_unres = T.unres != nullptr;
    // non-zero entries of the next pivot column cn as this pivot leaves it (all rows, row 0 included)
    auto count_col = [&]() {
        const double f_cn = frow[cn];
        int n = 0;
        for (int rb = 0; rb < H; rb += 8 * NT) {
            double a[8], cf[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rb + tid + k * NT;
                a[k] = r < H ? ldg_cg(src + (size_t)r * stride + cn) : 0.0;
                cf[k] = (r < H && r != rstar) ? ldg_cg(src + (size_t)r * stride + cstar) : 0.0;
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rb + tid + k * NT;
                if (r < H && nz16(new_entry(a[k], r == rstar, cf[k], f_cn, cn == cstar, q))) n++;
            }
        }
        return block_reduce_int<1>(n, s.red);
    };
    if (rnext >= 0 && T.stride <= 8 * NT) {
        // ---- phase 1 goes on, fast path (two L2 round trips after the partials): the whole derived row
        // rnext fits in eight registers per thread, so the entering-column scan (simplex.ts:56-76), the
        // pivot element and the normalised row staged for the next launch all come from ONE set of loads.
        const double *rowp = src + (size_t)rnext * stride;
        const bool is_prow = rnext == rstar;
        const double coef_r = is_prow ? 0.0 : ldg_cg(rowp + cstar);
        const int leaving = T.vrow[rnext];
        double ur[8], cv[8];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = tid + k * NT;
            ur[k] = c < W ? ldg_cg(rowp + c) : 0.0;
            cv[k] = c < W ? ldg_cg(src + c) : 0.0;
        }
        const VI einit = {-INFINITY, INT_MAX};
        VI e = einit;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = tid + k * NT;
            if (c >= W) continue;
            ur[k] = new_entry(ur[k], is_prow, coef_r, frow[c], c == cstar, q);
            if (c >= 1)
                entering_step(c, ur[k], has_unres && is_unres(T, T.vcol[c]), prec, e,
                              [&] { return new_entry(cv[k], false, coef0, frow[c], c == cstar, q); });
        }
        e = block_reduce_vi_rx<false>(e, einit, s.red);
        if (e.i == INT_MAX) {  // simplex.ts:73-76
            if (tid == 0) finish(ST_INFEASIBLE, 0, -1);
            return;
        }
        cn = e.i;
#pragma unroll
        for (int k = 0; k < 8; k++)
            if (tid + k * NT == cn) {  // the owner of column cn publishes the pivot element and the cost-row entry
                s.bq = ur[k];
                s.bc0 = new_entry(cv[k], false, coef0, frow[cn], cn == cstar, q);
            }
        __syncthreads();
        const double qn = s.bq;
        // Lazy-flush flag (simplex.ts:380): does any row other than rnext hold a non-zero entry in column
        // cn?  The cost row and the executing pivot's row are witnesses that cost nothing; only when
        // both are zero is the whole column derived and counted.
        bool flushn = nz16(s.bc0) || (rstar != rnext && nz16(frow[cn]));
        if (!flushn) flushn = flush_flag(count_col(), qn);
        const int entering = T.vcol[cn];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = tid + k * NT;
            if (c < T.stride) T.prow[c] = c < W ? norm_entry(ur[k], c == cn, qn, flushn) : 0.0;
        }
        __syncthreads();
        if (tid == 0) {
            stage_pivot(T, rec, log_n, 1, rnext, cn, leaving, entering, qn, 0, flushn, -1, 1);
            rec->done = launch + 1; rec->p1 = pcount + 1;
            __threadfence();     // prow and the record are read by the next launch
            flip();
        }
        return;
    }
    if (rnext >= 0) {
        // ---- phase 1 goes on (wide tableau: more than eight columns per thread), same steps with reloads
        const double *rowp = src + (size_t)rnext * stride;
        const bool is_prow = rnext == rstar;
        const double coef_r = is_prow ? 0.0 : ldg_cg(rowp + cstar);
        const VI einit = {-INFINITY, INT_MAX};
        VI e = einit;
        for (int c0 = 1; c0 < W; c0 += 8 * NT) {
            double rv[8], cv[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int c = c0 + tid + k * NT;
                rv[k] = c < W ? ldg_cg(rowp + c) : 0.0;
                cv[k] = c < W ? ldg_cg(src + c) : 0.0;
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int c = c0 + tid + k * NT;
                if (c >= W) continue;
                entering_step(c, new_entry(rv[k], is_prow, coef_r, frow[c], c == cstar, q),
                              has_unres && is_unres(T, T.vcol[c]), prec, e,
                              [&] { return new_entry(cv[k], false, coef0, frow[c], c == cstar, q); });
            }
        }
        e = block_reduce_vi_rx<false>(e, einit, s.red);
        if (e.i == INT_MAX) {  // simplex.ts:73-76
            if (tid == 0) finish(ST_INFEASIBLE, 0, -1);
            return;
        }
        cn = e.i;
        cnt = count_col();
    } else {
        // ---- feasible after this pivot (simplex.ts:51-54), or already in phase 2
        if (phase_exec == 1 && only_phase == 1) {
            if (tid == 0) finish(ST_P1_DONE, 0, -1);
            return;
        }
        phase_next = 2;
        // pricing (simplex.ts:140-219) of the cost row as this pivot leaves it
        {
            const int bsz = T.use_partial ? T.batch_size : max(1, W - 1);
            PriceAcc acc;
            price_init(acc, prec);
            for (int c0 = 1; c0 < W; c0 += 8 * NT) {
                double cv[8];
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    const int c = c0 + tid + k * NT;
                    cv[k] = c < W ? ldg_cg(src + c) : 0.0;
                }
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    const int c = c0 + tid + k * NT;
                    if (c >= W) continue;
                    const double nc = new_entry(cv[k], false, coef0, frow[c], c == cstar, q);
                    int label = -1;
                    if (has_unres && nc < 0) label = T.vcol[c];
                    price_consider(T, acc, c, nc, label, bsz);
                }
            }
            price_finish_rx(T, s, acc, &cn, &isneg);
        }
        if (cn == 0) {  // optimal (simplex.ts:265-269)
            if (tid == 0) finish(ST_OPTIMAL, 2, -1);
            return;
        }
        // ratio test (simplex.ts:271-296) on the derived pivot column and right-hand side
        VI m = {INFINITY, INT_MAX};
        int dmin = INT_MAX;
        const double f_cn = frow[cn], f_0 = frow[0];
        for (int rb = 0; rb < H; rb += 8 * NT) {
            double a[8], b0[8], cf[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rb + tid + k * NT;
                a[k] = r < H ? ldg_cg(src + (size_t)r * stride + cn) : 0.0;
                b0[k] = r < H ? ldg_cg(src + (size_t)r * stride) : 0.0;
                cf[k] = (r < H && r != rstar) ? ldg_cg(src + (size_t)r * stride + cstar) : 0.0;
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int r = rb + tid + k * NT;
                if (r >= H) continue;
                const double col = new_entry(a[k], r == rstar, cf[k], f_cn, cn == cstar, q);
                T.pcol[r] = col;  // the step that executes this pivot runs in place and reads its column here
                ratio_step(r, col, new_entry(b0[k], r == rstar, cf[k], f_0, false, q), isneg, prec, dmin, m, cnt);
            }
        }
        { int okd = 1; block_reduce_ratio_rx(dmin, m, cnt, okd, s.red); }
        if (dmin != INT_MAX) rnext = dmin;
        else if (m.i != INT_MAX) rnext = m.i;
        else {  // unbounded (simplex.ts:298-303)
            if (tid == 0) finish(ST_UNBOUNDED, 2, T.vcol[cn]);
            return;
        }
    }
    // ---- stage pivot (rnext, cn): normalised row into the prow side buffer, labels, log, record
    const int leaving = T.vrow[rnext];
    const int entering = T.vcol[cn];
    __syncthreads();
    const double qn = stage_next_row(T, frow, rstar, cstar, q, rnext, cn, cnt);
    __syncthreads();
    if (tid == 0) {
        stage_pivot(T, rec, log_n, phase_next, rnext, cn, leaving, entering, qn, isneg, flush_flag(cnt, qn), -1, 1);
        rec->done = launch + 1;
        if (phase_exec == 1) rec->p1 = pcount + 1; else rec->p2 = pcount + 1;
        __threadfence();     // prow and the record are read by the next launch
        flip();
    }
}

// Selector S2 of a ping-pong step: stages the next pivot row (the row as the executing pivot leaves it, already
// normalised) into the prow side buffer, the TMA source of the next launch.
__device__ __forceinline__ void cta_selector_stage(const TabDev &T, SelSmem &s, const double *frow, int G, int rstar,
                                   int cstar, double q, int cn, int launch, bool stop_after) {
    if (cn == 0 || stop_after) return;
    int rnext, cnt;
    if (!cta_collect_partials(T, s, G, (unsigned int)(launch + 1), &rnext, &cnt)) return;  // S1 reports the error
    if (rnext < 0) return;
    // the other selector must also be done reading the prow buffer (slot G is its message)
    if (threadIdx.x == 0) part_wait(T.part + G, (unsigned int)(launch + 1));
    __syncthreads();
    stage_next_row(T, frow, rstar, cstar, q, rnext, cn, cnt);
}

// ---- the kernel ------------------------------------------------------------------------------------
// do_select: 0 = update only (two-kernel engine), 1 = the last CTA selects the next pivot,
// 2 = ping-pong: the grid carries two extra CTAs (the selectors); steps that are not eligible for the
// ping-pong path (phase 1, bootstrap, optional objectives) run in place on the first gridDim.x-2 CTAs.
// prow_arg / stride_arg duplicate TabDev.prow / stride (both immutable after jslp_tab_create) so the
// TMA copy of the pivot row can be issued before the descriptor has been fetched.
// RC < 0: the ping-pong step streams with update_rows_pp_flat<-RC> (the in-place instantiation of such a
// variant uses RC = 4).
template <int NTHREADS, int MINB, int RC, bool PF, bool PP>
__global__ void __launch_bounds__(NTHREADS, MINB)
    k_pivot_step(TabDev *Tp, Rec *rec, int do_select, const double *prow_arg, int stride_arg) {
    extern __shared__ __align__(128) double frow[];
    __shared__ TabDev T;
    __shared__ SelSmem sel;
    __shared__ uint64_t bar;
    __shared__ int s_last;
    __shared__ double s_coef[32];
    __shared__ long long s_t0;
    const int tid = threadIdx.x, NT = blockDim.x;
    // blockIdx.y = node slot (jslp_slots.cuh): every slot has its own descriptor, record and prow side buffer
    // (stride_arg doubles apart); a single-tableau launch has gridDim.y == 1.
    Tp += blockIdx.y;
    rec += blockIdx.y;
    prow_arg += (size_t)blockIdx.y * (size_t)stride_arg;
    // Programmatic dependent launch: let the next step's CTAs be scheduled while this grid drains,
    // and do not touch anything the previous step wrote before it has completed.  Both are no-ops
    // when the launch carries no programmatic dependency.
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;");
    // The head is one L2 round trip deep: the TMA copy of the pivot row needs only kernel parameters and
    // goes first; the record (one 128-byte line) and the descriptor are requested together, before the
    // first value is looked at.
    long long t0 = 0, t1 = 0, t2 = 0, t3 = 0, t4 = 0, g0 = 0;
    if (tid == 0) {
        t0 = clock64();
        s_t0 = t0;
        mbar_init(&bar, 1);
        fence_mbar_init();
        mbar_expect_tx(&bar, (uint32_t)stride_arg * 8u);
        tma_bulk_g2s(frow, prow_arg, (uint32_t)stride_arg * 8u, &bar);  // pivot row -> smem (TMA)
    }
    const int4 *rp = reinterpret_cast<const int4 *>(rec);
    // plain (L1-cached) loads: 2368 warps read this one line, L1 serves all but the first per SM
    const int4 ra = rp[0], rb = rp[1], rc = rp[2], rd = rp[3], re = rp[4];
    const double q = rec->q;
    if (tid == 0) T = *Tp;
    const int status = ra.x, phase = ra.y, has_pivot = ra.z, rstar = ra.w;
    const int cstar = rb.x, flush = rb.z, launch = rb.w;
    const int p1 = rc.x, p2 = rc.y, stop_at = rc.z, log_n0 = rc.w;
    const int only_phase = rd.y;
    const int lookahead = re.x, next_c = re.y, next_neg = re.z, prow_norm = re.w;
    if (status != ST_RUNNING || !has_pivot || (stop_at >= 0 && launch >= stop_at)) {
        if (tid == 0) mbar_wait(&bar, 0);  // do not exit with the TMA copy still in flight
        return;
    }
    const bool stop_after = stop_at >= 0 && launch + 1 >= stop_at;
    __syncthreads();
    const bool dbg = T.dbg != nullptr && launch < T.dbg_cap;
    if (dbg && tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g0));

    const int b = blockIdx.x;
    const int G = PP ? (int)gridDim.x - 2 : (int)gridDim.x;  // row CTAs (ping-pong: + 2 selector CTAs)
    const int base = T.H / G, rem = T.H % G;
    const int r0 = b * base + min(b, rem);
    const int nr = b < G ? base + (b < rem ? 1 : 0) : 0;
    const bool rows_fit = base + 1 <= NT;  // one row per thread in the look-ahead (uniform over the grid)

    if constexpr (PP) {
    // ------------------------------------------------------------------ ping-pong path
    // Grid = G row CTAs + 2 selector CTAs (decide, stage).  Eligible: phase 2 with the next entering
    // column already priced, no optional objectives, at most 32 rows per CTA (one warp runs the
    // look-ahead ratio test of the CTA's rows).
    // pp2: phase-2 pivot whose successor's entering column is priced (the steady state): row CTAs publish
    //      ratio-test partials, selector S1 decides from them, selector S2 stages the next pivot row.
    // pp1: phase-1 pivot: row CTAs publish min-RHS partials, S1 decides and stages everything.
    // pp0: phase-2 pivot without a priced successor: no partials, S1 derives the next pivot on its own.
    const bool pp2 = phase == 2 && next_c >= 0;
    const bool pp1 = phase == 1;
    {
        const bool want_partial = !stop_after && (pp1 || (pp2 && next_c > 0));
        const int lw = (NT >> 5) - 1;           // the warp that runs the look-ahead (last warp)
        const int lane = tid & 31;
        const bool la_warp = (tid >> 5) == lw && b < G;
        if (la_warp) {
            // Look-ahead ratio test of the NEXT pivot on this CTA's rows as this pivot leaves them: one
            // warp, shuffles only, published as one 16-byte message.  It needs just two entries of the
            // normalised pivot row (computed here from the raw side buffer), so it neither waits for the
            // whole-row normalisation nor delays the other warps.
            double la_col = 0.0, la_rhs = 0.0, la_coef = 0.0, raw_n = 0.0, raw_0 = 0.0;
            if (lane < nr) {  // this lane's row: pivot-column entry and the look-ahead operands
                const size_t off = (size_t)(r0 + lane) * T.stride;
                la_coef = ldg_cg(T.M + off + cstar);
                if (want_partial) {
                    if (!pp1) la_col = ldg_cg(T.M + off + next_c);
                    la_rhs = ldg_cg(T.M + off);
                }
            }
            if (want_partial) { if (!pp1) raw_n = ldg_cg(prow_arg + next_c); raw_0 = ldg_cg(prow_arg); }
            if (lane < nr) s_coef[lane] = la_coef;
            if (want_partial && pp1) {
                // phase 1: the most negative right-hand side of this CTA's rows after this pivot
                const double f_0 = prow_norm ? raw_0 : norm_entry(raw_0, false, q, flush);
                const bool is_prow = (r0 + lane) == rstar;
                const double rhs = new_entry(la_rhs, is_prow, la_coef, f_0, false, q);
                VI m = {INFINITY, INT_MAX};
                if (lane < nr && r0 + lane != 0 && rhs < -T.prec) { m.v = rhs; m.i = lane; }
                m = warp_reduce_vi<true>(m);
                if (lane == 0) {
                    mbar_wait(&bar, 0);  // a published partial also promises: this CTA is done reading prow
                    part_publish(T.part + b, m.v, m.i == INT_MAX ? 255 : m.i, 255, 0, (unsigned int)(launch + 1));
                    if (dbg) T.dbg[((size_t)launch * T.dbg_grid + b) * 8 + 2] = clock64() - s_t0;
                }
            } else if (want_partial) {
                const double f_n = prow_norm ? raw_n : norm_entry(raw_n, next_c == cstar, q, flush);
                const double f_0 = prow_norm ? raw_0 : norm_entry(raw_0, false, q, flush);
                const bool is_prow = (r0 + lane) == rstar;
                const double col = new_entry(la_col, is_prow, la_coef, f_n, next_c == cstar, q);
                const double rhs = new_entry(la_rhs, is_prow, la_coef, f_0, false, q);
                VI m = {INFINITY, INT_MAX};
                int dmin = INT_MAX, cnt = 0;
                if (lane < nr) ratio_step(r0 + lane, col, rhs, next_neg, T.prec, dmin, m, cnt);
                m = warp_reduce_vi<true>(m);
                dmin = __reduce_min_sync(0xffffffffu, dmin);
                cnt = __reduce_add_sync(0xffffffffu, cnt);
                if (lane == 0) {  // rows go out relative to r0
                    mbar_wait(&bar, 0);  // a published partial also promises: this CTA is done reading prow
                    part_publish(T.part + b, m.v, m.i == INT_MAX ? 255 : m.i - r0, dmin == INT_MAX ? 255 : dmin - r0, cnt,
                                 (unsigned int)(launch + 1));
                    if (dbg) T.dbg[((size_t)launch * T.dbg_grid + b) * 8 + 2] = clock64() - s_t0;
                }
            }
        }
        mbar_wait(&bar, 0);
        if (!prow_norm)
            for (int c = tid; c < T.stride; c += NT) frow[c] = norm_entry(frow[c], c == cstar, q, flush);
        __syncthreads();
        if (dbg && tid == 0) t1 = clock64();
        if (!pp2 && b == G) {
            cta_selector_decide_full(Tp, T, rec, sel, frow, G, rstar, cstar, q, launch, phase, phase == 1 ? p1 : p2, log_n0,
                                     stop_after, only_phase);
            if (dbg && tid == 0) t2 = t3 = clock64();
        } else if (!pp2 && b == G + 1) {
            // idle in a phase-1 step; tells the deciding selector that its TMA read of prow has landed
            if (tid == 0) part_publish(T.part + G + 1, 0.0, 255, 255, 0, (unsigned int)(launch + 1));
            if (dbg && tid == 0) t2 = t3 = clock64();
        } else if (b == G) {
            long long ts[3] = {0, 0, 0};
            // tell the staging selector that this CTA's TMA read of the prow buffer has landed
            if (tid == 0) part_publish(T.part + G, 0.0, 255, 255, 0, (unsigned int)(launch + 1));
            cta_selector_decide(Tp, T, rec, sel, frow, G, rstar, cstar, q, next_c, next_neg, launch, p2, log_n0, stop_after, ts);
            if (dbg && tid == 0) { t2 = ts[0]; t3 = ts[1]; g0 = ts[2] - t0; }  // partials in, reduced, first pricing pass
        } else if (b == G + 1) {
            cta_selector_stage(T, sel, frow, G, rstar, cstar, q, next_c, launch, stop_after);
            if (dbg && tid == 0) t2 = t3 = clock64();
        } else {
            if constexpr (RC < 0) update_rows_pp_flat<-RC>(T.M, T.M2, T.stride, frow, s_coef, r0, nr, rstar, cstar, q);
            else update_rows_pp<RC, PF>(T.M, T.M2, T.stride, frow, s_coef, r0, nr, rstar, cstar, q);
            if (dbg && tid == 0) t3 = clock64();
        }
        if (dbg && tid == 0) {
            t4 = clock64();
            unsigned int smid;
            asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
            long long *d = T.dbg + ((size_t)launch * T.dbg_grid + b) * 8;
            d[0] = g0; d[1] = t1 - t0; if (b >= G) d[2] = t2 - t0; d[3] = t3 - t0; d[4] = t4 - t0; d[5] = smid;
            d[6] = (b == G) ? 1 : (b == G + 1 ? 2 : 0); d[7] = nr;
        }
        return;
    }
    } else {
    // ------------------------------------------------------------------ in-place path
    // look-ahead operands of this thread's row, loaded while the TMA copy is in flight
    const bool fast = do_select && next_c >= 0 && !stop_after && rows_fit;
    const bool have = fast && next_c > 0 && tid < nr;
    double la_coef = 0.0, la_col = 0.0, la_rhs = 0.0;
    if (have) {
        const size_t off = (size_t)(r0 + tid) * T.stride;
        la_coef = T.pcol[r0 + tid];
        la_col = ldg_cg(T.M + off + next_c);
        la_rhs = ldg_cg(T.M + off);
    }

    mbar_wait(&bar, 0);
    if (!prow_norm)
        for (int c = tid; c < T.stride; c += NT) frow[c] = norm_entry(frow[c], c == cstar, q, flush);
    __syncthreads();
    if (dbg && tid == 0) t1 = clock64();

    update_rows<(RC < 0 ? 4 : RC), PF>(T, frow, r0, nr, rstar, cstar, q, b == G - 1);
    if (dbg && tid == 0) t2 = clock64();

    if (fast && next_c > 0) {
        __syncthreads();  // every warp is done reading this CTA's pcol entries before they are replaced
        const bool is_prow = (r0 + tid) == rstar;
        const double col = new_entry(la_col, is_prow, la_coef, frow[next_c], next_c == cstar, q);
        const double rhs = new_entry(la_rhs, is_prow, la_coef, frow[0], false, q);
        cta_ratio_partial(T, sel, r0, nr, have, col, rhs, next_neg);
    }
    __threadfence();
    __syncthreads();
    if (dbg && tid == 0) t3 = clock64();
    if (tid == 0) {
        const unsigned int t = atomicAdd(&rec->ticket, 1u);
        s_last = (t == (unsigned int)(G - 1));
    }
    __syncthreads();
    if (s_last) {
        __threadfence();
        if (tid == 0) {
            rec->ticket = 0;
            rec->done = launch + 1;
            if (phase == 1) rec->p1 = p1 + 1; else rec->p2 = p2 + 1;
            rec->has_pivot = 0;
        }
        if (do_select && !stop_after) {
            if (fast) {
                cta_tail_lookahead(T, rec, sel, G, next_c, next_neg, log_n0);
            } else {
                __syncthreads();
                cta_select(T, rec, sel);
                __syncthreads();
                if (lookahead && rec->has_pivot && rec->phase == 2 && T.nOpt == 0) cta_price_next(T, rec, sel);
            }
        }
    }
    if (dbg && tid == 0) {
        t4 = clock64();
        unsigned int smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        long long *d = T.dbg + ((size_t)launch * T.dbg_grid + b) * 8;
        d[0] = g0; d[1] = t1 - t0; d[2] = t2 - t0; d[3] = t3 - t0; d[4] = t4 - t0; d[5] = smid; d[6] = s_last; d[7] = nr;
    }
    }
}
