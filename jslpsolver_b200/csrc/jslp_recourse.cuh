// jslpsolver_b200/csrc/jslp_recourse.cuh -- the recourse LPs of a two-stage stochastic LP (included by jslp_api.cu
// after jslp_scenario.cuh).  One call is one iteration of the L-shaped method's second stage (DESIGN.md 2u): every case
// runs as a scenario of jslp_scenario_batch, and each case's certificate row -- row 0 at an optimum, the row phase 1
// stopped at when infeasible -- is reduced on the device to its multipliers of the recourse rows and, through the
// technology matrix, to the cut coefficients alpha.  Only cert_rhs and alpha leave the device beyond the scenario
// outputs: no tableau rows, no duals.
#pragma once

// alpha[s * n_first + j] = sum_i u[s * n_rows + i] * tech[(ts * n_rows + i) * n_first + j], ts = s or 0, over i in
// increasing order with unfused multiply and add: one thread per (s, j), a 32-wide tile of j by 8 cases per block, so a
// warp reads a contiguous run of one tech row and one broadcast multiplier.
__global__ void __launch_bounds__(256) k_recourse_alpha(const double *u, const double *tech, int n, int n_rows,
                                                        int n_first, int per_case, double *alpha) {
    const int j = blockIdx.x * 32 + threadIdx.x;
    if (j >= n_first) return;
    for (int s = blockIdx.y * 8 + threadIdx.y; s < n; s += gridDim.y * 8) {
        const double *us = u + (size_t)s * n_rows;
        const double *ts = tech + (per_case ? (size_t)s * n_rows * n_first : 0) + j;
        double acc = 0.0;
        for (int i = 0; i < n_rows; i++) acc = __dadd_rn(acc, __dmul_rn(us[i], ts[(size_t)i * n_first]));
        alpha[(size_t)s * n_first + j] = acc;
    }
}

// Device blocks of one jslp_recourse_batch call, freed when it returns.
struct RecourseBufs {
    double *u = nullptr, *tech = nullptr, *alpha = nullptr;
    int *pos = nullptr;
    ~RecourseBufs() { cudaFree(u); cudaFree(tech); cudaFree(alpha); cudaFree(pos); }
};

extern "C" int jslp_recourse_batch(jslp_tab *t, const jslp_scenario_edit *edits, const int32_t *offsets, int n_scenarios,
                                   const int32_t *rows, int n_rows, const double *tech, int n_first, int tech_per_case,
                                   int32_t *status, double *eval_raw, int32_t *p1, int32_t *p2, double *rhs,
                                   int32_t *vrow, double *cert_rhs, double *alpha) {
    int rc = scenario_check(t, edits, offsets, n_scenarios, status, eval_raw, p1, p2, rhs, vrow, "recourse_batch");
    if (rc) return rc;
    if (n_rows < 0 || n_first < 0 || (n_rows > 0 && !rows) || (n_rows > 0 && n_first > 0 && !tech))
        return fail(JSLP_E_INVALID, "recourse_batch: bad rows / tech arguments");
    if (n_scenarios == 0) return JSLP_OK;
    if (!cert_rhs || (n_first > 0 && !alpha)) return fail(JSLP_E_INVALID, "recourse_batch: bad output arguments");
    CK(cudaSetDevice(t->ctx->device));
    HostMaps m;
    rc = load_maps(t, m);
    if (rc) return rc;
    // every row label must name a row or a column of the tableau, once
    RecourseCert cert;
    cert.n_rows = n_rows;
    int n_labels = 0;
    for (int i = 0; i < n_rows; i++) {
        if (rows[i] < 0 || (m.row_of(rows[i]) < 0 && m.col_of(rows[i]) < 0))
            return fail(JSLP_E_INVALID, "recourse_batch: rows[" + std::to_string(i) + "] is not a label of the tableau");
        n_labels = std::max(n_labels, rows[i] + 1);
    }
    cert.pos.assign((size_t)n_labels, -1);
    for (int i = 0; i < n_rows; i++) {
        if (cert.pos[rows[i]] >= 0) return fail(JSLP_E_INVALID, "recourse_batch: a row label is listed twice");
        cert.pos[rows[i]] = i;
    }
    RecourseBufs b;
    cudaStream_t s = t->ctx->stream;
    const size_t n_tech = (size_t)(tech_per_case ? n_scenarios : 1) * n_rows * n_first;
    CK(cudaMalloc(&b.u, sizeof(double) * std::max<size_t>(1, (size_t)n_scenarios * n_rows)));
    CK(cudaMalloc(&b.pos, sizeof(int) * std::max<size_t>(1, cert.pos.size())));
    if (!cert.pos.empty())
        CK(cudaMemcpyAsync(b.pos, cert.pos.data(), sizeof(int) * cert.pos.size(), cudaMemcpyHostToDevice, s));
    cert.d_pos = b.pos;
    cert.d_u = b.u;
    rc = scenario_run(t, m, edits, offsets, n_scenarios, 1, status, eval_raw, p1, p2, rhs, vrow, &cert);
    if (rc) return rc;
    for (int i = 0; i < n_scenarios; i++) {
        const double *col = rhs + (size_t)i * t->H;
        const int cr = cert_row(t, status[i], col);
        cert_rhs[i] = cr >= 0 ? col[cr] : NAN;
    }
    if (n_first == 0) return JSLP_OK;
    CK(cudaMalloc(&b.alpha, sizeof(double) * (size_t)n_scenarios * n_first));
    if (n_tech > 0) {
        CK(cudaMalloc(&b.tech, sizeof(double) * n_tech));
        CK(cudaMemcpyAsync(b.tech, tech, sizeof(double) * n_tech, cudaMemcpyHostToDevice, s));
    }
    const dim3 grid((unsigned)((n_first + 31) / 32), (unsigned)std::min(65535, (n_scenarios + 7) / 8));
    k_recourse_alpha<<<grid, dim3(32, 8), 0, s>>>(b.u, b.tech, n_scenarios, n_rows, n_first, tech_per_case, b.alpha);
    t->ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(alpha, b.alpha, sizeof(double) * (size_t)n_scenarios * n_first, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return JSLP_OK;
}
