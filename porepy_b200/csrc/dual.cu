// dual.cu -- the mixed (dual) discretizations of Darcy flow, MVEM and RT0 (dual_cell.cuh), on a handle that keeps a
// grid's topology and the FACE x FACE mass pattern on the device, and their hybridization (dual_hybrid.cuh).
#include <climits>
#include <cstring>

#include "csr_build.cuh"
#include "dual_hybrid.cuh"

struct pb_dual {
    int nd = 0;
    int64_t nc = 0, nf = 0, nn = 0, ncf = 0, mass_nnz = -1;   // mass_nnz < 0: pattern not built yet
    Stream stream;
    DevBuf cf_ip, cf_ix, cf_sg, cf_cell, fc_ip, fc_cell, fn_ip, fn_ix, mass_ip, mass_ix;
    std::vector<int32_t> cf_ip_h;
    // values of the last pb_dual_discretize, kept for pb_dual_download and pb_dual_system
    bool have_values = false;
    int method = -1;
    DevBuf mass_val, proj_val;
    // geometry of the last pb_dual_discretize, for the hybridized solve of its saddle point
    DevBuf geo_nodes, geo_fn, geo_fc, geo_cc, geo_vol, geo_perm, geo_rot;
    // saddle-point pattern (pb_dual_system), built at its first call
    int64_t sys_nnz = -1;
    DevBuf sys_ip, sys_ix;
    // the stream's copies and kernels may still use the buffers, which go back to the pool right after
    ~pb_dual() { if (stream) cudaStreamSynchronize(stream); }
};

extern "C" void pb_dual_destroy(pb_dual *d) { delete d; }

extern "C" int pb_dual_create(int nd, int64_t nc, int64_t nf, int64_t nn, const int32_t *cf_indptr,
                              const int32_t *cf_indices, const int8_t *cf_data, const int32_t *fn_indptr,
                              const int32_t *fn_indices, pb_dual **out) {
    if (!out || !cf_indptr || !cf_indices || !cf_data || !fn_indptr || !fn_indices)
        return pb_fail_(PB_EINVAL, "null pointer");
    if (nd < 1 || nd > 3) return pb_fail_(PB_EINVAL, "MVEM / RT0 discretize grids of dimension 1, 2 or 3");
    if (nc <= 0 || nf <= 0 || nn <= 0 || nc >= INT_MAX || nf >= INT_MAX) return pb_fail_(PB_EINVAL, "grid size");
    if (int rc = pb_require_device()) return rc;
    const int64_t ncf = cf_indptr[nc];
    std::vector<int32_t> cf_cell((size_t)ncf), fc_ip((size_t)nf + 1, 0), fc_cell((size_t)ncf);
    for (int64_t c = 0; c < nc; ++c)
        for (int32_t q = cf_indptr[c]; q < cf_indptr[c + 1]; ++q) {
            const int32_t f = cf_indices[q];
            if (f < 0 || f >= nf) return pb_fail_(PB_EINVAL, "cell_faces index out of range");
            if (q > cf_indptr[c] && f <= cf_indices[q - 1])
                return pb_fail_(PB_EINVAL, "cell_faces: the faces of a cell must be sorted and distinct");
            if (cf_data[q] != 1 && cf_data[q] != -1) return pb_fail_(PB_EINVAL, "cell_faces data must be +-1");
            cf_cell[q] = (int32_t)c;
            ++fc_ip[f + 1];
        }
    for (int64_t f = 0; f < nf; ++f) {
        fc_ip[f + 1] += fc_ip[f];
        for (int32_t r = fn_indptr[f]; r < fn_indptr[f + 1]; ++r)
            if (fn_indices[r] < 0 || fn_indices[r] >= nn) return pb_fail_(PB_EINVAL, "face_nodes index out of range");
    }
    {
        std::vector<int32_t> next(fc_ip.begin(), fc_ip.end() - 1);
        for (int64_t q = 0; q < ncf; ++q) fc_cell[next[cf_indices[q]]++] = cf_cell[q];
    }
    std::unique_ptr<pb_dual> d(new pb_dual);
    d->nd = nd; d->nc = nc; d->nf = nf; d->nn = nn; d->ncf = ncf;
    d->cf_ip_h.assign(cf_indptr, cf_indptr + nc + 1);
    CUDA_TRY(d->stream.create());
    cudaStream_t st = d->stream;
    CUDA_TRY(d->cf_ip.upload(cf_indptr, (size_t)nc + 1, st));
    CUDA_TRY(d->cf_ix.upload(cf_indices, (size_t)ncf, st));
    CUDA_TRY(d->cf_sg.upload(cf_data, (size_t)ncf, st));
    CUDA_TRY(d->cf_cell.upload(cf_cell, st));
    CUDA_TRY(d->fc_ip.upload(fc_ip, st));
    CUDA_TRY(d->fc_cell.upload(fc_cell, st));
    CUDA_TRY(d->fn_ip.upload(fn_indptr, (size_t)nf + 1, st));
    CUDA_TRY(d->fn_ix.upload(fn_indices, (size_t)fn_indptr[nf], st));
    CUDA_TRY(cudaStreamSynchronize(st));
    *out = d.release();
    return PB_OK;
}

// Row f of the mass pattern: the sorted union of the faces of f's cells (pattern_kernel, counted, scanned, filled).
static int dual_build_pattern(pb_dual *d) {
    cudaStream_t st = d->stream;
    const int64_t nf = d->nf;
    DevBuf counts, flag;
    CUDA_TRY(counts.ensure((size_t)nf * sizeof(int32_t)));
    CUDA_TRY(flag.ensure(sizeof(int)));
    CUDA_TRY(cudaMemsetAsync(flag.p, 0, sizeof(int), st));
    CUDA_TRY(d->mass_ip.ensure((size_t)(nf + 1) * sizeof(int32_t)));
    const int grid = grid_stride_blocks(nf, 8, 8);
    pattern_kernel<256><<<grid, 256, 0, st>>>(nf, d->fc_ip.as<int32_t>(), d->fc_cell.as<int32_t>(),
                                              d->cf_ip.as<int32_t>(), d->cf_ix.as<int32_t>(), counts.as<int32_t>(),
                                              nullptr, nullptr, 0, flag.as<int>());
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    int over = 0;
    CUDA_TRY(cudaMemcpyAsync(&over, flag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    int64_t total = 0;
    const int rc = pb_scan_offsets_(counts.as<int32_t>(), d->mass_ip.as<int32_t>(), nf, st, &total);
    if (rc) return rc;
    if (over) return pb_fail_(PB_ENOTIMPL, "MVEM / RT0 mass pattern: the cells of a face have more than 256 faces");
    if (total >= 0x7FFFFFFFll) return pb_fail_(PB_ENOTIMPL, "MVEM / RT0 mass pattern exceeds 2^31 entries");
    CUDA_TRY(d->mass_ix.ensure((size_t)std::max<int64_t>(1, total) * sizeof(int32_t)));
    pattern_kernel<256><<<grid, 256, 0, st>>>(nf, d->fc_ip.as<int32_t>(), d->fc_cell.as<int32_t>(),
                                              d->cf_ip.as<int32_t>(), d->cf_ix.as<int32_t>(), nullptr,
                                              d->mass_ip.as<int32_t>(), d->mass_ix.as<int32_t>(), 1, flag.as<int>());
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(st));
    d->mass_nnz = total;
    return PB_OK;
}

extern "C" int pb_dual_mass_pattern(pb_dual *d, int64_t *nnz, int32_t *indptr, int32_t *indices) {
    if (!d || !nnz) return pb_fail_(PB_EINVAL, "null pointer");
    if (d->mass_nnz < 0) {
        const int rc = dual_build_pattern(d);
        if (rc) return rc;
    }
    *nnz = d->mass_nnz;
    cudaStream_t st = d->stream;
    if (indptr) CUDA_TRY(cudaMemcpyAsync(indptr, d->mass_ip.p, (size_t)(d->nf + 1) * sizeof(int32_t),
                                        cudaMemcpyDeviceToHost, st));
    if (indices) CUDA_TRY(cudaMemcpyAsync(indices, d->mass_ix.p, (size_t)d->mass_nnz * sizeof(int32_t),
                                         cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return PB_OK;
}

static pb::DualTopo dual_topo(pb_dual *d) {
    return pb::DualTopo{d->cf_ip.as<int32_t>(), d->cf_ix.as<int32_t>(), d->cf_cell.as<int32_t>(),
                        d->cf_sg.as<int8_t>(), d->fn_ip.as<int32_t>(), d->fn_ix.as<int32_t>(),
                        d->mass_ip.as<int32_t>(), d->mass_ix.as<int32_t>()};
}

template <int ND, int METHOD>
__global__ void dual_kernel(int64_t ncf, pb::DualTopo T, pb::DualGeo G, double *__restrict__ mass,
                            double *__restrict__ proj, int32_t *bad) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < ncf; q += (int64_t)gridDim.x * blockDim.x)
        pb::dual_row<ND>(METHOD, q, T, G, mass, proj, bad);
}

extern "C" int pb_dual_discretize(pb_dual *d, int method, const double *nodes, const double *face_normals,
                                  const double *face_centers, const double *cell_centers, const double *cell_volumes,
                                  const double *perm, const double *rot, double *mass, double *proj, int64_t *bad_cell,
                                  float *kernel_ms) {
    if (!d || !nodes || !face_normals || !face_centers || !cell_centers || !cell_volumes || !perm || !rot || !bad_cell)
        return pb_fail_(PB_EINVAL, "null pointer");
    if (method != PB_DUAL_MVEM && method != PB_DUAL_RT0) return pb_fail_(PB_EINVAL, "unknown dual method");
    const int nd = d->nd;
    const int64_t nc = d->nc, nf = d->nf, nn = d->nn, ncf = d->ncf;
    if (method == PB_DUAL_RT0)
        for (int64_t c = 0; c < nc; ++c)
            if (d->cf_ip_h[c + 1] - d->cf_ip_h[c] != nd + 1)
                return pb_fail_(PB_EINVAL, "RT0 needs simplices: cell " + std::to_string(c) + " has " +
                                                  std::to_string(d->cf_ip_h[c + 1] - d->cf_ip_h[c]) + " faces");
    if (d->mass_nnz < 0) {
        const int rc = dual_build_pattern(d);
        if (rc) return rc;
    }
    cudaStream_t st = d->stream;
    DevBuf &dn = d->geo_nodes, &dfn = d->geo_fn, &dfc = d->geo_fc, &dcc = d->geo_cc, &dvol = d->geo_vol,
           &dperm = d->geo_perm, &drot = d->geo_rot;
    DevBuf dbad;
    DevBuf &dmass = d->mass_val, &dproj = d->proj_val;
    d->have_values = false;
    CUDA_TRY(dn.upload(nodes, (size_t)3 * nn, st));
    CUDA_TRY(dfn.upload(face_normals, (size_t)3 * nf, st));
    CUDA_TRY(dfc.upload(face_centers, (size_t)3 * nf, st));
    CUDA_TRY(dcc.upload(cell_centers, (size_t)3 * nc, st));
    CUDA_TRY(dvol.upload(cell_volumes, (size_t)nc, st));
    CUDA_TRY(dperm.upload(perm, (size_t)9 * nc, st));
    CUDA_TRY(drot.upload(rot, (size_t)9, st));
    CUDA_TRY(dmass.ensure((size_t)std::max<int64_t>(1, d->mass_nnz) * sizeof(double)));
    CUDA_TRY(dproj.ensure((size_t)3 * ncf * sizeof(double)));
    CUDA_TRY(dbad.ensure(sizeof(int32_t)));
    CUDA_TRY(cudaMemsetAsync(dmass.p, 0, (size_t)d->mass_nnz * sizeof(double), st));
    const int32_t none = INT_MAX;
    CUDA_TRY(cudaMemcpyAsync(dbad.p, &none, sizeof(int32_t), cudaMemcpyHostToDevice, st));
    const pb::DualTopo T = dual_topo(d);
    const pb::DualGeo G{nn, nf, nc, dn.as<double>(), dfn.as<double>(), dfc.as<double>(), dcc.as<double>(),
                        dvol.as<double>(), dperm.as<double>(), drot.as<double>()};
    KernelTimer timer;
    CUDA_TRY(timer.create());
    CUDA_TRY(timer.mark(0, st));
    dispatch_nd<1, 2, 3>(nd, [&](auto ND) {
        auto kernel = method == PB_DUAL_MVEM ? dual_kernel<ND, pb::kDualMvem> : dual_kernel<ND, pb::kDualRt0>;
        kernel<<<grid_stride_blocks(ncf, 256, 16), 256, 0, st>>>(ncf, T, G, dmass.as<double>(), dproj.as<double>(),
                                                                 dbad.as<int32_t>());
    });
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(timer.mark(1, st));
    int32_t hbad = none;
    if (mass) CUDA_TRY(cudaMemcpyAsync(mass, dmass.p, (size_t)d->mass_nnz * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (proj) CUDA_TRY(cudaMemcpyAsync(proj, dproj.p, (size_t)3 * ncf * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&hbad, dbad.p, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    float ms = 0.0f;
    CUDA_TRY(timer.ms(&ms));
    if (kernel_ms) *kernel_ms = ms;
    *bad_cell = hbad == none ? -1 : (int64_t)hbad;
    d->have_values = hbad == none;
    d->method = method;
    return PB_OK;
}

extern "C" int pb_dual_download(pb_dual *d, double *mass, double *proj) {
    if (!d) return pb_fail_(PB_EINVAL, "null pointer");
    if (!d->have_values) return pb_fail_(PB_EINVAL, "pb_dual_download: no discretization on the handle");
    cudaStream_t st = d->stream;
    if (mass) CUDA_TRY(cudaMemcpyAsync(mass, d->mass_val.p, (size_t)d->mass_nnz * sizeof(double),
                                      cudaMemcpyDeviceToHost, st));
    if (proj) CUDA_TRY(cudaMemcpyAsync(proj, d->proj_val.p, (size_t)3 * d->ncf * sizeof(double),
                                      cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return PB_OK;
}

// ---- saddle-point system [[mass, div^T], [div, 0]], div = -cell_faces^T (dual_elliptic.py assemble_matrix_rhs) ----
// Row f < nf: the mass row of f, then column nf + c for every cell c of f (ascending).  Row nf + c: the faces of c.
__global__ void dual_sys_count_kernel(int64_t nf, int64_t nc, const int32_t *__restrict__ mass_ip,
                                      const int32_t *__restrict__ fc_ip, const int32_t *__restrict__ cf_ip,
                                      int32_t *__restrict__ count) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nf + nc; r += (int64_t)gridDim.x * blockDim.x)
        count[r] = r < nf ? mass_ip[r + 1] - mass_ip[r] + fc_ip[r + 1] - fc_ip[r]
                          : cf_ip[r - nf + 1] - cf_ip[r - nf];
}

__global__ void dual_sys_pattern_kernel(int64_t nf, int64_t nc, const int32_t *__restrict__ mass_ip,
                                        const int32_t *__restrict__ mass_ix, const int32_t *__restrict__ fc_ip,
                                        const int32_t *__restrict__ fc_cell, const int32_t *__restrict__ cf_ip,
                                        const int32_t *__restrict__ cf_ix, const int32_t *__restrict__ ip,
                                        int32_t *__restrict__ ix) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nf + nc; r += (int64_t)gridDim.x * blockDim.x) {
        int32_t o = ip[r];
        if (r < nf) {
            for (int32_t q = mass_ip[r]; q < mass_ip[r + 1]; ++q) ix[o++] = mass_ix[q];
            for (int32_t q = fc_ip[r]; q < fc_ip[r + 1]; ++q) ix[o++] = (int32_t)nf + fc_cell[q];
        } else {
            for (int32_t q = cf_ip[r - nf]; q < cf_ip[r - nf + 1]; ++q) ix[o++] = cf_ix[q];
        }
    }
}

// |mass|_inf: the largest absolute row sum, as the bits of a non-negative double (ordered like the values)
__global__ void dual_norm_kernel(int64_t nf, const int32_t *__restrict__ mass_ip, const double *__restrict__ mass,
                                 unsigned long long *norm_bits) {
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < nf; f += (int64_t)gridDim.x * blockDim.x) {
        double s = 0.0;
        for (int32_t q = mass_ip[f]; q < mass_ip[f + 1]; ++q) s += fabs(mass[q]);
        atomicMax(norm_bits, (unsigned long long)__double_as_longlong(s));
    }
}

// cf_ix position of face f among the faces of cell c
__device__ __forceinline__ int32_t dual_cf_pos(const int32_t *cf_ip, const int32_t *cf_ix, int32_t c, int32_t f) {
    int32_t lo = cf_ip[c], hi = cf_ip[c + 1];
    while (lo < hi) {
        const int32_t mid = (lo + hi) >> 1;
        if (cf_ix[mid] < f) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// Values and right-hand side row by row (assemble_neumann_robin, assemble_rhs): Neumann rows (not internal) are
// cleared with |mass|_inf on the diagonal, Robin rows get 1 / (robin_weight area) added to it; the face sign is that of
// the face's first cell.  codes: PB_BC_* per face, interior and internal faces PB_BC_INTERIOR.
__global__ void dual_sys_values_kernel(int64_t nf, int64_t nc, const int32_t *__restrict__ mass_ip,
                                       const int32_t *__restrict__ mass_ix, const double *__restrict__ mass,
                                       const int32_t *__restrict__ fc_ip, const int32_t *__restrict__ fc_cell,
                                       const int32_t *__restrict__ cf_ip, const int32_t *__restrict__ cf_ix,
                                       const int8_t *__restrict__ cf_sg, const double *__restrict__ proj,
                                       const uint8_t *__restrict__ codes, const double *__restrict__ robin_weight,
                                       const double *__restrict__ face_areas, const double *__restrict__ bc_values,
                                       const double *__restrict__ vsrc, const unsigned long long *__restrict__ norm_bits,
                                       const int32_t *__restrict__ ip, double *__restrict__ a, double *__restrict__ rhs) {
    const double norm = __longlong_as_double((long long)*norm_bits);
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nf + nc; r += (int64_t)gridDim.x * blockDim.x) {
        int32_t o = ip[r];
        if (r >= nf) {
            const int32_t c = (int32_t)(r - nf);
            for (int32_t q = cf_ip[c]; q < cf_ip[c + 1]; ++q) a[o++] = -(double)cf_sg[q];
            rhs[r] = 0.0;
            continue;
        }
        const int32_t f = (int32_t)r;
        const uint8_t code = codes[f];
        const double rob = code == PB_BC_ROB ? 1.0 / (robin_weight[f] * face_areas[f]) : 0.0;
        for (int32_t q = mass_ip[f]; q < mass_ip[f + 1]; ++q) {
            const bool diag = mass_ix[q] == f;
            a[o++] = code == PB_BC_NEU ? (diag ? norm : 0.0) : (diag ? mass[q] + rob : mass[q]);
        }
        double b = 0.0, sign = 0.0;
        for (int32_t q = fc_ip[f]; q < fc_ip[f + 1]; ++q) {
            const int32_t c = fc_cell[q];
            const int32_t p = dual_cf_pos(cf_ip, cf_ix, c, f);
            if (q == fc_ip[f]) sign = (double)cf_sg[p];
            a[o++] = code == PB_BC_NEU ? 0.0 : -(double)cf_sg[p];
            if (vsrc) {
                const int32_t n = cf_ip[c + 1] - cf_ip[c], i = p - cf_ip[c];
                for (int k = 0; k < 3; ++k)
                    b += proj[3 * (int64_t)cf_ip[c] + k * n + i] * vsrc[3 * (int64_t)c + k];
            }
        }
        if (code == PB_BC_DIR) b += -sign * bc_values[f];
        if (code == PB_BC_ROB) b += -sign * bc_values[f] / robin_weight[f];
        if (code == PB_BC_NEU) b = sign * norm * bc_values[f];
        rhs[f] = b;
    }
}

extern "C" int pb_dual_system(pb_dual *d, const uint8_t *codes, const double *robin_weight, const double *face_areas,
                              const double *bc_values, const double *vector_source, pb_csr **out, double *rhs,
                              double *norm) {
    if (!d || !codes || !robin_weight || !face_areas || !bc_values || !out || !rhs || !norm)
        return pb_fail_(PB_EINVAL, "null pointer");
    if (!d->have_values) return pb_fail_(PB_EINVAL, "pb_dual_system: no discretization on the handle");
    const int64_t nf = d->nf, nc = d->nc;
    for (int64_t f = 0; f < nf; ++f)
        if (codes[f] > PB_BC_ROB) return pb_fail_(PB_EINVAL, "boundary code out of range");
    cudaStream_t st = d->stream;
    const int grid = grid_stride_blocks(nf + nc, 256, 16);
    if (d->sys_nnz < 0) {
        DevBuf count;
        CUDA_TRY(count.ensure((size_t)(nf + nc) * sizeof(int32_t)));
        CUDA_TRY(d->sys_ip.ensure((size_t)(nf + nc + 1) * sizeof(int32_t)));
        dual_sys_count_kernel<<<grid, 256, 0, st>>>(nf, nc, d->mass_ip.as<int32_t>(), d->fc_ip.as<int32_t>(),
                                                    d->cf_ip.as<int32_t>(), count.as<int32_t>());
        pb_count_launch_();
        CUDA_TRY(cudaGetLastError());
        int64_t total = 0;
        const int rc = pb_scan_offsets_(count.as<int32_t>(), d->sys_ip.as<int32_t>(), nf + nc, st, &total);
        if (rc) return rc;
        if (total >= 0x7FFFFFFFll) return pb_fail_(PB_ENOTIMPL, "MVEM / RT0 system exceeds 2^31 entries");
        CUDA_TRY(d->sys_ix.ensure((size_t)std::max<int64_t>(1, total) * sizeof(int32_t)));
        dual_sys_pattern_kernel<<<grid, 256, 0, st>>>(nf, nc, d->mass_ip.as<int32_t>(), d->mass_ix.as<int32_t>(),
                                                      d->fc_ip.as<int32_t>(), d->fc_cell.as<int32_t>(),
                                                      d->cf_ip.as<int32_t>(), d->cf_ix.as<int32_t>(),
                                                      d->sys_ip.as<int32_t>(), d->sys_ix.as<int32_t>());
        pb_count_launch_();
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaStreamSynchronize(st));
        d->sys_nnz = total;
    }
    CsrPtr a;
    int rc = pb_csr_from_device_pattern_(nf + nc, nf + nc, d->sys_nnz, d->sys_ip.as<int32_t>(), d->sys_ix.as<int32_t>(),
                                         a);
    if (rc) return rc;
    DevBuf dcodes, drw, darea, dbc, dvs, dnorm, drhs;
    CUDA_TRY(dcodes.upload(codes, (size_t)nf, st));
    CUDA_TRY(drw.upload(robin_weight, (size_t)nf, st));
    CUDA_TRY(darea.upload(face_areas, (size_t)nf, st));
    CUDA_TRY(dbc.upload(bc_values, (size_t)nf, st));
    if (vector_source) CUDA_TRY(dvs.upload(vector_source, (size_t)3 * nc, st));
    CUDA_TRY(dnorm.ensure(sizeof(unsigned long long)));
    CUDA_TRY(drhs.ensure((size_t)(nf + nc) * sizeof(double)));
    CUDA_TRY(cudaMemsetAsync(dnorm.p, 0, sizeof(unsigned long long), st));
    dual_norm_kernel<<<grid, 256, 0, st>>>(nf, d->mass_ip.as<int32_t>(), d->mass_val.as<double>(),
                                           dnorm.as<unsigned long long>());
    dual_sys_values_kernel<<<grid, 256, 0, st>>>(
        nf, nc, d->mass_ip.as<int32_t>(), d->mass_ix.as<int32_t>(), d->mass_val.as<double>(), d->fc_ip.as<int32_t>(),
        d->fc_cell.as<int32_t>(), d->cf_ip.as<int32_t>(), d->cf_ix.as<int32_t>(), d->cf_sg.as<int8_t>(),
        d->proj_val.as<double>(), dcodes.as<uint8_t>(), drw.as<double>(), darea.as<double>(), dbc.as<double>(),
        vector_source ? dvs.as<double>() : nullptr, dnorm.as<unsigned long long>(), d->sys_ip.as<int32_t>(),
        pb_csr_view_(a.get()).data, drhs.as<double>());
    pb_count_launch_(); pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    unsigned long long nb = 0;
    CUDA_TRY(cudaMemcpyAsync(rhs, drhs.p, (size_t)(nf + nc) * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&nb, dnorm.p, sizeof(nb), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    std::memcpy(norm, &nb, sizeof(double));
    *out = a.release();
    return PB_OK;
}

// ---- hybridization (dual_hybrid.cuh): one warp per cell, lane i on local face i ----
constexpr int kHybridWarps = 4;

// The cell's local matrix, inverted in place by the Gauss-Jordan steps of group_inv_kernel (gmres.cu), then z, r and
// lambda.  Returns false when a pivot is zero or not finite (every lane agrees).
template <int ND, int METHOD>
__device__ bool hybrid_cell(int64_t c, int lane, const pb::DualTopo &T, const pb::DualGeo &G, const pb::HybridIn &H,
                            const double *lam, double *A, double *E, double *z, double *r, double *lv, int32_t *bad) {
    const int n = T.cf_ip[c + 1] - T.cf_ip[c];
    if (lane < n) {
        pb::hybrid_local_row<ND>(METHOD, c, lane, T, G, H, A, bad);
        pb::group_identity_row(E, n, lane);
    }
    __syncwarp();
    for (int k = 0; k < n; ++k) {
        const int p = pb::group_pivot(A, n, k);   // every lane finds the same pivot
        if (p < 0) return false;
        __syncwarp();
        if (lane < n) pb::group_swap_col(A, E, n, k, p, lane);
        __syncwarp();
        if (lane < n && lane != k) pb::group_eliminate_row(A, E, n, k, lane);
        __syncwarp();
        if (lane == k) pb::group_scale_row(A, E, n, k);
        __syncwarp();
    }
    if (lane < n) pb::hybrid_vectors(c, lane, T, H, E, lam, z, r, lv);
    __syncwarp();
    return true;
}

// lam == NULL: condensation into hval / rhs; else recovery of u / p.  singular: smallest cell with a singular A.
template <int ND, int METHOD>
__global__ void hybrid_cell_kernel(int64_t nc, pb::DualTopo T, pb::DualGeo G, pb::HybridIn H, int nmax,
                                   const double *__restrict__ lam, double *__restrict__ hval, double *__restrict__ rhs,
                                   double *__restrict__ u, double *__restrict__ p, int32_t *bad, int32_t *singular) {
    extern __shared__ double sm[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    double *A = sm + (size_t)wid * pb::hybrid_cell_doubles(nmax);
    double *E = A + nmax * nmax, *z = E + nmax * nmax, *r = z + nmax, *lv = r + nmax;
    for (int64_t c = (int64_t)blockIdx.x * kHybridWarps + wid; c < nc; c += (int64_t)gridDim.x * kHybridWarps) {
        const int n = T.cf_ip[c + 1] - T.cf_ip[c];
        if (!hybrid_cell<ND, METHOD>(c, lane, T, G, H, lam, A, E, z, r, lv, bad)) {
            if (lane == 0) atomicMin(singular, (int32_t)c);
        } else if (lane < n) {
            if (lam) pb::hybrid_recover_row(c, lane, T, H, E, z, r, lv, u, p);
            else pb::hybrid_condense_row(c, lane, T, H, E, z, r, hval, rhs);
        }
        __syncwarp();
    }
}

__global__ void hybrid_bc_kernel(int64_t nf, pb::DualTopo T, pb::HybridIn H, const double *__restrict__ robin_weight,
                                 const double *__restrict__ face_areas, const unsigned long long *__restrict__ norm_bits,
                                 double *__restrict__ hval, double *__restrict__ rhs) {
    const double norm = __longlong_as_double((long long)*norm_bits);
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < nf; f += (int64_t)gridDim.x * blockDim.x)
        pb::hybrid_bc_row((int32_t)f, T, H, robin_weight, face_areas, norm, hval, rhs);
}

// Everything both entry points share: the checks, the geometry (uploaded, or that of the last pb_dual_discretize), the
// values and codes, and one timed launch of hybrid_cell_kernel.
struct HybridRun {
    DevBuf geo[7], aper, vals, codes, lam, flags;
    pb::DualGeo G{};
    pb::HybridIn H{};
    int method = 0, nmax = 0;
};

static int hybrid_prepare(pb_dual *d, int mode, const double *const geo[7], const double *aperture,
                          const uint8_t *codes, const double *values, HybridRun &R) {
    if (mode != PB_DUAL_HYBRID_VEM && mode != PB_DUAL_HYBRID_SADDLE) return pb_fail_(PB_EINVAL, "unknown hybrid mode");
    const int64_t nc = d->nc, nf = d->nf, nn = d->nn;
    for (int64_t c = 0; c < nc; ++c)
        R.nmax = std::max<int>(R.nmax, d->cf_ip_h[c + 1] - d->cf_ip_h[c]);
    if (R.nmax > pb::kHybridMaxFaces)
        return pb_fail_(PB_ENOTIMPL, "hybridization: a cell has " + std::to_string(R.nmax) +
                                         " faces; one warp condenses one cell of at most 32 faces");
    for (int64_t f = 0; f < nf; ++f)
        if (codes[f] > PB_BC_ROB) return pb_fail_(PB_EINVAL, "boundary code out of range");
    if (d->mass_nnz < 0) {
        const int rc = dual_build_pattern(d);
        if (rc) return rc;
    }
    cudaStream_t st = d->stream;
    const double *const *g = geo;
    const DevBuf *src[7];
    if (mode == PB_DUAL_HYBRID_VEM) {
        for (int k = 0; k < 7; ++k)
            if (!geo[k]) return pb_fail_(PB_EINVAL, "null pointer");
        if (!aperture) return pb_fail_(PB_EINVAL, "null pointer");
        const size_t sizes[7] = {(size_t)3 * nn, (size_t)3 * nf, (size_t)3 * nf, (size_t)3 * nc, (size_t)nc,
                                 (size_t)9 * nc, 9};
        for (int k = 0; k < 7; ++k) {
            CUDA_TRY(R.geo[k].upload(g[k], sizes[k], st));
            src[k] = &R.geo[k];
        }
        CUDA_TRY(R.aper.upload(aperture, (size_t)nc, st));
        R.method = PB_DUAL_MVEM;
    } else {
        if (!d->have_values)
            return pb_fail_(PB_EINVAL, "hybridization of the saddle point: no discretization on the handle");
        const DevBuf *kept[7] = {&d->geo_nodes, &d->geo_fn, &d->geo_fc, &d->geo_cc, &d->geo_vol, &d->geo_perm,
                                 &d->geo_rot};
        for (int k = 0; k < 7; ++k) src[k] = kept[k];
        R.method = d->method;
    }
    CUDA_TRY(R.vals.upload(values, (size_t)(nf + nc), st));
    CUDA_TRY(R.codes.upload(codes, (size_t)nf, st));
    R.G = pb::DualGeo{nn, nf, nc, src[0]->as<double>(), src[1]->as<double>(), src[2]->as<double>(),
                      src[3]->as<double>(), src[4]->as<double>(), src[5]->as<double>(), src[6]->as<double>()};
    R.H = pb::HybridIn{mode, nf, d->fc_ip.as<int32_t>(), d->fc_cell.as<int32_t>(),
                       mode == PB_DUAL_HYBRID_VEM ? R.aper.as<double>() : nullptr, R.vals.as<double>(),
                       R.codes.as<uint8_t>()};
    CUDA_TRY(R.flags.ensure(2 * sizeof(int32_t)));
    CUDA_TRY(cudaMemsetAsync(R.flags.p, 0x7f, 2 * sizeof(int32_t), st));
    return PB_OK;
}

// One timed launch of hybrid_cell_kernel; then the two flags: MVEM consistency (AssertionError in Python) and a
// singular local matrix.
static int hybrid_run(pb_dual *d, HybridRun &R, const double *lam, double *hval, double *rhs, double *u, double *p,
                      int64_t *bad_cell, float *kernel_ms) {
    cudaStream_t st = d->stream;
    const pb::DualTopo T = dual_topo(d);
    const size_t smem = (size_t)kHybridWarps * pb::hybrid_cell_doubles(R.nmax) * sizeof(double);
    int32_t *flags = R.flags.as<int32_t>();
    KernelTimer timer;
    CUDA_TRY(timer.create());
    CUDA_TRY(timer.mark(0, st));
    const int rc = dispatch_nd<1, 2, 3>(d->nd, [&](auto ND) {
        auto kernel = R.method == PB_DUAL_MVEM ? hybrid_cell_kernel<ND, pb::kDualMvem>
                                               : hybrid_cell_kernel<ND, pb::kDualRt0>;
        CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kernel<<<grid_stride_blocks(d->nc, kHybridWarps, 32), 32 * kHybridWarps, smem, st>>>(
            d->nc, T, R.G, R.H, R.nmax, lam, hval, rhs, u, p, flags, flags + 1);
        return PB_OK;
    });
    if (rc) return rc;
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(timer.mark(1, st));
    int32_t hf[2];
    CUDA_TRY(cudaMemcpyAsync(hf, flags, sizeof(hf), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    float ms = 0.0f;
    CUDA_TRY(timer.ms(&ms));
    if (kernel_ms) *kernel_ms = ms;
    if (hf[1] != 0x7f7f7f7f)
        return pb_fail_(PB_ESINGULAR, "hybridization: the local matrix of cell " + std::to_string(hf[1]) +
                                          " is singular");
    if (bad_cell) *bad_cell = hf[0] == 0x7f7f7f7f ? -1 : (int64_t)hf[0];
    return PB_OK;
}

extern "C" int pb_dual_hybrid_system(pb_dual *d, int mode, const double *nodes, const double *face_normals,
                                     const double *face_centers, const double *cell_centers,
                                     const double *cell_volumes, const double *perm, const double *rot,
                                     const double *aperture, const uint8_t *codes, const double *robin_weight,
                                     const double *face_areas, const double *values, pb_csr **out, double *rhs,
                                     int64_t *bad_cell, float *kernel_ms) {
    if (!d || !codes || !robin_weight || !face_areas || !values || !out || !rhs || !bad_cell)
        return pb_fail_(PB_EINVAL, "null pointer");
    const double *const geo[7] = {nodes, face_normals, face_centers, cell_centers, cell_volumes, perm, rot};
    HybridRun R;
    int rc = hybrid_prepare(d, mode, geo, aperture, codes, values, R);
    if (rc) return rc;
    const int64_t nf = d->nf;
    cudaStream_t st = d->stream;
    CsrPtr a;
    rc = pb_csr_from_device_pattern_(nf, nf, d->mass_nnz, d->mass_ip.as<int32_t>(), d->mass_ix.as<int32_t>(), a);
    if (rc) return rc;
    double *hval = pb_csr_view_(a.get()).data;
    DevBuf drhs, drw, darea, dnorm;
    CUDA_TRY(drhs.ensure((size_t)nf * sizeof(double)));
    CUDA_TRY(drw.upload(robin_weight, (size_t)nf, st));
    CUDA_TRY(darea.upload(face_areas, (size_t)nf, st));
    CUDA_TRY(dnorm.ensure(sizeof(unsigned long long)));
    CUDA_TRY(cudaMemsetAsync(hval, 0, (size_t)d->mass_nnz * sizeof(double), st));
    CUDA_TRY(cudaMemsetAsync(drhs.p, 0, (size_t)nf * sizeof(double), st));
    CUDA_TRY(cudaMemsetAsync(dnorm.p, 0, sizeof(unsigned long long), st));
    rc = hybrid_run(d, R, nullptr, hval, drhs.as<double>(), nullptr, nullptr, bad_cell, kernel_ms);
    if (rc) return rc;
    // |H|_inf before the boundary conditions (hybrid.py), or |mass|_inf of the saddle-point system
    const int grid = grid_stride_blocks(nf, 256, 16);
    dual_norm_kernel<<<grid, 256, 0, st>>>(nf, d->mass_ip.as<int32_t>(),
                                           mode == PB_DUAL_HYBRID_VEM ? hval : d->mass_val.as<double>(),
                                           dnorm.as<unsigned long long>());
    hybrid_bc_kernel<<<grid, 256, 0, st>>>(nf, dual_topo(d), R.H, drw.as<double>(), darea.as<double>(),
                                           dnorm.as<unsigned long long>(), hval, drhs.as<double>());
    pb_count_launch_(); pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(rhs, drhs.p, (size_t)nf * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    *out = a.release();
    return PB_OK;
}

extern "C" int pb_dual_hybrid_recover(pb_dual *d, int mode, const double *nodes, const double *face_normals,
                                      const double *face_centers, const double *cell_centers,
                                      const double *cell_volumes, const double *perm, const double *rot,
                                      const double *aperture, const uint8_t *codes, const double *values,
                                      const double *lambda, double *up, float *kernel_ms) {
    if (!d || !codes || !values || !lambda || !up) return pb_fail_(PB_EINVAL, "null pointer");
    const double *const geo[7] = {nodes, face_normals, face_centers, cell_centers, cell_volumes, perm, rot};
    HybridRun R;
    int rc = hybrid_prepare(d, mode, geo, aperture, codes, values, R);
    if (rc) return rc;
    const int64_t nf = d->nf, nc = d->nc;
    cudaStream_t st = d->stream;
    DevBuf dup;
    CUDA_TRY(R.lam.upload(lambda, (size_t)nf, st));
    CUDA_TRY(dup.ensure((size_t)(nf + nc) * sizeof(double)));
    CUDA_TRY(cudaMemsetAsync(dup.p, 0, (size_t)(nf + nc) * sizeof(double), st));
    double *u = dup.as<double>();
    rc = hybrid_run(d, R, R.lam.as<double>(), nullptr, nullptr, u, u + nf, nullptr, kernel_ms);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(up, dup.p, (size_t)(nf + nc) * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return PB_OK;
}
