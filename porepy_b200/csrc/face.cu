// face.cu -- per-face discretizations (two-point flux approximation, first-order upwinding) on a light
// face-indexed grid handle: the face -> cell table and the three geometry arrays these schemes read.  Works
// for grids of any dimension (the reference delegates its 1-D MPFA / MPSA to TPFA, numerics/fv/mpfa.py:
// 690-712, mpsa.py:666-697); no interaction-region plan is built.
#include "csr_build.cuh"
#include "tpfa_diff.cuh"
#include "tpsa_face.cuh"
#include "tpsa_system.cuh"

#include <array>

// {nd, scalar balances, flux-pattern nnz}: what a TPSA row pattern was built for; nd = 0: no pattern
using TpsaKey = std::array<int64_t, 3>;

// The row pattern of one TPSA system: CSR arrays of nnz entries and, for the poromechanics and contact systems, the
// first entry of each block row.  Rebuilt when a call asks for another key.
struct TpsaPattern {
    TpsaKey key{};
    int64_t nnz = 0;
    DevBuf blk, ip, ix;
};

struct pb_facegrid {
    int64_t nc = 0, nf = 0;
    Stream stream;
    DevBuf face_cells, fnorm, fcent, ccent, farea, tmp;   // farea: set by pb_facegrid_set_face_areas
    DevBuf cf_ip, cf_ix;                                  // cell -> face lists (cell_faces, CSC)
    std::vector<uint8_t> face_ncell;                      // host: cells per face
    GeoView geo{};
    // TPSA systems: the neighbour lists of every cell (npairs < 0: not built yet), the face values of the last assembly
    // (read again by the pb_tpsa*_rhs calls) and the row pattern of each system; the three patterns live side by side
    int terms_nd = 0;
    int64_t npairs = -1;
    DevBuf fc_ptr, cc_ptr, cc_ix, cc_cell, terms[PB_TPSA_NTERMS];
    TpsaPattern sys, poro, ctc;
    // TPSA contact system: the interfaces of the last call (host copies of their topology)
    int64_t ctc_nm = -1, ctc_nk = -1;
    double ctc_ct = 0.0;
    std::vector<int32_t> ctc_face_h, ctc_cell_h;
    DevBuf ctc_fm, ctc_face, ctc_cell, ctc_pair, ctc_w, ctc_frame;
    // the stream's copies and kernels may still use the buffers, which go back to the pool right after
    ~pb_facegrid() { if (stream) cudaStreamSynchronize(stream); }
};

// one thread per cell: claim the first free slot of each of its faces
__global__ void face_cells_kernel(int64_t nc, const int32_t *__restrict__ cf_ip, const int32_t *__restrict__ cf_ix,
                                  const int8_t *__restrict__ cf_da, int32_t *__restrict__ fc, int *bad) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += (int64_t)gridDim.x * blockDim.x)
        for (int q = cf_ip[c]; q < cf_ip[c + 1]; ++q) {
            const int32_t f = cf_ix[q];
            const int32_t enc = (int32_t)((c << 1) | (cf_da[q] < 0 ? 1 : 0));
            if (atomicCAS(fc + 2 * (int64_t)f, -1, enc) != -1)
                if (atomicCAS(fc + 2 * (int64_t)f + 1, -1, enc) != -1) atomicExch(bad, 1);
        }
}
// slot 0 = the smaller cell index (the order of the host construction in plan_host.hpp)
__global__ void face_cells_order_kernel(int64_t nf, int32_t *__restrict__ fc) {
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < nf; f += (int64_t)gridDim.x * blockDim.x) {
        const int32_t a = fc[2 * f], b = fc[2 * f + 1];
        if (b >= 0 && b < a) { fc[2 * f] = b; fc[2 * f + 1] = a; }
    }
}

extern "C" int pb_facegrid_create(int64_t nc, int64_t nf, const int32_t *cf_indptr, const int32_t *cf_indices,
                                  const int8_t *cf_data, const double *face_normals, const double *face_centers,
                                  const double *cell_centers, pb_facegrid **out) {
    if (!out || !cf_indptr || !cf_indices || !cf_data || !face_normals || !face_centers || !cell_centers)
        return pb_fail_(PB_EINVAL, "null pointer");
    if (nc <= 0 || nf <= 0) return pb_fail_(PB_EINVAL, "empty grid");
    if (int rc = pb_require_device()) return rc;
    std::vector<uint8_t> ncell((size_t)nf, 0);
    for (int64_t q = 0; q < cf_indptr[nc]; ++q) {
        if (cf_indices[q] < 0 || cf_indices[q] >= nf) return pb_fail_(PB_EINVAL, "cell_faces index out of range");
        if (ncell[cf_indices[q]] < 255) ++ncell[cf_indices[q]];
    }
    std::unique_ptr<pb_facegrid> g(new pb_facegrid);
    g->nc = nc; g->nf = nf;
    g->face_ncell.swap(ncell);
    CUDA_TRY(g->stream.create());
    cudaStream_t st = g->stream;
    DevBuf &ip = g->cf_ip, &ix = g->cf_ix, da, bad;
    CUDA_TRY(ip.upload(cf_indptr, (size_t)nc + 1, st));
    CUDA_TRY(ix.upload(cf_indices, (size_t)cf_indptr[nc], st));
    CUDA_TRY(da.upload(cf_data, (size_t)cf_indptr[nc], st));
    CUDA_TRY(bad.ensure(sizeof(int)));
    CUDA_TRY(cudaMemsetAsync(bad.p, 0, sizeof(int), st));
    CUDA_TRY(g->face_cells.ensure((size_t)2 * nf * sizeof(int32_t)));
    CUDA_TRY(cudaMemsetAsync(g->face_cells.p, 0xFF, (size_t)2 * nf * sizeof(int32_t), st));
    face_cells_kernel<<<grid_stride_blocks(nc, 256, 16), 256, 0, st>>>(
        nc, ip.as<int32_t>(), ix.as<int32_t>(), da.as<int8_t>(), g->face_cells.as<int32_t>(), bad.as<int>());
    face_cells_order_kernel<<<grid_stride_blocks(nf, 256, 16), 256, 0, st>>>(nf, g->face_cells.as<int32_t>());
    pb_count_launch_(); pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    if (int rc = pb_upload_repacked_(st, g->tmp, g->fnorm, face_normals, 3, nf)) return rc;
    if (int rc = pb_upload_repacked_(st, g->tmp, g->fcent, face_centers, 3, nf)) return rc;
    if (int rc = pb_upload_repacked_(st, g->tmp, g->ccent, cell_centers, 3, nc)) return rc;
    int hbad = 0;
    CUDA_TRY(cudaMemcpyAsync(&hbad, bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (hbad) return pb_fail_(PB_EINVAL, "face with more than two neighbouring cells");
    g->geo = GeoView{nullptr, g->fnorm.as<double>(), g->fcent.as<double>(), nullptr, g->ccent.as<double>(), nullptr,
                     1, 3, 1, 3, 1, 3};
    *out = g.release();
    return PB_OK;
}

extern "C" void pb_facegrid_destroy(pb_facegrid *g) { delete g; }

__global__ void tpfa_kernel(int64_t nf, GeoView G, const double *__restrict__ perm, int64_t perm_cs,
                            int64_t perm_es, const uint8_t *__restrict__ bc,
                            const int32_t *__restrict__ face_cells, const int32_t *__restrict__ fc_ptr,
                            int vdim, TpfaOut o) {
    for (int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; f < nf; f += (int64_t)gridDim.x * blockDim.x)
        tpfa_face(f, G, perm, perm_cs, perm_es, bc, face_cells, fc_ptr, vdim, o);
}

template <int ND>
__global__ void tpsa_kernel(int64_t nf, GeoView G, const double *__restrict__ mu, const uint8_t *__restrict__ codes,
                            const double *__restrict__ robw, const uint8_t *__restrict__ flags,
                            const int32_t *__restrict__ face_cells, const int32_t *__restrict__ fc_ptr, TpsaOut o) {
    for (int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; f < nf; f += (int64_t)gridDim.x * blockDim.x)
        tpsa_face<ND>(f, G, mu, codes, robw, flags, face_cells, fc_ptr, o);
}

__global__ void upwind_kernel(int64_t nf, const double *__restrict__ q, const uint8_t *__restrict__ bc,
                              const int32_t *__restrict__ face_cells, int32_t *__restrict__ up_col,
                              double *__restrict__ neu_diag, double *__restrict__ dir_diag) {
    for (int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; f < nf; f += (int64_t)gridDim.x * blockDim.x)
        upwind_face(f, q, bc, face_cells, up_col, neu_diag, dir_diag);
}

extern "C" int pb_tpfa(pb_facegrid *g, const double *permeability, const uint8_t *bc_bits, const int32_t *fc_indptr,
                       int vdim, double *flux, double *bound_pressure_cell, double *vector_source,
                       double *bound_pressure_vector_source, double *bound_flux_diag,
                       double *bound_pressure_face_diag) {
    if (!g || !permeability || !bc_bits || !fc_indptr) return pb_fail_(PB_EINVAL, "null pointer");
    if (vdim < 1 || vdim > 3) return pb_fail_(PB_EINVAL, "1 <= vdim <= 3");
    cudaStream_t st = g->stream;
    const int64_t nf = g->nf, nc = g->nc;
    const size_t nnz = (size_t)fc_indptr[nf];
    DevBuf perm, bc, ip, o_flux, o_bpc, o_vs, o_bpvs, o_bf, o_bpf;
    { int rcs = pb_upload_repacked_(st, g->tmp, perm, permeability, 9, nc); if (rcs) return rcs; }
    CUDA_TRY(bc.upload(bc_bits, (size_t)nf, st));
    CUDA_TRY(ip.upload(fc_indptr, (size_t)nf + 1, st));
    CUDA_TRY(o_flux.ensure(nnz * sizeof(double)));
    CUDA_TRY(o_bpc.ensure(nnz * sizeof(double)));
    CUDA_TRY(o_vs.ensure(nnz * vdim * sizeof(double)));
    CUDA_TRY(o_bpvs.ensure(nnz * vdim * sizeof(double)));
    CUDA_TRY(o_bf.ensure((size_t)nf * sizeof(double)));
    CUDA_TRY(o_bpf.ensure((size_t)nf * sizeof(double)));
    TpfaOut o{o_flux.as<double>(), o_bpc.as<double>(), o_vs.as<double>(), o_bpvs.as<double>(),
              o_bf.as<double>(), o_bpf.as<double>()};
    tpfa_kernel<<<grid_stride_blocks(nf, 256, 16), 256, 0, st>>>(
        nf, g->geo, perm.as<double>(), 1, 9, bc.as<uint8_t>(), g->face_cells.as<int32_t>(), ip.as<int32_t>(), vdim, o);
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    auto down = [&](double *h, DevBuf &d, size_t n) -> cudaError_t {
        return h ? cudaMemcpyAsync(h, d.p, n * sizeof(double), cudaMemcpyDeviceToHost, st) : cudaSuccess;
    };
    CUDA_TRY(down(flux, o_flux, nnz));
    CUDA_TRY(down(bound_pressure_cell, o_bpc, nnz));
    CUDA_TRY(down(vector_source, o_vs, nnz * vdim));
    CUDA_TRY(down(bound_pressure_vector_source, o_bpvs, nnz * vdim));
    CUDA_TRY(down(bound_flux_diag, o_bf, (size_t)nf));
    CUDA_TRY(down(bound_pressure_face_diag, o_bpf, (size_t)nf));
    CUDA_TRY(cudaStreamSynchronize(st));
    return PB_OK;
}

__global__ void tpfa_diff_kernel(int64_t nf, GeoView G, const double *__restrict__ k,
                                 const int32_t *__restrict__ face_cells, const int32_t *__restrict__ fc_ptr,
                                 double *__restrict__ t_hf, double *__restrict__ T, double *__restrict__ dT_dk) {
    for (int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; f < nf; f += (int64_t)gridDim.x * blockDim.x)
        tpfa_diff_face(f, G, k, face_cells, fc_ptr, t_hf, T, dT_dk);
}

// Differentiable TPFA (tpfa_diff.cuh): k = 9 * nc doubles, cell-major; fc_indptr as for pb_tpfa; outputs t_hf (nhf),
// T (nf), dT_dk (nhf * 9); host pointers.
extern "C" int pb_tpfa_diff(pb_facegrid *g, const double *k, const int32_t *fc_indptr, double *t_hf, double *T,
                            double *dT_dk) {
    if (!g || !k || !fc_indptr || !t_hf || !T || !dT_dk) return pb_fail_(PB_EINVAL, "null pointer");
    cudaStream_t st = g->stream;
    const int64_t nf = g->nf, nc = g->nc;
    const size_t nhf = (size_t)fc_indptr[nf];
    DevBuf dk, ip, o_t, o_T, o_d;
    CUDA_TRY(dk.upload(k, (size_t)9 * nc, st));
    CUDA_TRY(ip.upload(fc_indptr, (size_t)nf + 1, st));
    CUDA_TRY(o_t.ensure(nhf * sizeof(double)));
    CUDA_TRY(o_T.ensure((size_t)nf * sizeof(double)));
    CUDA_TRY(o_d.ensure(nhf * 9 * sizeof(double)));
    tpfa_diff_kernel<<<grid_stride_blocks(nf, 256, 16), 256, 0, st>>>(
        nf, g->geo, dk.as<double>(), g->face_cells.as<int32_t>(), ip.as<int32_t>(), o_t.as<double>(), o_T.as<double>(),
        o_d.as<double>());
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(t_hf, o_t.p, nhf * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(T, o_T.p, (size_t)nf * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(dT_dk, o_d.p, nhf * 9 * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return PB_OK;
}

extern "C" int pb_upwind(pb_facegrid *g, const double *darcy_flux, const uint8_t *bc_bits, int32_t *upstream_cell,
                         double *neumann_diag, double *dirichlet_diag) {
    if (!g || !darcy_flux || !bc_bits || !upstream_cell || !neumann_diag || !dirichlet_diag)
        return pb_fail_(PB_EINVAL, "null pointer");
    cudaStream_t st = g->stream;
    const int64_t nf = g->nf;
    DevBuf q, bc, up, neu, dir;
    CUDA_TRY(q.upload(darcy_flux, (size_t)nf, st));
    CUDA_TRY(bc.upload(bc_bits, (size_t)nf, st));
    CUDA_TRY(up.ensure((size_t)nf * sizeof(int32_t)));
    CUDA_TRY(neu.ensure((size_t)nf * sizeof(double)));
    CUDA_TRY(dir.ensure((size_t)nf * sizeof(double)));
    upwind_kernel<<<grid_stride_blocks(nf, 256, 16), 256, 0, st>>>(nf, q.as<double>(), bc.as<uint8_t>(),
                                                                   g->face_cells.as<int32_t>(), up.as<int32_t>(),
                                                                   neu.as<double>(), dir.as<double>());
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(upstream_cell, up.p, (size_t)nf * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(neumann_diag, neu.p, (size_t)nf * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(dirichlet_diag, dir.p, (size_t)nf * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return PB_OK;
}

// ---- interface upwinding (UpwindCoupling.discretize, numerics/fv/upwind.py:427-528): per mortar cell the sign of
// the interface flux and the two upstream masks (flux > 0: the higher-dimensional side is upstream)
__global__ void upwind_coupling_kernel(int64_t n, const double *__restrict__ lam, double *__restrict__ sgn,
                                       double *__restrict__ from_primary, double *__restrict__ from_secondary) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double v = lam[i];
        const double s = v > 0.0 ? 1.0 : (v < 0.0 ? -1.0 : (v == 0.0 ? 0.0 : v));   // np.sign (nan stays nan)
        sgn[i] = s;
        from_primary[i] = s > 0.0 ? 1.0 : 0.0;
        from_secondary[i] = s > 0.0 ? 0.0 : 1.0;
    }
}

extern "C" int pb_upwind_coupling(int64_t n, const double *interface_flux, double *sign, double *from_primary,
                                  double *from_secondary) {
    if (n < 0 || (n > 0 && (!interface_flux || !sign || !from_primary || !from_secondary)))
        return pb_fail_(PB_EINVAL, "bad arguments");
    if (n == 0) return PB_OK;
    if (int rc = pb_require_device()) return rc;
    DevBuf in, o0, o1, o2;
    CUDA_TRY(in.upload(interface_flux, (size_t)n, 0));
    CUDA_TRY(o0.ensure((size_t)n * 8)); CUDA_TRY(o1.ensure((size_t)n * 8)); CUDA_TRY(o2.ensure((size_t)n * 8));
    upwind_coupling_kernel<<<grid_stride_blocks(n, 256, 16), 256>>>(n, in.as<double>(), o0.as<double>(),
                                                                    o1.as<double>(), o2.as<double>());
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpy(sign, o0.p, (size_t)n * 8, cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(from_primary, o1.p, (size_t)n * 8, cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(from_secondary, o2.p, (size_t)n * 8, cudaMemcpyDeviceToHost));
    return PB_OK;
}

extern "C" int pb_facegrid_set_face_areas(pb_facegrid *g, const double *face_areas) {
    if (!g || !face_areas) return pb_fail_(PB_EINVAL, "null pointer");
    CUDA_TRY(g->farea.upload(face_areas, (size_t)g->nf, g->stream));
    CUDA_TRY(cudaStreamSynchronize(g->stream));
    g->geo.farea = g->farea.as<double>();
    return PB_OK;
}

// ---- TPSA: the per-face terms (tpsa_face.cuh) and the assembled systems (tpsa_system.cuh) -------------------------
// Inputs of the TPSA calls on the device.
struct TpsaInputs {
    DevBuf mu, lam, vol, codes, rob, flags;
    bool any_rob = false;
};

// Checks the inputs and uploads them: lambda and cell_volumes only when given (the systems), the cells of each face from
// fc_indptr when given (pb_tpsa), else from the handle, whose fc_ptr is then built once.
static int tpsa_prepare(pb_facegrid *g, int nd, const double *mu, const double *lambda, const double *cell_volumes,
                        const uint8_t *codes, const double *robin_diag, const uint8_t *face_flags,
                        const int32_t *fc_indptr, TpsaInputs &in) {
    if (nd != 2 && nd != 3) return pb_fail_(PB_EINVAL, "Tpsa is only implemented for 2d and 3d grids.");
    if (!g->geo.farea) return pb_fail_(PB_EINVAL, "face areas not set (pb_facegrid_set_face_areas)");
    const int64_t nf = g->nf, nc = g->nc;
    for (int64_t c = 0; c < nc; ++c) {   // the scheme divides by mu and by mu / distance, the systems by lambda
        if (!(mu[c] > 0.0) || !std::isfinite(mu[c])) return pb_fail_(PB_EINVAL, "shear modulus must be finite and > 0");
        if (lambda && (!(lambda[c] > 0.0) || !std::isfinite(lambda[c])))
            return pb_fail_(PB_EINVAL, "first Lame parameter lambda must be finite and > 0");
    }
    for (int64_t q = 0; q < nd * nf; ++q) {
        if (codes[q] > PB_BC_ROB) return pb_fail_(PB_EINVAL, "boundary code out of range");
        in.any_rob |= codes[q] == PB_BC_ROB;
    }
    if (in.any_rob && !robin_diag) return pb_fail_(PB_EINVAL, "Robin faces need robin_diag");
    for (int64_t f = 0; f < nf; ++f) {
        const int len = fc_indptr ? fc_indptr[f + 1] - fc_indptr[f] : g->face_ncell[f];
        if (len < 1 || len > 2) return pb_fail_(PB_EINVAL, "fc_indptr: a face has one or two cells");
        if (face_flags[f] && len != 1) return pb_fail_(PB_EINVAL, "sign of internal faces does not make sense");
    }
    cudaStream_t st = g->stream;
    if (!fc_indptr && !g->fc_ptr.p) {   // CSR-by-face row pointer of cell_faces: where each face's (face, cell) values start
        std::vector<int32_t> fp((size_t)nf + 1, 0);
        for (int64_t f = 0; f < nf; ++f) fp[f + 1] = fp[f] + g->face_ncell[f];
        CUDA_TRY(g->fc_ptr.upload(fp, st));
        CUDA_TRY(cudaStreamSynchronize(st));
    }
    CUDA_TRY(in.mu.upload(mu, (size_t)nc, st));
    if (lambda) CUDA_TRY(in.lam.upload(lambda, (size_t)nc, st));
    if (cell_volumes) CUDA_TRY(in.vol.upload(cell_volumes, (size_t)nc, st));
    CUDA_TRY(in.codes.upload(codes, (size_t)nd * nf, st));
    if (in.any_rob) CUDA_TRY(in.rob.upload(robin_diag, (size_t)nd * nf, st));
    CUDA_TRY(in.flags.upload(face_flags, (size_t)nf, st));
    return PB_OK;
}

// The per-face kernel on the inputs in; fc_ptr[f]: the first (face, cell) entry of face f.
static int tpsa_face_launch(pb_facegrid *g, int nd, const TpsaInputs &in, const int32_t *fc_ptr, const TpsaOut &o) {
    const int64_t nf = g->nf;
    const double *rw = in.any_rob ? in.rob.as<double>() : nullptr;
    dispatch_nd<2, 3>(nd, [&](auto ND) {
        tpsa_kernel<ND><<<grid_stride_blocks(nf, 256, 16), 256, 0, g->stream>>>(
            nf, g->geo, in.mu.as<double>(), in.codes.as<uint8_t>(), rw, in.flags.as<uint8_t>(),
            g->face_cells.as<int32_t>(), fc_ptr, o);
    });
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}

// Two-point stress approximation (tpsa_face.cuh): value arrays of the 14 terms, layouts in include/poreb200.h.
extern "C" int pb_tpsa(pb_facegrid *g, int nd, const double *mu, const uint8_t *codes, const double *robin_diag,
                       const uint8_t *face_flags, const int32_t *fc_indptr, double **out, float *kernel_ms) {
    if (!g || !mu || !codes || !face_flags || !fc_indptr || !out) return pb_fail_(PB_EINVAL, "null pointer");
    TpsaInputs in;
    int rc = tpsa_prepare(g, nd, mu, nullptr, nullptr, codes, robin_diag, face_flags, fc_indptr, in);
    if (rc) return rc;
    cudaStream_t st = g->stream;
    const int64_t nf = g->nf;
    DevBuf dip, o_buf[PB_TPSA_NTERMS];
    CUDA_TRY(dip.upload(fc_indptr, (size_t)nf + 1, st));
    TpsaOut o{};
    size_t count[PB_TPSA_NTERMS];
    for (int k = 0; k < PB_TPSA_NTERMS; ++k) {
        count[k] = tpsa_term_size(k, nd, (size_t)fc_indptr[nf], (size_t)nf);
        if (!out[k]) continue;
        CUDA_TRY(o_buf[k].ensure(count[k] * sizeof(double)));
        o.t[k] = o_buf[k].as<double>();
    }
    KernelTimer timer;
    if (kernel_ms) {
        CUDA_TRY(timer.create());
        CUDA_TRY(timer.mark(0, st));
    }
    if ((rc = tpsa_face_launch(g, nd, in, dip.as<int32_t>(), o))) return rc;
    if (kernel_ms) CUDA_TRY(timer.mark(1, st));
    for (int k = 0; k < PB_TPSA_NTERMS; ++k)
        if (out[k]) CUDA_TRY(cudaMemcpyAsync(out[k], o_buf[k].p, count[k] * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (kernel_ms) CUDA_TRY(timer.ms(kernel_ms));
    return PB_OK;
}

// Stage 1 of the systems: the ten face terms they read, into buffers kept on the handle (T points at them).
static int tpsa_face_terms(pb_facegrid *g, int nd, const TpsaInputs &in, TpsaTerms &T) {
    const int64_t nf = g->nf;
    int64_t nfc = 0;   // (face, cell) entries
    for (int64_t f = 0; f < nf; ++f) nfc += g->face_ncell[f];
    const bool used[PB_TPSA_NTERMS] = {true, true, true, true, true, true, true, false, false, false, true, true, true,
                                       false};
    TpsaOut o{};
    for (int k = 0; k < PB_TPSA_NTERMS; ++k) {
        if (!used[k]) continue;
        CUDA_TRY(g->terms[k].ensure(tpsa_term_size(k, nd, (size_t)nfc, (size_t)nf) * sizeof(double)));
        o.t[k] = g->terms[k].as<double>();
        T.t[k] = o.t[k];
    }
    return tpsa_face_launch(g, nd, in, g->fc_ptr.as<int32_t>(), o);
}

static TpsaTopo tpsa_topo(pb_facegrid *g) {
    return TpsaTopo{g->nc, g->cf_ip.as<int32_t>(), g->cf_ix.as<int32_t>(), g->face_cells.as<int32_t>(),
                    g->fc_ptr.as<int32_t>()};
}

static TpsaMortars tpsa_mortars(pb_facegrid *g) {
    const int64_t nm = g->ctc_nm;
    const double *w = g->ctc_w.as<double>();
    return TpsaMortars{nm, g->ctc_nk, g->ctc_face.as<int32_t>(), g->ctc_cell.as<int32_t>(), g->ctc_fm.as<int32_t>(),
                       g->ctc_pair.as<int32_t>(), w, w + nm, w + 2 * nm, w + 3 * nm, g->ctc_frame.as<double>(), g->ctc_ct};
}

// ---- neighbour lists and row patterns ------------------------------------------------------------------------------
__global__ void tpsa_nb_count_kernel(TpsaTopo t, int32_t *__restrict__ count, int *bad) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < t.nc; c += (int64_t)gridDim.x * blockDim.x) {
        int32_t nb[kTpsaMaxNb];
        int n = tpsa_cell_neighbours(c, t, nb);
        if (n < 0) { atomicExch(bad, 1); n = 0; }
        count[c] = n;
    }
}

__global__ void tpsa_nb_list_kernel(TpsaTopo t, const int32_t *__restrict__ cc_ptr, int32_t *__restrict__ cc_ix,
                                    int32_t *__restrict__ cc_cell) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < t.nc; c += (int64_t)gridDim.x * blockDim.x) {
        int32_t nb[kTpsaMaxNb];
        const int n = tpsa_cell_neighbours(c, t, nb);
        for (int j = 0; j < n; ++j) { cc_ix[cc_ptr[c] + j] = nb[j]; cc_cell[cc_ptr[c] + j] = (int32_t)c; }
    }
}

// The neighbour lists of every cell, built once per handle and read by the patterns and block kernels of every TPSA
// system: cc_ix[cc_ptr[c] ..] the distinct cells sharing a face with c, c included, ascending; cc_cell the cell of
// each of the npairs entries.
static int tpsa_neighbours(pb_facegrid *g) {
    if (g->npairs >= 0) return PB_OK;
    cudaStream_t st = g->stream;
    const int64_t nc = g->nc;
    const TpsaTopo t = tpsa_topo(g);
    DevBuf count, bad;
    CUDA_TRY(count.ensure((size_t)nc * sizeof(int32_t)));
    CUDA_TRY(bad.ensure(sizeof(int)));
    CUDA_TRY(cudaMemsetAsync(bad.p, 0, sizeof(int), st));
    tpsa_nb_count_kernel<<<grid_stride_blocks(nc, 256, 16), 256, 0, st>>>(t, count.as<int32_t>(), bad.as<int>());
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(g->cc_ptr.ensure((size_t)(nc + 1) * sizeof(int32_t)));
    int hbad = 0;
    CUDA_TRY(cudaMemcpyAsync(&hbad, bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    int64_t total = 0;
    const int rc = pb_scan_offsets_(count.as<int32_t>(), g->cc_ptr.as<int32_t>(), nc, st, &total);
    if (rc) return rc;
    if (hbad) return pb_fail_(PB_ENOTIMPL, "Tpsa system: a cell has more than 31 face neighbours");
    CUDA_TRY(g->cc_ix.ensure((size_t)std::max<int64_t>(1, total) * sizeof(int32_t)));
    CUDA_TRY(g->cc_cell.ensure((size_t)std::max<int64_t>(1, total) * sizeof(int32_t)));
    tpsa_nb_list_kernel<<<grid_stride_blocks(nc, 256, 16), 256, 0, st>>>(
        t, g->cc_ptr.as<int32_t>(), g->cc_ix.as<int32_t>(), g->cc_cell.as<int32_t>());
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    g->npairs = total;
    return PB_OK;
}

// Sizes the CSR arrays of P for nrows rows and nnz entries and writes the last row pointer; the pattern kernels write
// the others.
static int tpsa_pattern_alloc(pb_facegrid *g, TpsaPattern &P, int64_t nrows, int64_t nnz) {
    if (nnz >= 0x7FFFFFFFll) return pb_fail_(PB_ENOTIMPL, "Tpsa system: the matrix does not fit int32 indices");
    CUDA_TRY(P.ip.ensure((size_t)(nrows + 1) * sizeof(int32_t)));
    CUDA_TRY(P.ix.ensure((size_t)std::max<int64_t>(1, nnz) * sizeof(int32_t)));
    const int32_t last = (int32_t)nnz;
    CUDA_TRY(cudaMemcpyAsync(P.ip.as<int32_t>() + nrows, &last, sizeof(int32_t), cudaMemcpyHostToDevice, g->stream));
    P.nnz = nnz;
    return PB_OK;
}

// P.blk: the first entry of every block row, from the entries per row that count(n) writes into n; *total: their sum.
template <class Count>
static int tpsa_block_offsets(pb_facegrid *g, TpsaPattern &P, int64_t *total, Count &&count) {
    DevBuf n;
    CUDA_TRY(n.ensure((size_t)g->nc * sizeof(int32_t)));
    count(n.as<int32_t>());
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(P.blk.ensure((size_t)(g->nc + 1) * sizeof(int64_t)));
    return pb_scan_offsets_(n.as<int32_t>(), P.blk.as<int64_t>(), g->nc, g->stream, total);
}

// Makes P the row pattern for key unless it already is: build(ND), ND = key[0], sizes P and launches the pattern
// kernels on the neighbour lists.
template <class Build>
static int tpsa_pattern(pb_facegrid *g, TpsaPattern &P, const TpsaKey &key, Build &&build) {
    if (P.key == key) return PB_OK;
    P.key = {};
    int rc = tpsa_neighbours(g);
    if (!rc) dispatch_nd<2, 3>((int)key[0], [&](auto ND) { rc = build(ND); });
    if (rc) return rc;
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(g->stream));
    P.key = key;
    return PB_OK;
}

template <int ND>
__global__ void tpsa_pattern_kernel(int64_t nc, const int32_t *__restrict__ cc_ptr, const int32_t *__restrict__ cc_ix,
                                    int32_t *__restrict__ ip, int32_t *__restrict__ ix) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += (int64_t)gridDim.x * blockDim.x)
        tpsa_pattern_rows<ND>(c, cc_ptr[c + 1] - cc_ptr[c], cc_ix + cc_ptr[c], cc_ptr[c], ip, ix);
}

// Row pattern of the three-field system: NZ entries per neighbour.
template <int ND>
static int tpsa_sys_pattern(pb_facegrid *g) {
    const int64_t nc = g->nc;
    TpsaPattern &P = g->sys;
    const int rc = tpsa_pattern_alloc(g, P, nc * TpsaDims<ND>::B, (int64_t)TpsaDims<ND>::NZ * g->npairs);
    if (rc) return rc;
    tpsa_pattern_kernel<ND><<<grid_stride_blocks(nc, 256, 16), 256, 0, g->stream>>>(
        nc, g->cc_ptr.as<int32_t>(), g->cc_ix.as<int32_t>(), P.ip.as<int32_t>(), P.ix.as<int32_t>());
    return PB_OK;
}

template <int ND, int NS>
__global__ void tpsa_poro_count_kernel(int64_t nc, const int32_t *__restrict__ cc_ptr, const int32_t *__restrict__ fp_ip,
                                       const int32_t *__restrict__ fp_ix, int32_t *__restrict__ count) {
    // clamped: a row past the int32 limit still makes the total overflow the limit of the caller
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += (int64_t)gridDim.x * blockDim.x)
        count[c] = (int32_t)min(tpsa_poro_row_count<ND, NS>(c, cc_ptr[c + 1] - cc_ptr[c], fp_ip, fp_ix), (int64_t)0x7fffffff);
}

template <int ND, int NS>
__global__ void tpsa_poro_pattern_kernel(int64_t nc, const int32_t *__restrict__ cc_ptr,
                                         const int32_t *__restrict__ cc_ix, const int64_t *__restrict__ blk_ptr,
                                         const int32_t *__restrict__ fp_ip, const int32_t *__restrict__ fp_ix,
                                         int32_t *__restrict__ ip, int32_t *__restrict__ ix) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += (int64_t)gridDim.x * blockDim.x)
        tpsa_poro_pattern_rows<ND, NS>(c, cc_ptr[c + 1] - cc_ptr[c], cc_ix + cc_ptr[c], blk_ptr[c], fp_ip, fp_ix, ip, ix);
}

// Row pattern of the system with NS scalar balances on the flux pattern fp (nc x nc, sorted rows).
template <int ND, int NS>
static int tpsa_poro_pattern(pb_facegrid *g, const CsrView &fp) {
    const int64_t nc = g->nc;
    const int32_t *cc_ptr = g->cc_ptr.as<int32_t>();
    TpsaPattern &P = g->poro;
    int64_t nnz = 0;
    int rc = tpsa_block_offsets(g, P, &nnz, [&](int32_t *count) {
        tpsa_poro_count_kernel<ND, NS><<<grid_stride_blocks(nc, 256, 16), 256, 0, g->stream>>>(nc, cc_ptr, fp.indptr,
                                                                                               fp.indices, count);
    });
    if (rc || (rc = tpsa_pattern_alloc(g, P, nc * TpsaPoroDims<ND, NS>::B, nnz))) return rc;
    tpsa_poro_pattern_kernel<ND, NS><<<grid_stride_blocks(nc, 256, 16), 256, 0, g->stream>>>(
        nc, cc_ptr, g->cc_ix.as<int32_t>(), P.blk.as<int64_t>(), fp.indptr, fp.indices, P.ip.as<int32_t>(),
        P.ix.as<int32_t>());
    return PB_OK;
}

template <int ND>
__global__ void tpsa_contact_count_kernel(TpsaTopo t, const int32_t *__restrict__ cc_ptr,
                                          const int32_t *__restrict__ face_mortar, int32_t *__restrict__ count) {
    using D = TpsaContactDims<ND>;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < t.nc; c += (int64_t)gridDim.x * blockDim.x)
        count[c] = D::M::NZ * (cc_ptr[c + 1] - cc_ptr[c]) + D::EXT * tpsa_contact_nfrac(c, t, face_mortar);
}

template <int ND>
__global__ void tpsa_contact_pattern_kernel(TpsaTopo t, const int32_t *__restrict__ cc_ptr,
                                            const int32_t *__restrict__ cc_ix, const int64_t *__restrict__ blk_ptr,
                                            TpsaMortars I, int32_t *__restrict__ ip, int32_t *__restrict__ ix) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < t.nc; c += (int64_t)gridDim.x * blockDim.x)
        tpsa_contact_pattern_rows<ND>(c, cc_ptr[c + 1] - cc_ptr[c], cc_ix + cc_ptr[c], blk_ptr[c], t, I, ip, ix);
}

// one thread per interface row (force and contact rows)
template <int ND>
__global__ void tpsa_contact_iface_pattern_kernel(TpsaTopo t, const int64_t *__restrict__ blk_ptr, TpsaMortars I,
                                                  int32_t *__restrict__ ip, int32_t *__restrict__ ix) {
    const int64_t n = (int64_t)ND * (I.nm + I.nk);
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (int64_t)gridDim.x * blockDim.x)
        tpsa_contact_iface_pattern<ND>(q, t.nc, blk_ptr[t.nc], t, I, ip, ix);
}

// Row pattern of the contact system, from the interface topology already on the handle: the block rows, then ND nm
// force rows of LF entries and ND nk contact rows of LC entries.
template <int ND>
static int tpsa_contact_pattern(pb_facegrid *g) {
    using D = TpsaContactDims<ND>;
    const int64_t nc = g->nc, ni = (int64_t)ND * (g->ctc_nm + g->ctc_nk);
    const int32_t *cc_ptr = g->cc_ptr.as<int32_t>();
    const TpsaTopo t = tpsa_topo(g);
    const TpsaMortars I = tpsa_mortars(g);
    TpsaPattern &P = g->ctc;
    int64_t ncell = 0;
    int rc = tpsa_block_offsets(g, P, &ncell, [&](int32_t *count) {
        tpsa_contact_count_kernel<ND><<<grid_stride_blocks(nc, 256, 16), 256, 0, g->stream>>>(t, cc_ptr, I.face_mortar,
                                                                                              count);
    });
    const int64_t nnz = ncell + (int64_t)ND * I.nm * D::LF + (int64_t)ND * I.nk * D::LC;
    if (rc || (rc = tpsa_pattern_alloc(g, P, nc * D::B + ni, nnz))) return rc;
    tpsa_contact_pattern_kernel<ND><<<grid_stride_blocks(nc, 256, 16), 256, 0, g->stream>>>(
        t, cc_ptr, g->cc_ix.as<int32_t>(), P.blk.as<int64_t>(), I, P.ip.as<int32_t>(), P.ix.as<int32_t>());
    if (ni) tpsa_contact_iface_pattern_kernel<ND><<<grid_stride_blocks(ni, 256, 16), 256, 0, g->stream>>>(
        t, P.blk.as<int64_t>(), I, P.ip.as<int32_t>(), P.ix.as<int32_t>());
    return PB_OK;
}

// ---- assembly ------------------------------------------------------------------------------------------------------
// A TPSA system on the pattern P (nrows x nrows), in two stages: the face terms (tpsa_face_terms), then
// launch(ND, T, values of A), which gathers the blocks of A from them.  stage_ms (optional): the two stage times in ms.
template <class Launch>
static int tpsa_assemble(pb_facegrid *g, int nd, const TpsaInputs &in, const TpsaPattern &P, int64_t nrows,
                         pb_csr **out, float *stage_ms, Launch &&launch) {
    CsrPtr a;
    int rc = pb_csr_from_device_pattern_(nrows, nrows, P.nnz, P.ip.as<int32_t>(), P.ix.as<int32_t>(), a);
    if (rc) return rc;
    cudaStream_t st = g->stream;
    KernelTimer timer;
    if (stage_ms) {
        CUDA_TRY(timer.create(3));
        CUDA_TRY(timer.mark(0, st));
    }
    TpsaTerms T{};
    if ((rc = tpsa_face_terms(g, nd, in, T))) return rc;
    if (stage_ms) CUDA_TRY(timer.mark(1, st));
    dispatch_nd<2, 3>(nd, [&](auto ND) { launch(ND, T, pb_csr_view_(a.get()).data); });
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    if (stage_ms) CUDA_TRY(timer.mark(2, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (stage_ms) {
        CUDA_TRY(timer.ms(stage_ms, 0));
        CUDA_TRY(timer.ms(stage_ms + 1, 1));
    }
    g->terms_nd = nd;
    *out = a.release();
    return PB_OK;
}

// one thread per row of b: the mechanics rows of every cell, its NS scalar rows (0: they are written at every
// linearization), then the ND (nm + nk) interface rows of the contact system (none for the others: I.nm = I.nk = 0)
template <int ND, int NS>
__global__ void tpsa_rhs_kernel(TpsaTopo t, TpsaMortars I, TpsaTerms T, const double *__restrict__ g,
                                const double *__restrict__ f, const double *__restrict__ sr,
                                const double *__restrict__ sp, double *__restrict__ b) {
    constexpr int NR = TpsaDims<ND>::NR, B = TpsaDims<ND>::B + NS;
    const int64_t ncell = t.nc * B, n = ncell + (int64_t)ND * (I.nm + I.nk);
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (int64_t)gridDim.x * blockDim.x) {
        if (q >= ncell) { b[q] = tpsa_contact_iface_rhs<ND>(q - ncell, t, I, T, g); continue; }
        const int64_t c = q / B;
        const int l = (int)(q - c * B);
        if (l > ND + NR) { b[q] = 0.0; continue; }
        const double src = l < ND ? (f ? f[c * ND + l] : 0.0)
                                   : (l < ND + NR ? (sr ? sr[c * NR + l - ND] : 0.0) : (sp ? sp[c] : 0.0));
        b[q] = tpsa_rhs_row<ND>(c, l, t, T, g, src);
    }
}

// b of the last assembly on the handle (dimension nd, NS scalar balances, with the interface rows when contact): the
// boundary values and the optional sources uploaded, the boundary terms read from the handle.
template <int NS>
static int tpsa_rhs(pb_facegrid *g, int nd, bool contact, const double *bc_values, const double *body_force,
                    const double *angular_source, const double *mass_source, double *rhs_dev) {
    const int64_t nf = g->nf, nc = g->nc;
    const int nr = nd == 3 ? 3 : 1;
    cudaStream_t st = g->stream;
    DevBuf dg, df, dsr, dsp;
    CUDA_TRY(dg.upload(bc_values, (size_t)nd * nf, st));
    if (body_force) CUDA_TRY(df.upload(body_force, (size_t)nd * nc, st));
    if (angular_source) CUDA_TRY(dsr.upload(angular_source, (size_t)nr * nc, st));
    if (mass_source) CUDA_TRY(dsp.upload(mass_source, (size_t)nc, st));
    TpsaTerms T{};
    for (int k = PB_TPSA_BOUND_STRESS; k <= PB_TPSA_BOUND_MASS_DISPLACEMENT; ++k) T.t[k] = g->terms[k].as<double>();
    const TpsaTopo t = tpsa_topo(g);
    const TpsaMortars I = contact ? tpsa_mortars(g) : TpsaMortars{};
    const int64_t rows = nc * (nd + nr + 1 + NS) + (int64_t)nd * (I.nm + I.nk);
    const double *pf = body_force ? df.as<double>() : nullptr, *psr = angular_source ? dsr.as<double>() : nullptr,
                 *psp = mass_source ? dsp.as<double>() : nullptr;
    dispatch_nd<2, 3>(nd, [&](auto ND) {
        tpsa_rhs_kernel<ND, NS><<<grid_stride_blocks(rows, 256, 16), 256, 0, st>>>(t, I, T, dg.as<double>(), pf, psr,
                                                                                   psp, rhs_dev);
    });
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(st));
    return PB_OK;
}

// ---- TPSA three-field system ---------------------------------------------------------------------------------------
// one thread per block (c, k) of A, i.e. per entry of the neighbour lists: consecutive threads write consecutive
// segments of the same rows
template <int ND>
__global__ void tpsa_system_kernel(int64_t npairs, TpsaTopo t, const int32_t *__restrict__ cc_ptr,
                                   const int32_t *__restrict__ cc_ix, const int32_t *__restrict__ cc_cell, TpsaTerms T,
                                   const double *__restrict__ mu, const double *__restrict__ lam,
                                   const double *__restrict__ vol, double *__restrict__ a) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < npairs; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t c = cc_cell[e];
        tpsa_system_block<ND>(c, (int)(e - cc_ptr[c]), t, cc_ptr, cc_ix, T, mu, lam, vol, a);
    }
}

extern "C" int pb_tpsa_system(pb_facegrid *g, int nd, const double *mu, const double *lambda,
                              const double *cell_volumes, const uint8_t *codes, const double *robin_diag,
                              const uint8_t *face_flags, pb_csr **out, float *stage_ms) {
    if (!g || !mu || !lambda || !cell_volumes || !codes || !face_flags || !out)
        return pb_fail_(PB_EINVAL, "null pointer");
    TpsaInputs in;
    int rc = tpsa_prepare(g, nd, mu, lambda, cell_volumes, codes, robin_diag, face_flags, nullptr, in);
    if (rc) return rc;
    rc = tpsa_pattern(g, g->sys, {nd, 0, 0}, [&](auto ND) { return tpsa_sys_pattern<ND>(g); });
    if (rc) return rc;
    const TpsaTopo t = tpsa_topo(g);
    const int64_t np = g->npairs;
    return tpsa_assemble(g, nd, in, g->sys, g->nc * (nd == 3 ? 7 : 4), out, stage_ms,
                         [&](auto ND, const TpsaTerms &T, double *a) {
        tpsa_system_kernel<ND><<<grid_stride_blocks(np, 256, 16), 256, 0, g->stream>>>(
            np, t, g->cc_ptr.as<int32_t>(), g->cc_ix.as<int32_t>(), g->cc_cell.as<int32_t>(), T, in.mu.as<double>(),
            in.lam.as<double>(), in.vol.as<double>(), a);
    });
}

extern "C" int pb_tpsa_rhs(pb_facegrid *g, const double *bc_values, const double *body_force,
                           const double *angular_source, const double *mass_source, double *rhs_dev) {
    if (!g || !bc_values || !rhs_dev) return pb_fail_(PB_EINVAL, "null pointer");
    const int nd = g->terms_nd;
    if (nd != 2 && nd != 3) return pb_fail_(PB_EINVAL, "pb_tpsa_system has not been called");
    return tpsa_rhs<0>(g, nd, false, bc_values, body_force, angular_source, mass_source, rhs_dev);
}

// ---- TPSA poromechanics (NS = 1) and thermo-poromechanics (NS = 2) systems -----------------------------------------
// one thread per block (c, k), as tpsa_system_kernel
template <int ND, int NS>
__global__ void tpsa_poro_system_kernel(int64_t npairs, TpsaTopo t, const int32_t *__restrict__ cc_ptr,
                                        const int32_t *__restrict__ cc_ix, const int32_t *__restrict__ cc_cell,
                                        const int64_t *__restrict__ blk_ptr, TpsaTerms T, const double *__restrict__ mu,
                                        const double *__restrict__ lam, const double *__restrict__ alpha,
                                        const double *__restrict__ vol, double *__restrict__ a) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < npairs; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t c = cc_cell[e];
        tpsa_poro_block<ND, NS>(c, (int)(e - cc_ptr[c]), t, cc_ptr, cc_ix, blk_ptr, T, mu, lam, alpha, vol, a);
    }
}

// one thread per cell: its scalar rows; the mechanics rows of the block row come first
template <int ND, int NS>
__global__ void tpsa_poro_fluid_kernel(int64_t nc, const int32_t *__restrict__ cc_ptr,
                                       const int64_t *__restrict__ blk_ptr, const int32_t *__restrict__ ix,
                                       const int32_t *__restrict__ jf_ip, const int32_t *__restrict__ jf_ix,
                                       const double *__restrict__ jf_a, const double *__restrict__ neg_res,
                                       double *__restrict__ a, double *__restrict__ b, int *__restrict__ missing) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row0 = blk_ptr[c] + (int64_t)TpsaPoroDims<ND, NS>::NZ * (cc_ptr[c + 1] - cc_ptr[c]);
        const int m = tpsa_poro_fluid_row<ND, NS>(c, nc, blk_ptr, row0, ix, jf_ip, jf_ix, jf_a, neg_res, a, b);
        if (m && missing) atomicAdd(missing, m);
    }
}

// The names the poromechanics (NS = 1) and thermo-poromechanics (NS = 2) entry points report in their errors.
template <int NS>
struct TpsaPoroNames;
template <>
struct TpsaPoroNames<1> {
    static constexpr const char *system = "pb_tpsa_poro_system", *model = "TPSA poromechanics",
                                *jac = "fluid Jacobian must be num_cells x 2 num_cells ([p_t | p])";
};
template <>
struct TpsaPoroNames<2> {
    static constexpr const char *system = "pb_tpsa_thm_system", *model = "TPSA thermo-poromechanics",
                                *jac = "balance Jacobian must be 2 num_cells x 3 num_cells ([p_t | p | T])";
};

template <int NS>
static int tpsa_poro_system(pb_facegrid *g, int nd, const double *mu, const double *lambda, const double *alpha,
                            const double *cell_volumes, const uint8_t *codes, const double *robin_diag,
                            const uint8_t *face_flags, const pb_csr *flux_pattern, pb_csr **out, float *stage_ms) {
    if (!g || !mu || !lambda || !alpha || !cell_volumes || !codes || !face_flags || !flux_pattern || !out)
        return pb_fail_(PB_EINVAL, "null pointer");
    const int64_t nc = g->nc;
    for (int64_t c = 0; c < nc; ++c)
        if (!std::isfinite(alpha[c])) return pb_fail_(PB_EINVAL, "Biot coefficient alpha must be finite");
    const CsrView fp = pb_csr_view_(flux_pattern);
    if (fp.nrows != nc || fp.ncols != nc) return pb_fail_(PB_EINVAL, "flux pattern must be num_cells x num_cells");
    TpsaInputs in;
    int rc = tpsa_prepare(g, nd, mu, lambda, cell_volumes, codes, robin_diag, face_flags, nullptr, in);
    if (rc) return rc;
    rc = tpsa_pattern(g, g->poro, {nd, NS, fp.nnz}, [&](auto ND) { return tpsa_poro_pattern<ND, NS>(g, fp); });
    if (rc) return rc;
    DevBuf dal;
    CUDA_TRY(dal.upload(alpha, (size_t)nc, g->stream));
    const TpsaTopo t = tpsa_topo(g);
    const int64_t np = g->npairs;
    return tpsa_assemble(g, nd, in, g->poro, nc * ((nd == 3 ? 7 : 4) + NS), out, stage_ms,
                         [&](auto ND, const TpsaTerms &T, double *a) {
        tpsa_poro_system_kernel<ND, NS><<<grid_stride_blocks(np, 256, 16), 256, 0, g->stream>>>(
            np, t, g->cc_ptr.as<int32_t>(), g->cc_ix.as<int32_t>(), g->cc_cell.as<int32_t>(), g->poro.blk.as<int64_t>(),
            T, in.mu.as<double>(), in.lam.as<double>(), dal.as<double>(), in.vol.as<double>(), a);
    });
}

template <int NS>
static int tpsa_poro_rhs(pb_facegrid *g, const double *bc_values, const double *body_force,
                         const double *angular_source, const double *mass_source, double *rhs_dev) {
    if (!g || !bc_values || !rhs_dev) return pb_fail_(PB_EINVAL, "null pointer");
    const int nd = (int)g->poro.key[0];
    if ((nd != 2 && nd != 3) || g->poro.key[1] != NS || g->terms_nd != nd)
        return pb_fail_(PB_EINVAL, std::string(TpsaPoroNames<NS>::system) + " has not been called");
    return tpsa_rhs<NS>(g, nd, false, bc_values, body_force, angular_source, mass_source, rhs_dev);
}

template <int NS>
static int tpsa_poro_fluid_rows(pb_facegrid *g, pb_csr *a, const pb_csr *jf, const double *neg_res_dev,
                                double *rhs_dev, int *missing_dev, uint64_t stream) {
    if (!g || !a || !jf || !neg_res_dev || !rhs_dev) return pb_fail_(PB_EINVAL, "null pointer");
    const int nd = (int)g->poro.key[0];
    if ((nd != 2 && nd != 3) || g->poro.key[1] != NS)
        return pb_fail_(PB_EINVAL, std::string(TpsaPoroNames<NS>::system) + " has not been called");
    const int64_t nc = g->nc;
    const int B = (nd == 3 ? 7 : 4) + NS;
    const CsrView va = pb_csr_view_(a), vj = pb_csr_view_(jf);
    if (va.nrows != nc * B || va.ncols != nc * B || va.nnz != g->poro.nnz)
        return pb_fail_(PB_EINVAL, std::string("the matrix is not the ") + TpsaPoroNames<NS>::model +
                                       " system of this grid");
    if (vj.nrows != NS * nc || vj.ncols != (1 + NS) * nc) return pb_fail_(PB_EINVAL, TpsaPoroNames<NS>::jac);
    dispatch_nd<2, 3>(nd, [&](auto ND) {
        tpsa_poro_fluid_kernel<ND, NS><<<grid_stride_blocks(nc, 256, 16), 256, 0, (cudaStream_t)stream>>>(
            nc, g->cc_ptr.as<int32_t>(), g->poro.blk.as<int64_t>(), va.indices, vj.indptr, vj.indices, vj.data,
            neg_res_dev, va.data, rhs_dev, missing_dev);
    });
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}

extern "C" int pb_tpsa_poro_system(pb_facegrid *g, int nd, const double *mu, const double *lambda, const double *alpha,
                                   const double *cell_volumes, const uint8_t *codes, const double *robin_diag,
                                   const uint8_t *face_flags, const pb_csr *flux_pattern, pb_csr **out,
                                   float *stage_ms) {
    return tpsa_poro_system<1>(g, nd, mu, lambda, alpha, cell_volumes, codes, robin_diag, face_flags, flux_pattern, out,
                               stage_ms);
}
extern "C" int pb_tpsa_poro_rhs(pb_facegrid *g, const double *bc_values, const double *body_force,
                                const double *angular_source, const double *mass_source, double *rhs_dev) {
    return tpsa_poro_rhs<1>(g, bc_values, body_force, angular_source, mass_source, rhs_dev);
}
extern "C" int pb_tpsa_poro_fluid_rows(pb_facegrid *g, pb_csr *a, const pb_csr *jf, const double *neg_res_dev,
                                       double *rhs_dev, int *missing_dev, uint64_t stream) {
    return tpsa_poro_fluid_rows<1>(g, a, jf, neg_res_dev, rhs_dev, missing_dev, stream);
}

extern "C" int pb_tpsa_thm_system(pb_facegrid *g, int nd, const double *mu, const double *lambda, const double *alpha,
                                  const double *cell_volumes, const uint8_t *codes, const double *robin_diag,
                                  const uint8_t *face_flags, const pb_csr *flux_pattern, pb_csr **out, float *stage_ms) {
    return tpsa_poro_system<2>(g, nd, mu, lambda, alpha, cell_volumes, codes, robin_diag, face_flags, flux_pattern, out,
                               stage_ms);
}
extern "C" int pb_tpsa_thm_rhs(pb_facegrid *g, const double *bc_values, const double *body_force,
                               const double *angular_source, const double *mass_source, double *rhs_dev) {
    return tpsa_poro_rhs<2>(g, bc_values, body_force, angular_source, mass_source, rhs_dev);
}
extern "C" int pb_tpsa_thm_balance_rows(pb_facegrid *g, pb_csr *a, const pb_csr *jf, const double *neg_res_dev,
                                        double *rhs_dev, int *missing_dev, uint64_t stream) {
    return tpsa_poro_fluid_rows<2>(g, a, jf, neg_res_dev, rhs_dev, missing_dev, stream);
}

// ---- TPSA elasticity with fractures in frictional contact ----------------------------------------------------------
// one thread per block (c, k), as tpsa_system_kernel
template <int ND>
__global__ void tpsa_contact_block_kernel(int64_t npairs, TpsaTopo t, const int32_t *__restrict__ cc_ptr,
                                          const int32_t *__restrict__ cc_ix, const int32_t *__restrict__ cc_cell,
                                          const int64_t *__restrict__ blk_ptr, TpsaMortars I, TpsaTerms T,
                                          const double *__restrict__ mu, const double *__restrict__ lam,
                                          const double *__restrict__ vol, double *__restrict__ a) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < npairs; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t c = cc_cell[e];
        tpsa_contact_block<ND>(c, (int)(e - cc_ptr[c]), t, cc_ptr, cc_ix, blk_ptr, I, T, mu, lam, vol, a);
    }
}

template <int ND>
__global__ void tpsa_contact_iface_kernel(TpsaTopo t, const int64_t *__restrict__ blk_ptr, TpsaMortars I, TpsaTerms T,
                                          double *__restrict__ a) {
    const int64_t n = (int64_t)ND * (I.nm + I.nk);
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (int64_t)gridDim.x * blockDim.x)
        tpsa_contact_iface_row<ND>(q, blk_ptr[t.nc], t, I, T, a);
}

// one thread per contact row
template <int ND>
__global__ void tpsa_contact_law_kernel(int64_t nrows, int64_t c0, int64_t row0, int64_t e0,
                                        const int32_t *__restrict__ ix, const int32_t *__restrict__ jc_ip,
                                        const int32_t *__restrict__ jc_ix, const double *__restrict__ jc_a,
                                        const double *__restrict__ neg_res, double *__restrict__ a,
                                        double *__restrict__ b, int *__restrict__ missing) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        const int m = tpsa_contact_law_row<ND>(r, c0, e0, row0 + r, ix, jc_ip, jc_ix, jc_a, neg_res, a, b);
        if (m && missing) atomicAdd(missing, m);
    }
}

// Checks the interface description and puts it on the handle; *same: its topology is the one of the cached pattern.
static int tpsa_contact_interfaces(pb_facegrid *g, int nd, int64_t nm, int64_t nk, const int32_t *mortar_face,
                                   const int32_t *mortar_cell, const double *m2p, const double *p2m, const double *sign,
                                   const double *vol, const double *frames, double ct, bool *same) {
    const int64_t nf = g->nf;
    if (nm < 0 || nk < 0 || nm != 2 * nk) return pb_fail_(PB_EINVAL, "every fracture cell needs two mortar cells");
    if (nm && (!mortar_face || !mortar_cell || !m2p || !p2m || !sign || !vol || !frames))
        return pb_fail_(PB_EINVAL, "null pointer");
    if (!std::isfinite(ct)) return pb_fail_(PB_EINVAL, "characteristic traction must be finite");
    std::vector<int32_t> fm((size_t)nf, -1), pair((size_t)2 * nk, -1);
    for (int64_t m = 0; m < nm; ++m) {
        const int32_t f = mortar_face[m], k = mortar_cell[m];
        if (f < 0 || f >= nf || k < 0 || k >= nk) return pb_fail_(PB_EINVAL, "mortar face or fracture cell out of range");
        if (fm[f] >= 0) return pb_fail_(PB_EINVAL, "a face with more than one mortar cell (non-matching mortar grid)");
        if (g->face_ncell[f] != 1) return pb_fail_(PB_EINVAL, "a fracture face must have exactly one cell");
        fm[f] = (int32_t)m;
        if (pair[2 * k] < 0) pair[2 * k] = (int32_t)m;
        else if (pair[2 * k + 1] < 0) pair[2 * k + 1] = (int32_t)m;
        else return pb_fail_(PB_EINVAL, "a fracture cell with more than two mortar cells");
        for (const double *v : {m2p + m, p2m + m, sign + m, vol + m})
            if (!std::isfinite(*v)) return pb_fail_(PB_EINVAL, "mortar weights must be finite");
    }
    for (int64_t q = 0; q < (int64_t)nd * nd * nk; ++q)
        if (!std::isfinite(frames[q])) return pb_fail_(PB_EINVAL, "local coordinates must be finite");
    *same = g->ctc_nm == nm && g->ctc_nk == nk &&
            std::equal(mortar_face, mortar_face + nm, g->ctc_face_h.begin()) &&
            std::equal(mortar_cell, mortar_cell + nm, g->ctc_cell_h.begin());
    cudaStream_t st = g->stream;
    std::vector<double> w((size_t)std::max<int64_t>(1, 4 * nm));
    for (int64_t m = 0; m < nm; ++m) { w[m] = m2p[m]; w[nm + m] = p2m[m]; w[2 * nm + m] = sign[m]; w[3 * nm + m] = vol[m]; }
    std::vector<int32_t> face_h(mortar_face, mortar_face + nm), cell_h(mortar_cell, mortar_cell + nm);
    face_h.push_back(0);
    cell_h.push_back(0);
    for (int64_t k = 0; k < nk; ++k)
        if (pair[2 * k] > pair[2 * k + 1]) std::swap(pair[2 * k], pair[2 * k + 1]);
    pair.push_back(0);
    CUDA_TRY(g->ctc_fm.upload(fm, st));
    CUDA_TRY(g->ctc_face.upload(face_h, st));
    CUDA_TRY(g->ctc_cell.upload(cell_h, st));
    CUDA_TRY(g->ctc_pair.upload(pair, st));
    CUDA_TRY(g->ctc_w.upload(w, st));
    std::vector<double> fr((size_t)nd * nd * nk + 1, 0.0);
    if (nk) std::copy(frames, frames + (size_t)nd * nd * nk, fr.begin());
    CUDA_TRY(g->ctc_frame.upload(fr, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    face_h.pop_back();
    cell_h.pop_back();
    g->ctc_face_h = face_h;
    g->ctc_cell_h = cell_h;
    g->ctc_nm = nm;
    g->ctc_nk = nk;
    g->ctc_ct = ct;
    return PB_OK;
}

extern "C" int pb_tpsa_contact_system(pb_facegrid *g, int nd, const double *mu, const double *lambda,
                                      const double *cell_volumes, const uint8_t *codes, const double *robin_diag,
                                      const uint8_t *face_flags, int64_t num_mortar, int64_t num_fracture_cells,
                                      const int32_t *mortar_face, const int32_t *mortar_cell, const double *m2p_weight,
                                      const double *p2m_weight, const double *mortar_sign, const double *mortar_volume,
                                      const double *frames, double characteristic_traction, pb_csr **out,
                                      float *stage_ms) {
    if (!g || !mu || !lambda || !cell_volumes || !codes || !face_flags || !out)
        return pb_fail_(PB_EINVAL, "null pointer");
    TpsaInputs in;
    int rc = tpsa_prepare(g, nd, mu, lambda, cell_volumes, codes, robin_diag, face_flags, nullptr, in);
    if (rc) return rc;
    bool same = false;
    const TpsaKey key{nd, 0, 0}, had = g->ctc.key;
    g->ctc.key = {};   // set again once the pattern on the handle belongs to the interfaces uploaded below
    rc = tpsa_contact_interfaces(g, nd, num_mortar, num_fracture_cells, mortar_face, mortar_cell, m2p_weight,
                                 p2m_weight, mortar_sign, mortar_volume, frames, characteristic_traction, &same);
    if (rc) return rc;
    if (same) g->ctc.key = had;
    rc = tpsa_pattern(g, g->ctc, key, [&](auto ND) { return tpsa_contact_pattern<ND>(g); });
    if (rc) return rc;
    const TpsaTopo t = tpsa_topo(g);
    const TpsaMortars I = tpsa_mortars(g);
    const int64_t np = g->npairs, ni = (int64_t)nd * (g->ctc_nm + g->ctc_nk);
    return tpsa_assemble(g, nd, in, g->ctc, g->nc * (nd == 3 ? 7 : 4) + ni, out, stage_ms,
                         [&](auto ND, const TpsaTerms &T, double *a) {
        tpsa_contact_block_kernel<ND><<<grid_stride_blocks(np, 256, 16), 256, 0, g->stream>>>(
            np, t, g->cc_ptr.as<int32_t>(), g->cc_ix.as<int32_t>(), g->cc_cell.as<int32_t>(), g->ctc.blk.as<int64_t>(),
            I, T, in.mu.as<double>(), in.lam.as<double>(), in.vol.as<double>(), a);
        if (ni) tpsa_contact_iface_kernel<ND><<<grid_stride_blocks(ni, 256, 16), 256, 0, g->stream>>>(
            t, g->ctc.blk.as<int64_t>(), I, T, a);
    });
}

extern "C" int pb_tpsa_contact_rhs(pb_facegrid *g, const double *bc_values, const double *body_force,
                                   const double *angular_source, const double *mass_source, double *rhs_dev) {
    if (!g || !bc_values || !rhs_dev) return pb_fail_(PB_EINVAL, "null pointer");
    const int nd = (int)g->ctc.key[0];
    if ((nd != 2 && nd != 3) || g->terms_nd != nd) return pb_fail_(PB_EINVAL, "pb_tpsa_contact_system has not been called");
    return tpsa_rhs<0>(g, nd, true, bc_values, body_force, angular_source, mass_source, rhs_dev);
}

extern "C" int pb_tpsa_contact_rows(pb_facegrid *g, pb_csr *a, const pb_csr *jc, const double *neg_res_dev,
                                    double *rhs_dev, int *missing_dev, uint64_t stream) {
    if (!g || !a || !jc || !neg_res_dev || !rhs_dev) return pb_fail_(PB_EINVAL, "null pointer");
    const int nd = (int)g->ctc.key[0];
    if (nd != 2 && nd != 3) return pb_fail_(PB_EINVAL, "pb_tpsa_contact_system has not been called");
    const int64_t nc = g->nc, nm = g->ctc_nm, nk = g->ctc_nk, c0 = nc * (nd == 3 ? 7 : 4);
    const int64_t nrows = c0 + (int64_t)nd * (nm + nk);
    const CsrView va = pb_csr_view_(a), vj = pb_csr_view_(jc);
    if (va.nrows != nrows || va.ncols != nrows || va.nnz != g->ctc.nnz)
        return pb_fail_(PB_EINVAL, "the matrix is not the TPSA contact system of this grid");
    if (vj.nrows != (int64_t)nd * nk || vj.ncols != (int64_t)nd * (nk + nm))
        return pb_fail_(PB_EINVAL, "contact Jacobian must be nd num_fracture_cells x nd (num_fracture_cells + num_mortar) "
                                   "([t | u_j])");
    if (!nk) return PB_OK;
    // the contact rows are the last nd nk rows, of 3 nd entries each
    const int64_t n = (int64_t)nd * nk, e0 = g->ctc.nnz - n * 3 * nd;
    dispatch_nd<2, 3>(nd, [&](auto ND) {
        tpsa_contact_law_kernel<ND><<<grid_stride_blocks(n, 256, 16), 256, 0, (cudaStream_t)stream>>>(
            n, c0, c0 + (int64_t)nd * nm, e0, va.indices, vj.indptr, vj.indices, vj.data, neg_res_dev, va.data, rhs_dev,
            missing_dev);
    });
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    return PB_OK;
}
