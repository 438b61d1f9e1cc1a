// geometry.cu -- Grid.compute_geometry for 3-D grids on the device (SURVEY.md 8(f) rank 4; reference
// grids/grid.py:362-381 dispatch, :572-778 _compute_geometry_3d).  One thread per face, then one thread per cell
// (geometry_kernels.cuh); at 10^6 cells the reference spends seconds in NumPy / scipy here, in front of every
// discretization of a new mesh.
//
// Algorithmic traffic: nodes 24 B x (nodes per face) per face + the (3, nf) / (3, nc) outputs; the cell pass re-reads
// the nodes of its faces through L2 (every face is visited by its two cells).  HBM-bound and tiny next to the
// assembly kernels (10^6 tets: ~0.3 GB).
#include "plan.hpp"
#include "geometry_kernels.cuh"

__global__ void geom_face_kernel(int64_t nf, const int32_t *__restrict__ fn_ip, const int32_t *__restrict__ fn_ix,
                                 const double *__restrict__ nodes, GeomOut o) {
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < nf; f += (int64_t)gridDim.x * blockDim.x)
        geom_face(f, fn_ip, fn_ix, nodes, 1, 3, o);
}

__global__ void geom_cell_kernel(int64_t nc, const int32_t *__restrict__ cf_ip, const int32_t *__restrict__ cf_ix,
                                 const int8_t *__restrict__ cf_sg, const int32_t *__restrict__ fn_ip,
                                 const int32_t *__restrict__ fn_ix, const double *__restrict__ nodes, GeomOut o,
                                 int *bad) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += (int64_t)gridDim.x * blockDim.x)
        if (!geom_cell(c, cf_ip, cf_ix, cf_sg, fn_ip, fn_ix, nodes, 1, 3, o)) atomicMin(bad, (int)c);
}

// Host arrays in the reference's layouts: CSC of cell_faces (nf x nc; indices ascending inside a column, data +-1) and
// of face_nodes (nn x nf; the nodes of a face in loop order), nodes (3, nn) row-major; outputs (3, nf) / (nf) /
// (3, nc) / (nc).  kernel_ms (may be NULL): device time of the two kernels.  PB_EINVAL with the cell index in
// pb_last_error_node() when a sub-tetrahedron has negative volume (the reference raises ValueError, grid.py:754).
extern "C" int pb_compute_geometry_3d(int64_t nc, int64_t nf, int64_t nn, const int32_t *cf_indptr,
                                      const int32_t *cf_indices, const int8_t *cf_data, const int32_t *fn_indptr,
                                      const int32_t *fn_indices, const double *nodes, double *face_normals,
                                      double *face_centers, double *face_areas, double *cell_centers,
                                      double *cell_volumes, float *kernel_ms) {
    if (!cf_indptr || !cf_indices || !cf_data || !fn_indptr || !fn_indices || !nodes || !face_normals || !face_centers ||
        !face_areas || !cell_centers || !cell_volumes || nc < 0 || nf < 0 || nn < 0)
        return pb_fail_(PB_EINVAL, "pb_compute_geometry_3d: null pointer or negative size");
    if (int rc = pb_require_device()) return rc;
    Stream st;
    KernelTimer timer;
    CUDA_TRY(st.create());
    CUDA_TRY(timer.create());
    DevBuf d_cf_ip, d_cf_ix, d_cf_sg, d_fn_ip, d_fn_ix, d_nodes, tmp, d_fn, d_fc, d_fa, d_cc, d_cv, d_bad;
    CUDA_TRY(d_cf_ip.upload(cf_indptr, (size_t)nc + 1, st));
    CUDA_TRY(d_cf_ix.upload(cf_indices, (size_t)cf_indptr[nc], st));
    CUDA_TRY(d_cf_sg.upload(cf_data, (size_t)cf_indptr[nc], st));
    CUDA_TRY(d_fn_ip.upload(fn_indptr, (size_t)nf + 1, st));
    CUDA_TRY(d_fn_ix.upload(fn_indices, (size_t)fn_indptr[nf], st));
    if (int rc = pb_upload_repacked_(st, tmp, d_nodes, nodes, 3, nn)) return rc;
    CUDA_TRY(d_fn.ensure((size_t)3 * nf * sizeof(double)));
    CUDA_TRY(d_fc.ensure((size_t)3 * nf * sizeof(double)));
    CUDA_TRY(d_fa.ensure((size_t)nf * sizeof(double)));
    CUDA_TRY(d_cc.ensure((size_t)3 * nc * sizeof(double)));
    CUDA_TRY(d_cv.ensure((size_t)nc * sizeof(double)));
    CUDA_TRY(d_bad.ensure(sizeof(int)));
    int init = INT_MAX;
    CUDA_TRY(cudaMemcpyAsync(d_bad.p, &init, sizeof(int), cudaMemcpyHostToDevice, st));
    // outputs straight in the reference's (3, n) row-major layout: component stride n, entity stride 1
    GeomOut o{d_fn.as<double>(), d_fc.as<double>(), d_fa.as<double>(), d_cc.as<double>(), d_cv.as<double>(), nf, 1, nc, 1};
    CUDA_TRY(timer.mark(0, st));
    geom_face_kernel<<<grid_stride_blocks(nf, 128, 16), 128, 0, st>>>(nf, d_fn_ip.as<int32_t>(), d_fn_ix.as<int32_t>(),
                                                                      d_nodes.as<double>(), o);
    pb_count_launch_();
    geom_cell_kernel<<<grid_stride_blocks(nc, 128, 16), 128, 0, st>>>(
        nc, d_cf_ip.as<int32_t>(), d_cf_ix.as<int32_t>(), d_cf_sg.as<int8_t>(), d_fn_ip.as<int32_t>(),
        d_fn_ix.as<int32_t>(), d_nodes.as<double>(), o, d_bad.as<int>());
    pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(timer.mark(1, st));
    int bad = INT_MAX;
    CUDA_TRY(cudaMemcpyAsync(face_normals, d_fn.p, (size_t)3 * nf * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(face_centers, d_fc.p, (size_t)3 * nf * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(face_areas, d_fa.p, (size_t)nf * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(cell_centers, d_cc.p, (size_t)3 * nc * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(cell_volumes, d_cv.p, (size_t)nc * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&bad, d_bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (kernel_ms) CUDA_TRY(timer.ms(kernel_ms));
    if (bad != INT_MAX) {
        pb_set_error_node_(bad);
        return pb_fail_(PB_EINVAL, "Some tetrahedra have negative volume (cell " + std::to_string(bad) + ")");
    }
    return PB_OK;
}
