// plan_device.cu -- the sub-cell topology plan built ON THE DEVICE.
//
// Same output as plan_host.hpp::build_host_plan (which stays as the fallback for interaction regions too large for
// the per-node shared-memory sort, and as the host build of the test harness): what the reference derives with
// np.lexsort + sparse products in SubcellTopology.__init__ (numerics/fv/_fvutils.py:51-172).  A counting sort of the
// (cell, face, node) incidences by node:
//   1. count the incidences ("sub-half-faces") and the sub-faces of every node          (atomics, one thread per cell-face)
//   2. exclusive scans -> node offsets
//   3. scatter the incidences into their node's bucket                                   (order inside a bucket arbitrary)
//   4. one warp per node: sort the bucket by (cell, face) in shared memory, number the sub-cells and the sub-faces,
//      pair the two sides of every sub-face, number the boundary sub-faces
//   5. nodes per cell, cell -> node lists, boundary faces per node, face -> cell table
// Only three per-node integer arrays (sub-cell / sub-face / boundary counts) return to the host, where the solver
// classes and the position-map offsets are derived from them.
#include "csr_build.cuh"

struct HalfFace { int32_t c, f, u, sg; };

__global__ void pd_count_kernel(int64_t nc, const int32_t *__restrict__ cf_ip, const int32_t *__restrict__ cf_ix,
                                const int32_t *__restrict__ fn_ip, const int32_t *__restrict__ fn_ix,
                                int32_t *__restrict__ hcount, int32_t *__restrict__ ncn_x_nd) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += (int64_t)gridDim.x * blockDim.x) {
        int tot = 0;
        for (int i = cf_ip[c]; i < cf_ip[c + 1]; ++i) {
            const int f = cf_ix[i];
            for (int q = fn_ip[f]; q < fn_ip[f + 1]; ++q) { atomicAdd(hcount + fn_ix[q], 1); ++tot; }
        }
        ncn_x_nd[c] = tot;   // = nd * (nodes of the cell)
    }
}

__global__ void pd_count_sf_kernel(int64_t U, const int32_t *__restrict__ fn_ix, int32_t *__restrict__ sfcount) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < U; q += (int64_t)gridDim.x * blockDim.x)
        atomicAdd(sfcount + fn_ix[q], 1);
}

__global__ void pd_scatter_kernel(int64_t nc, const int32_t *__restrict__ cf_ip, const int32_t *__restrict__ cf_ix,
                                  const int8_t *__restrict__ cf_da, const int32_t *__restrict__ fn_ip,
                                  const int32_t *__restrict__ fn_ix, const int32_t *__restrict__ hptr_nd /* sc_ptr */,
                                  int nd, int32_t *__restrict__ fill, HalfFace *__restrict__ hf) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += (int64_t)gridDim.x * blockDim.x)
        for (int i = cf_ip[c]; i < cf_ip[c + 1]; ++i) {
            const int f = cf_ix[i];
            const int sg = cf_da[i];
            for (int q = fn_ip[f]; q < fn_ip[f + 1]; ++q) {
                const int s = fn_ix[q];
                const int pos = atomicAdd(fill + s, 1);
                hf[(int64_t)hptr_nd[s] * nd + pos] = HalfFace{(int32_t)c, f, q, sg};
            }
        }
}

// one warp per node; shared memory per warp: CAP x {64-bit key (cell << 32 | face), payload (u << 1 | sign<0), sorted
// u's, min side, max side, side count}
template <int CAP>
__global__ void pd_node_kernel(int64_t nn, int nd, int64_t nf, const HalfFace *__restrict__ hf,
                               const int32_t *__restrict__ sc_ptr, const int32_t *__restrict__ sf_ptr,
                               const int32_t *__restrict__ fn_ip, int32_t *__restrict__ sc_cell,
                               uint16_t *__restrict__ slot_sf, int32_t *__restrict__ sf_face,
                               uint32_t *__restrict__ sf_sides, uint16_t *__restrict__ sf_bloc,
                               int32_t *__restrict__ node_nb, int *bad, int *maxima) {
    extern __shared__ unsigned char pd_smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    unsigned long long *key = (unsigned long long *)pd_smem + (size_t)wib * CAP;
    int32_t *i32 = (int32_t *)((unsigned long long *)pd_smem + (size_t)wpb * CAP);
    int32_t *pay = i32 + ((size_t)0 * wpb + wib) * CAP;
    int32_t *us = i32 + ((size_t)1 * wpb + wib) * CAP;
    int32_t *smin = i32 + ((size_t)2 * wpb + wib) * CAP;
    int32_t *smax = i32 + ((size_t)3 * wpb + wib) * CAP;
    int32_t *scnt = i32 + ((size_t)4 * wpb + wib) * CAP;
    int mx_sf = 0, mx_sc = 0, mx_nb = 0;
    for (int64_t s = (int64_t)blockIdx.x * wpb + wib; s < nn; s += (int64_t)gridDim.x * wpb) {
        const int nsc = sc_ptr[s + 1] - sc_ptr[s];
        const int nh = nsc * nd;
        const int nsf = sf_ptr[s + 1] - sf_ptr[s];
        const int64_t b = (int64_t)sc_ptr[s] * nd;
        const int64_t sc_fill = sc_ptr[s], sf_fill = sf_ptr[s];
        if (nh == 0) {
            if (lane == 0) { node_nb[s] = 0; if (nsf) atomicOr(bad, 4); }
            continue;
        }
        if (nh > CAP || nsf > CAP) { if (lane == 0) atomicOr(bad, 64); continue; }   // -> host fallback
        int P = 1;
        while (P < nh) P <<= 1;
        for (int i = lane; i < P; i += 32) {
            if (i < nh) {
                const HalfFace h = hf[b + i];
                key[i] = ((unsigned long long)(unsigned)h.c << 32) | (unsigned)h.f;
                pay[i] = (h.u << 1) | (h.sg < 0 ? 1 : 0);
                us[i] = h.u;
            } else { key[i] = ~0ull; pay[i] = 0; us[i] = 0x7fffffff; }
        }
        __syncwarp();
        // bitonic sorts in one network: (key, pay) by (cell, face); us by u
        warp_bitonic_sort(P, [&](int i, int l, bool asc) {
            if (warp_cas(key, i, l, asc)) { const int t = pay[i]; pay[i] = pay[l]; pay[l] = t; }
            warp_cas(us, i, l, asc);
        });
        // unique sub-faces: in-place compaction of the sorted u's
        const int cnt = warp_unique(us, nh, us);
        if (cnt != nsf) { if (lane == 0) atomicOr(bad, 4); continue; }
        for (int i = lane; i < nsf; i += 32) { smin[i] = 0x7fffffff; smax[i] = -1; scnt[i] = 0; }
        __syncwarp();
        // sub-cells: groups of nd consecutive entries share the cell and consecutive groups differ; slots and sides
        int lbad = 0;
        for (int j = lane; j < nh; j += 32) {
            const int k = j / nd, m = j - k * nd;
            const unsigned cell = (unsigned)(key[j] >> 32);
            if ((unsigned)(key[k * nd] >> 32) != cell) lbad |= 3;
            if (m == 0) {
                if (k > 0 && (unsigned)(key[(k - 1) * nd] >> 32) == cell) lbad |= 3;
                sc_cell[sc_fill + k] = (int32_t)cell;
            }
            const int u = pay[j] >> 1;
            int lo = 0, hi = nsf;
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (us[mid] < u) lo = mid + 1; else hi = mid; }
            slot_sf[(sc_fill + k) * nd + m] = (uint16_t)((lo << 1) | (pay[j] & 1));
            atomicMin(&smin[lo], j);   // side = k*nd + m = j: the smaller cell index is side 1 (_fvutils.py:163)
            atomicMax(&smax[lo], j);
            atomicAdd(&scnt[lo], 1);
        }
        __syncwarp();
        // faces of the sub-faces, the pair of sides, boundary numbering (sub-faces with one side)
        int nb = 0;
        for (int i0 = 0; i0 < nsf; i0 += 32) {
            const int i = i0 + lane;
            bool bnd = false;
            if (i < nsf) {
                const int u = us[i];
                int64_t lo = 0, hi = nf - 1;          // largest f with fn_ip[f] <= u
                while (lo < hi) { const int64_t mid = (lo + hi + 1) >> 1; if (fn_ip[mid] <= u) lo = mid; else hi = mid - 1; }
                sf_face[sf_fill + i] = (int32_t)lo;
                const int c = scnt[i];
                if (c < 1 || c > 2) lbad |= 16;
                bnd = c == 1;
                sf_sides[sf_fill + i] = (uint32_t)smin[i] | (bnd ? 0xFFFF0000u : ((uint32_t)smax[i] << 16));
            }
            const unsigned m = __ballot_sync(0xffffffffu, bnd);
            if (i < nsf) sf_bloc[sf_fill + i] = bnd ? (uint16_t)(nb + __popc(m & ((1u << lane) - 1u))) : (uint16_t)0xFFFF;
            nb += __popc(m);
        }
        for (int o = 16; o > 0; o >>= 1) lbad |= __shfl_xor_sync(0xffffffffu, lbad, o);
        if (lbad) { if (lane == 0) atomicOr(bad, lbad); continue; }
        if (lane == 0) node_nb[s] = nb;
        mx_sf = max(mx_sf, nsf); mx_sc = max(mx_sc, nsc); mx_nb = max(mx_nb, nb);
        __syncwarp();
    }
    if (lane == 0) { atomicMax(maxima, mx_sf); atomicMax(maxima + 1, mx_sc); atomicMax(maxima + 2, mx_nb); }
}

// out = in / nd (in place allowed); with `bad`, flags 3 where nd does not divide the count
__global__ void pd_div_kernel(int64_t n, int nd, const int32_t *in, int32_t *out, int *bad) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        if (bad && in[i] % nd) atomicExch(bad, 3);
        out[i] = in[i] / nd;
    }
}

// cell -> nodes (order inside a cell arbitrary) and boundary faces of every node (local boundary order)
__global__ void pd_adjacency_kernel(int64_t nn, const int32_t *__restrict__ sc_ptr, const int32_t *__restrict__ sc_cell,
                                    const int32_t *__restrict__ cn_ptr, int32_t *__restrict__ cfill,
                                    int32_t *__restrict__ cn_idx, const int32_t *__restrict__ sf_ptr,
                                    const int32_t *__restrict__ sf_face, const uint16_t *__restrict__ sf_bloc,
                                    const int32_t *__restrict__ nbf_ptr, int32_t *__restrict__ nbf_idx) {
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < nn; s += (int64_t)gridDim.x * blockDim.x) {
        for (int q = sc_ptr[s]; q < sc_ptr[s + 1]; ++q) {
            const int c = sc_cell[q];
            cn_idx[cn_ptr[c] + atomicAdd(cfill + c, 1)] = (int32_t)s;
        }
        for (int q = sf_ptr[s]; q < sf_ptr[s + 1]; ++q)
            if (sf_bloc[q] != 0xFFFF) nbf_idx[nbf_ptr[s] + sf_bloc[q]] = sf_face[q];
    }
}

__global__ void pd_face_cells_kernel(int64_t nc, const int32_t *__restrict__ cf_ip, const int32_t *__restrict__ cf_ix,
                                     const int8_t *__restrict__ cf_da, int32_t *__restrict__ fc, int *bad) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += (int64_t)gridDim.x * blockDim.x)
        for (int q = cf_ip[c]; q < cf_ip[c + 1]; ++q) {
            const int32_t f = cf_ix[q];
            const int32_t enc = (int32_t)((c << 1) | (cf_da[q] < 0 ? 1 : 0));
            if (atomicCAS(fc + 2 * (int64_t)f, -1, enc) != -1)
                if (atomicCAS(fc + 2 * (int64_t)f + 1, -1, enc) != -1) atomicExch(bad, 16);
        }
}
__global__ void pd_face_cells_order_kernel(int64_t nf, int32_t *__restrict__ fc) {
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < nf; f += (int64_t)gridDim.x * blockDim.x) {
        const int32_t a = fc[2 * f], b = fc[2 * f + 1];
        if (b >= 0 && b < a) { fc[2 * f] = b; fc[2 * f + 1] = a; }
    }
}

// Returns PB_OK, an error code (pb_fail_), or -1 when the per-node sort capacity was exceeded (caller falls back to
// the host plan).  On success the plan's topology DevBufs are filled and H holds the sizes and the three per-node arrays.
int pb_build_device_topology_(pb_plan *p, int nd, int64_t nc, int64_t nf, int64_t nn, const int32_t *cf_indptr,
                              const int32_t *cf_indices, const int8_t *cf_data, const int32_t *fn_indptr,
                              const int32_t *fn_indices, DevBuf &fn_idx_dev) {
    HostPlan &H = p->H;
    cudaStream_t st = p->stream;
    if (nd != 2 && nd != 3) return pb_fail_(PB_EINVAL, "nd must be 2 or 3");
    if (nc <= 0 || nf <= 0 || nn <= 0) return pb_fail_(PB_EINVAL, "empty grid");
    const int64_t U = fn_indptr[nf], CF = cf_indptr[nc];
    H.nd = nd; H.nc = nc; H.nf = nf; H.nn = nn; H.U = U;
    // cheap host validation of the index ranges (one pass over the inputs; also needed before trusting them on the device)
    for (int64_t q = 0; q < CF; ++q) {
        if (cf_indices[q] < 0 || cf_indices[q] >= nf) return pb_fail_(PB_EINVAL, "cell_faces index out of range");
        if (cf_data[q] != 1 && cf_data[q] != -1) return pb_fail_(PB_EINVAL, "cell_faces data must be +-1");
    }
    for (int64_t q = 0; q < U; ++q)
        if (fn_indices[q] < 0 || fn_indices[q] >= nn) return pb_fail_(PB_EINVAL, "face_nodes index out of range");
    DevBuf cf_ip, cf_ix, cf_da, hcount, sfcount, ncnx, fill, hfbuf, flags, cfill;
    CUDA_TRY(cf_ip.upload(cf_indptr, (size_t)nc + 1, st));
    CUDA_TRY(cf_ix.upload(cf_indices, (size_t)CF, st));
    CUDA_TRY(cf_da.upload(cf_data, (size_t)CF, st));
    CUDA_TRY(p->fn_indptr.upload(fn_indptr, (size_t)nf + 1, st));
    CUDA_TRY(fn_idx_dev.upload(fn_indices, (size_t)U, st));
    CUDA_TRY(hcount.ensure((size_t)(nn + 1) * 4));
    CUDA_TRY(sfcount.ensure((size_t)(nn + 1) * 4));
    CUDA_TRY(fill.ensure((size_t)(nn + 1) * 4));
    CUDA_TRY(ncnx.ensure((size_t)nc * 4));
    CUDA_TRY(flags.ensure(8 * sizeof(int)));
    CUDA_TRY(cudaMemsetAsync(hcount.p, 0, (size_t)(nn + 1) * 4, st));
    CUDA_TRY(cudaMemsetAsync(sfcount.p, 0, (size_t)(nn + 1) * 4, st));
    CUDA_TRY(cudaMemsetAsync(fill.p, 0, (size_t)(nn + 1) * 4, st));
    CUDA_TRY(cudaMemsetAsync(flags.p, 0, 8 * sizeof(int), st));
    const int block = 256;   // one thread per cell (gc), node (gn), face (gf) or sub-face (gu)
    const int gc = grid_stride_blocks(nc, block, 16), gn = grid_stride_blocks(nn, block, 16),
              gf = grid_stride_blocks(nf, block, 16), gu = grid_stride_blocks(U, block, 16);
    pd_count_kernel<<<gc, block, 0, st>>>(nc, cf_ip.as<int32_t>(), cf_ix.as<int32_t>(), p->fn_indptr.as<int32_t>(),
                                          fn_idx_dev.as<int32_t>(), hcount.as<int32_t>(), ncnx.as<int32_t>());
    pd_count_sf_kernel<<<gu, block, 0, st>>>(U, fn_idx_dev.as<int32_t>(), sfcount.as<int32_t>());
    // sub-cells per node = half-faces per node / nd
    pd_div_kernel<<<gn, block, 0, st>>>(nn, nd, hcount.as<int32_t>(), hcount.as<int32_t>(), flags.as<int>());
    CUDA_TRY(p->node_sc_ptr.ensure((size_t)(nn + 1) * 4));
    CUDA_TRY(p->node_sf_ptr.ensure((size_t)(nn + 1) * 4));
    int64_t S = 0, sf_total = 0;
    int rc = pb_scan_offsets_(hcount.as<int32_t>(), p->node_sc_ptr.as<int32_t>(), nn, st, &S);
    if (rc) return rc;
    rc = pb_scan_offsets_(sfcount.as<int32_t>(), p->node_sf_ptr.as<int32_t>(), nn, st, &sf_total);
    if (rc) return rc;
    H.node_sc_ptr.resize(nn + 1);
    H.node_sf_ptr.resize(nn + 1);
    CUDA_TRY(cudaMemcpyAsync(H.node_sc_ptr.data(), p->node_sc_ptr.p, (size_t)(nn + 1) * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(H.node_sf_ptr.data(), p->node_sf_ptr.p, (size_t)(nn + 1) * 4, cudaMemcpyDeviceToHost, st));
    int hflags[8];
    CUDA_TRY(cudaMemcpyAsync(hflags, flags.p, sizeof(hflags), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (S > 0x7fffffffll || sf_total > 0x7fffffffll)
        return pb_fail_(PB_EINVAL, "grid too large for 32-bit sub-cell indices; split the grid");
    if (hflags[0] == 3) return pb_fail_(PB_ECELLTYPE, "cells must have exactly nd faces meeting in each vertex");
    const int64_t Hh = S * nd;
    H.S = S; H.H = Hh;
    if (sf_total != U) return pb_fail_(PB_EINVAL, "internal: sub-face count");
    CUDA_TRY(hfbuf.ensure((size_t)std::max<int64_t>(1, Hh) * sizeof(HalfFace)));
    pd_scatter_kernel<<<gc, block, 0, st>>>(nc, cf_ip.as<int32_t>(), cf_ix.as<int32_t>(), cf_da.as<int8_t>(),
                                            p->fn_indptr.as<int32_t>(), fn_idx_dev.as<int32_t>(),
                                            p->node_sc_ptr.as<int32_t>(), nd, fill.as<int32_t>(), hfbuf.as<HalfFace>());
    CUDA_TRY(p->sc_cell.ensure((size_t)std::max<int64_t>(1, S) * 4));
    CUDA_TRY(p->slot_sf.ensure((size_t)std::max<int64_t>(1, Hh) * 2));
    CUDA_TRY(p->sf_face.ensure((size_t)std::max<int64_t>(1, U) * 4));
    CUDA_TRY(p->sf_sides.ensure((size_t)std::max<int64_t>(1, U) * 4));
    CUDA_TRY(p->sf_bloc.ensure((size_t)std::max<int64_t>(1, U) * 2));
    CUDA_TRY(p->node_nb.ensure((size_t)(nn + 1) * 4));
    constexpr int CAP = 1024, WPB = 4;
    const size_t smem = (size_t)WPB * CAP * (8 + 5 * 4);
    CUDA_TRY(cudaFuncSetAttribute(pd_node_kernel<CAP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int gridn = grid_stride_blocks(nn, WPB, 2);
    pd_node_kernel<CAP><<<gridn, WPB * 32, smem, st>>>(nn, nd, nf, hfbuf.as<HalfFace>(), p->node_sc_ptr.as<int32_t>(),
                                                       p->node_sf_ptr.as<int32_t>(), p->fn_indptr.as<int32_t>(),
                                                       p->sc_cell.as<int32_t>(), p->slot_sf.as<uint16_t>(),
                                                       p->sf_face.as<int32_t>(), p->sf_sides.as<uint32_t>(),
                                                       p->sf_bloc.as<uint16_t>(), p->node_nb.as<int32_t>(),
                                                       flags.as<int>() + 1, flags.as<int>() + 4);
    // nodes per cell, cell -> nodes, boundary faces per node, face -> cells
    CUDA_TRY(p->sc_ncn.ensure((size_t)nc * 4));
    pd_div_kernel<<<gc, block, 0, st>>>(nc, nd, ncnx.as<int32_t>(), p->sc_ncn.as<int32_t>(), nullptr);
    CUDA_TRY(p->cn_ptr.ensure((size_t)(nc + 1) * 4));
    CUDA_TRY(p->nbf_ptr.ensure((size_t)(nn + 1) * 4));
    int64_t cn_total = 0, nbf_total = 0;
    rc = pb_scan_offsets_(p->sc_ncn.as<int32_t>(), p->cn_ptr.as<int32_t>(), nc, st, &cn_total);
    if (rc) return rc;
    rc = pb_scan_offsets_(p->node_nb.as<int32_t>(), p->nbf_ptr.as<int32_t>(), nn, st, &nbf_total);
    if (rc) return rc;
    H.node_nb.resize(nn);
    CUDA_TRY(cudaMemcpyAsync(H.node_nb.data(), p->node_nb.p, (size_t)nn * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(hflags, flags.p, sizeof(hflags), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (hflags[1] & 64) return -1;   // an interaction region exceeds the shared-memory sort: host plan
    if (hflags[1] & 3) return pb_fail_(PB_ECELLTYPE, "cells must have exactly nd faces meeting in each vertex");
    if (hflags[1] & 4) return pb_fail_(PB_EINVAL, "face_nodes holds nodes without neighbouring cells");
    if (hflags[1] & 16) return pb_fail_(PB_EINVAL, "face with more than two neighbouring cells");
    if (hflags[1]) return pb_fail_(PB_EINVAL, "internal: topology plan");
    H.max_nsf = hflags[4]; H.max_nsc = hflags[5]; H.max_nb = hflags[6];
    if (H.max_nsf > 32767 || H.max_nsc > 21000) return pb_fail_(PB_EINVAL, "interaction region too large");
    CUDA_TRY(cfill.ensure((size_t)nc * 4));
    CUDA_TRY(cudaMemsetAsync(cfill.p, 0, (size_t)nc * 4, st));
    CUDA_TRY(p->cn_idx.ensure((size_t)std::max<int64_t>(1, S) * 4));
    CUDA_TRY(p->nbf_idx.ensure((size_t)std::max<int64_t>(1, nbf_total) * 4));
    pd_adjacency_kernel<<<gn, block, 0, st>>>(nn, p->node_sc_ptr.as<int32_t>(), p->sc_cell.as<int32_t>(),
                                              p->cn_ptr.as<int32_t>(), cfill.as<int32_t>(), p->cn_idx.as<int32_t>(),
                                              p->node_sf_ptr.as<int32_t>(), p->sf_face.as<int32_t>(),
                                              p->sf_bloc.as<uint16_t>(), p->nbf_ptr.as<int32_t>(),
                                              p->nbf_idx.as<int32_t>());
    CUDA_TRY(p->face_cells.ensure((size_t)2 * nf * 4));
    CUDA_TRY(cudaMemsetAsync(p->face_cells.p, 0xFF, (size_t)2 * nf * 4, st));
    pd_face_cells_kernel<<<gc, block, 0, st>>>(nc, cf_ip.as<int32_t>(), cf_ix.as<int32_t>(), cf_da.as<int8_t>(),
                                               p->face_cells.as<int32_t>(), flags.as<int>() + 2);
    pd_face_cells_order_kernel<<<gf, block, 0, st>>>(nf, p->face_cells.as<int32_t>());
    for (int i = 0; i < 9; ++i) pb_count_launch_();
    CUDA_TRY(cudaGetLastError());
    // position-map offsets on the host from the three per-node arrays
    H.posfc_ptr.assign(nn + 1, 0); H.posfb_ptr.assign(nn + 1, 0);
    H.poscc_ptr.assign(nn + 1, 0); H.poscb_ptr.assign(nn + 1, 0);
    for (int64_t s = 0; s < nn; ++s) {
        const int64_t nsc = H.node_sc_ptr[s + 1] - H.node_sc_ptr[s];
        const int64_t nsf = H.node_sf_ptr[s + 1] - H.node_sf_ptr[s];
        const int64_t nb = H.node_nb[s];
        H.posfc_ptr[s + 1] = H.posfc_ptr[s] + nsf * nsc;
        H.posfb_ptr[s + 1] = H.posfb_ptr[s] + nsf * nb;
        H.poscc_ptr[s + 1] = H.poscc_ptr[s] + nsc * nsc;
        H.poscb_ptr[s + 1] = H.poscb_ptr[s] + nsc * nb;
    }
    CUDA_TRY(p->posfc_ptr.upload(H.posfc_ptr, st));
    CUDA_TRY(p->posfb_ptr.upload(H.posfb_ptr, st));
    CUDA_TRY(p->poscc_ptr.upload(H.poscc_ptr, st));
    CUDA_TRY(p->poscb_ptr.upload(H.poscb_ptr, st));
    CUDA_TRY(cudaMemcpyAsync(hflags, flags.p, sizeof(hflags), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (hflags[2]) return pb_fail_(PB_EINVAL, "face with more than two neighbouring cells");
    p->cf_ip = std::move(cf_ip);
    p->cf_ix = std::move(cf_ix);
    p->cf_sg = std::move(cf_da);
    return PB_OK;
}
