// emu_dual.cpp -- TEST INFRASTRUCTURE ONLY: runs the per-(cell, face) routines of the mixed schemes MVEM and RT0
// (porepy_b200/csrc/dual_cell.cuh), which dual.cu's dual_kernel runs one thread per entry of cell_faces, on the host one
// entry after the other, with the mass pattern built by a plain sorted union.  Built by tests/emu_dual.py with g++ into
// tests/emu/_emu_dual.so; the product never builds, links or loads it.
#include <algorithm>
#include <climits>
#include <cstdint>
#include <vector>

#include "../../porepy_b200/csrc/dual_cell.cuh"

using namespace pb;

extern "C" {

// Row f: the sorted union of the faces of f's cells.  indptr / indices may be NULL (size query in *nnz).
int emu_dual_pattern(int64_t nc, int64_t nf, const int32_t *cf_ip, const int32_t *cf_ix, int64_t *nnz, int32_t *ip,
                     int32_t *ix) {
    std::vector<std::vector<int32_t>> rows((size_t)nf);
    for (int64_t c = 0; c < nc; ++c)
        for (int q = cf_ip[c]; q < cf_ip[c + 1]; ++q)
            for (int r = cf_ip[c]; r < cf_ip[c + 1]; ++r) rows[cf_ix[q]].push_back(cf_ix[r]);
    int64_t n = 0;
    for (int64_t f = 0; f < nf; ++f) {
        auto &v = rows[f];
        std::sort(v.begin(), v.end());
        v.erase(std::unique(v.begin(), v.end()), v.end());
        if (ip) ip[f] = (int32_t)n;
        if (ix) std::copy(v.begin(), v.end(), ix + n);
        n += (int64_t)v.size();
    }
    if (ip) ip[nf] = (int32_t)n;
    *nnz = n;
    return 0;
}

// Arrays as pb_dual_discretize (include/poreb200.h); mass zeroed by the caller.  Returns the first cell failing the MVEM
// consistency test, or -1.
int64_t emu_dual_discretize(int nd, int method, int64_t nc, int64_t nf, int64_t nn, const int32_t *cf_ip,
                            const int32_t *cf_ix, const int8_t *cf_sg, const int32_t *fn_ip, const int32_t *fn_ix,
                            const int32_t *mass_ip, const int32_t *mass_ix, const double *nodes, const double *fnorm,
                            const double *fcent, const double *ccent, const double *vol, const double *perm,
                            const double *rot, double *mass, double *proj) {
    std::vector<int32_t> cell((size_t)cf_ip[nc]);
    for (int64_t c = 0; c < nc; ++c)
        for (int q = cf_ip[c]; q < cf_ip[c + 1]; ++q) cell[q] = (int32_t)c;
    const DualTopo T{cf_ip, cf_ix, cell.data(), cf_sg, fn_ip, fn_ix, mass_ip, mass_ix};
    const DualGeo G{nn, nf, nc, nodes, fnorm, fcent, ccent, vol, perm, rot};
    int32_t bad = INT_MAX;
    for (int64_t q = 0; q < cf_ip[nc]; ++q) {
        if (nd == 1) dual_row<1>(method, q, T, G, mass, proj, &bad);
        else if (nd == 2) dual_row<2>(method, q, T, G, mass, proj, &bad);
        else dual_row<3>(method, q, T, G, mass, proj, &bad);
    }
    return bad == INT_MAX ? -1 : bad;
}
}
