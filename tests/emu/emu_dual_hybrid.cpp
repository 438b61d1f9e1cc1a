// emu_dual_hybrid.cpp -- TEST INFRASTRUCTURE ONLY: runs the lane routines of the hybridization of MVEM and RT0
// (porepy_b200/csrc/dual_hybrid.cuh), which dual.cu's hybrid_cell_kernel runs one warp per cell with lane i on local
// face i, on the host one lane after the other, and the boundary rows of hybrid_bc_kernel one face after the other.
// Built by tests/emu_dual_hybrid.py with g++ into tests/emu/_emu_dual_hybrid.so; the product never builds, links or
// loads it.
#include <climits>
#include <cmath>
#include <cstdint>
#include <vector>

#include "../../porepy_b200/csrc/dual_hybrid.cuh"

using namespace pb;

extern "C" {

// ---- hybridization (porepy_b200/csrc/dual_hybrid.cuh), the lanes of one cell one after the other ----
// Arrays as pb_dual_hybrid_system / pb_dual_hybrid_recover (include/poreb200.h), with the topology and mass pattern
// passed in.  lam == NULL: the face matrix (hval, zeroed by the caller, in the mass pattern) and rhs (zeroed), with
// mass_norm = |mass|_inf for the saddle mode; else [u; p] into up.  Returns the first cell failing the MVEM
// consistency test, -1, or -2 - c for a singular local matrix of cell c.
int64_t emu_dual_hybrid(int nd, int method, int mode, int64_t nc, int64_t nf, int64_t nn, const int32_t *cf_ip,
                        const int32_t *cf_ix, const int8_t *cf_sg, const int32_t *fn_ip, const int32_t *fn_ix,
                        const int32_t *mass_ip, const int32_t *mass_ix, const double *nodes, const double *fnorm,
                        const double *fcent, const double *ccent, const double *vol, const double *perm,
                        const double *rot, const double *aperture, const uint8_t *codes, const double *robin_weight,
                        const double *face_areas, const double *values, double mass_norm, const double *lam,
                        double *hval, double *rhs, double *up) {
    const int64_t ncf = cf_ip[nc];
    std::vector<int32_t> cell((size_t)ncf), fc_ip((size_t)nf + 1, 0), fc_cell((size_t)ncf);
    for (int64_t c = 0; c < nc; ++c)
        for (int q = cf_ip[c]; q < cf_ip[c + 1]; ++q) {
            cell[q] = (int32_t)c;
            ++fc_ip[cf_ix[q] + 1];
        }
    for (int64_t f = 0; f < nf; ++f) fc_ip[f + 1] += fc_ip[f];
    {
        std::vector<int32_t> next(fc_ip.begin(), fc_ip.end() - 1);
        for (int64_t q = 0; q < ncf; ++q) fc_cell[next[cf_ix[q]]++] = cell[q];
    }
    const DualTopo T{cf_ip, cf_ix, cell.data(), cf_sg, fn_ip, fn_ix, mass_ip, mass_ix};
    const DualGeo G{nn, nf, nc, nodes, fnorm, fcent, ccent, vol, perm, rot};
    const HybridIn H{mode, nf, fc_ip.data(), fc_cell.data(), mode == PB_DUAL_HYBRID_VEM ? aperture : nullptr, values,
                     codes};
    int32_t bad = INT_MAX;
    std::vector<double> A, E, z, r, lv;
    for (int64_t c = 0; c < nc; ++c) {
        const int n = cf_ip[c + 1] - cf_ip[c];
        A.assign((size_t)n * n, 0.0); E.assign((size_t)n * n, 0.0);
        z.assign(n, 0.0); r.assign(n, 0.0); lv.assign(n, 0.0);
        for (int i = 0; i < n; ++i) {
            if (nd == 1) hybrid_local_row<1>(method, c, i, T, G, H, A.data(), &bad);
            else if (nd == 2) hybrid_local_row<2>(method, c, i, T, G, H, A.data(), &bad);
            else hybrid_local_row<3>(method, c, i, T, G, H, A.data(), &bad);
        }
        if (group_invert_serial(A.data(), E.data(), n) >= 0) return -2 - c;
        for (int i = 0; i < n; ++i) hybrid_vectors(c, i, T, H, E.data(), lam, z.data(), r.data(), lv.data());
        for (int i = 0; i < n; ++i) {
            if (lam) hybrid_recover_row(c, i, T, H, E.data(), z.data(), r.data(), lv.data(), up, up + nf);
            else hybrid_condense_row(c, i, T, H, E.data(), z.data(), r.data(), hval, rhs);
        }
    }
    if (!lam) {
        double norm = mass_norm;
        if (mode == PB_DUAL_HYBRID_VEM) {
            norm = 0.0;
            for (int64_t f = 0; f < nf; ++f) {
                double s = 0.0;
                for (int32_t q = mass_ip[f]; q < mass_ip[f + 1]; ++q) s += std::fabs(hval[q]);
                norm = s > norm ? s : norm;
            }
        }
        for (int64_t f = 0; f < nf; ++f) hybrid_bc_row((int32_t)f, T, H, robin_weight, face_areas, norm, hval, rhs);
    }
    return bad == INT_MAX ? -1 : bad;
}
}
