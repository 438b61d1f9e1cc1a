// emu_tpsa_thm.cpp -- TEST INFRASTRUCTURE ONLY: the host build of the TPSA thermo-poromechanics system
// (porepy_b200/csrc/tpsa_system.cuh with NS = 2 scalar balances, run on the device by face.cu's pb_tpsa_thm_system /
// pb_tpsa_thm_rhs / pb_tpsa_thm_balance_rows): the per-face routine of tpsa_face.cuh over all faces, the row pattern, the
// mechanics blocks, the right-hand side and the mass and energy rows, one loop step where the device runs one thread,
// so the arithmetic and the layout can be checked on a box without a GPU.  Built by tests/emu_tpsa_thm.py with g++ into
// tests/emu/_emu_tpsa_thm.so; the product never builds, links or loads it.
#include <cstdint>
#include <vector>

#include "../../porepy_b200/csrc/tpsa_face.cuh"
#include "../../porepy_b200/csrc/tpsa_system.cuh"

using namespace pb;

namespace {
struct System {
    int64_t nrows = 0;
    std::vector<int32_t> ip, ix;
    std::vector<double> a, b;
};

// The five-field system: mechanics rows and pattern as pb_tpsa_thm_system, b0 as pb_tpsa_thm_rhs.
template <int ND, int NS>
int assemble_poro(System &S, int64_t nc, int64_t nf, const int32_t *cf_ip, const int32_t *cf_ix, const int32_t *fc,
                  const GeoView &G, const double *mu, const double *lam, const double *alpha, const double *vol,
                  const uint8_t *codes, const double *robw, const uint8_t *flags, const int32_t *fp_ip,
                  const int32_t *fp_ix, const double *g, const double *f, const double *sr, const double *sp) {
    using D = TpsaPoroDims<ND, NS>;
    constexpr int NR = D::NR, B = D::B;
    std::vector<int32_t> fc_ptr(nf + 1, 0);
    for (int64_t k = 0; k < nf; ++k) fc_ptr[k + 1] = fc_ptr[k] + (fc[2 * k] >= 0) + (fc[2 * k + 1] >= 0);
    const size_t nfc = fc_ptr[nf];
    const size_t per[14] = {ND, ND * NR, ND, NR * ND, NR * NR, ND, 1, ND, ND * NR, ND, ND, NR * ND, ND, ND};
    std::vector<std::vector<double>> buf(14);
    TpsaOut o{};
    TpsaTerms T{};
    for (int k = 0; k < 14; ++k) {
        buf[k].assign(per[k] * (k < 10 ? nfc : (size_t)nf), 0.0);
        o.t[k] = buf[k].data();
        T.t[k] = buf[k].data();
    }
    for (int64_t k = 0; k < nf; ++k) tpsa_face<ND>(k, G, mu, codes, robw, flags, fc, fc_ptr.data(), o);
    const TpsaTopo t{nc, cf_ip, cf_ix, fc, fc_ptr.data()};
    std::vector<int32_t> cc_ptr(nc + 1, 0), nb(kTpsaMaxNb);
    for (int64_t c = 0; c < nc; ++c) {
        const int n = tpsa_cell_neighbours(c, t, nb.data());
        if (n < 0) return 2;
        cc_ptr[c + 1] = cc_ptr[c] + n;
    }
    std::vector<int32_t> cc_ix(cc_ptr[nc]);
    std::vector<int64_t> blk_ptr(nc + 1, 0);
    for (int64_t c = 0; c < nc; ++c)
        blk_ptr[c + 1] = blk_ptr[c] + tpsa_poro_row_count<ND, NS>(c, cc_ptr[c + 1] - cc_ptr[c], fp_ip, fp_ix);
    S.nrows = nc * B;
    S.ip.assign(S.nrows + 1, 0);
    S.ix.assign((size_t)blk_ptr[nc], 0);
    S.a.assign(S.ix.size(), 0.0);
    S.b.assign(S.nrows, 0.0);
    for (int64_t c = 0; c < nc; ++c) {
        const int n = tpsa_cell_neighbours(c, t, nb.data());
        for (int j = 0; j < n; ++j) cc_ix[cc_ptr[c] + j] = nb[j];
        tpsa_poro_pattern_rows<ND, NS>(c, n, nb.data(), blk_ptr[c], fp_ip, fp_ix, S.ip.data(), S.ix.data());
    }
    S.ip[S.nrows] = (int32_t)S.ix.size();
    for (int64_t c = 0; c < nc; ++c)
        for (int j = 0; j < cc_ptr[c + 1] - cc_ptr[c]; ++j)
            tpsa_poro_block<ND, NS>(c, j, t, cc_ptr.data(), cc_ix.data(), blk_ptr.data(), T, mu, lam, alpha, vol,
                                S.a.data());
    for (int64_t c = 0; c < nc; ++c)
        for (int l = 0; l < B - NS; ++l) {
            const double src = l < ND ? (f ? f[c * ND + l] : 0.0)
                                       : (l < ND + NR ? (sr ? sr[c * NR + l - ND] : 0.0) : (sp ? sp[c] : 0.0));
            S.b[c * B + l] = tpsa_rhs_row<ND>(c, l, t, T, g, src);
        }
    return 0;
}

template <int ND, int NS>
int balance_rows(int64_t nc, const int32_t *ip, const int32_t *ix, const int32_t *jf_ip, const int32_t *jf_ix,
               const double *jf_a, const double *neg_res, double *a, double *b) {
    constexpr int B = TpsaPoroDims<ND, NS>::B;
    std::vector<int64_t> blk_ptr(nc + 1);
    for (int64_t c = 0; c <= nc; ++c) blk_ptr[c] = ip[c * B];
    int missing = 0;
    for (int64_t c = 0; c < nc; ++c)
        missing += tpsa_poro_fluid_row<ND, NS>(c, nc, blk_ptr.data(), ip[c * B + B - NS], ix, jf_ip, jf_ix, jf_a,
                                               neg_res, a, b);
    return missing;
}

int face_cells(int64_t nc, int64_t nf, const int32_t *cf_ip, const int32_t *cf_ix, const int8_t *cf_da,
               std::vector<int32_t> &fc) {
    fc.assign(2 * nf, -1);
    for (int64_t c = 0; c < nc; ++c)
        for (int q = cf_ip[c]; q < cf_ip[c + 1]; ++q) {
            const int32_t k = cf_ix[q];
            const int32_t enc = (int32_t)((c << 1) | (cf_da[q] < 0 ? 1 : 0));
            if (fc[2 * k] < 0) fc[2 * k] = enc;
            else if (fc[2 * k + 1] < 0) fc[2 * k + 1] = enc;
            else return 1;   // a face with more than two cells
        }
    return 0;
}
}  // namespace

extern "C" {

// The thermo-poromechanics system of pb_tpsa_thm_system (mechanics rows, mass and energy rows 0) and b0 of
// pb_tpsa_thm_rhs; fp_ip / fp_ix: the sorted CSR pattern of the Darcy and Fourier div @ flux.  *out: a handle for
// emu_tpsa_thm_get.
int emu_tpsa_thm_system(int64_t nc, int64_t nf, const int32_t *cf_ip, const int32_t *cf_ix, const int8_t *cf_da,
                         const double *fnorm, const double *fcent, const double *farea, const double *ccent, int nd,
                         const double *mu, const double *lam, const double *alpha, const double *vol,
                         const uint8_t *codes, const double *robw, const uint8_t *flags, const int32_t *fp_ip,
                         const int32_t *fp_ix, const double *g, const double *f, const double *sr, const double *sp,
                         void **out, int64_t *nrows, int64_t *nnz) {
    std::vector<int32_t> fc;
    if (face_cells(nc, nf, cf_ip, cf_ix, cf_da, fc)) return 1;
    GeoView G{nullptr, fnorm, fcent, farea, ccent, nullptr, 0, 1, nf, 1, nc, 1};
    System *S = new System;
    const int rc = nd == 3 ? assemble_poro<3, 2>(*S, nc, nf, cf_ip, cf_ix, fc.data(), G, mu, lam, alpha, vol, codes, robw,
                                              flags, fp_ip, fp_ix, g, f, sr, sp)
                           : assemble_poro<2, 2>(*S, nc, nf, cf_ip, cf_ix, fc.data(), G, mu, lam, alpha, vol, codes, robw,
                                              flags, fp_ip, fp_ix, g, f, sr, sp);
    if (rc) { delete S; return rc; }
    *out = S;
    *nrows = S->nrows;
    *nnz = (int64_t)S->ix.size();
    return 0;
}

// The mass and energy rows of pb_tpsa_thm_balance_rows on host arrays (ip / ix / a: the system, b: its right-hand
// side); returns the number of Jacobian entries outside the pattern.
int emu_tpsa_thm_balance_rows(int nd, int64_t nc, const int32_t *ip, const int32_t *ix, const int32_t *jf_ip,
                              const int32_t *jf_ix, const double *jf_a, const double *neg_res, double *a, double *b) {
    return nd == 3 ? balance_rows<3, 2>(nc, ip, ix, jf_ip, jf_ix, jf_a, neg_res, a, b)
                   : balance_rows<2, 2>(nc, ip, ix, jf_ip, jf_ix, jf_a, neg_res, a, b);
}

// copy the system out (indptr nrows + 1, indices / data nnz, rhs nrows) and free the handle
void emu_tpsa_thm_get(void *h, int32_t *ip, int32_t *ix, double *a, double *b) {
    System *S = (System *)h;
    for (size_t q = 0; q < S->ip.size(); ++q) ip[q] = S->ip[q];
    for (size_t q = 0; q < S->ix.size(); ++q) { ix[q] = S->ix[q]; a[q] = S->a[q]; }
    for (size_t q = 0; q < S->b.size(); ++q) b[q] = S->b[q];
    delete S;
}
}
