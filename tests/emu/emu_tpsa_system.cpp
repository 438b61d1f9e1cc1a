// emu_tpsa_system.cpp -- TEST INFRASTRUCTURE ONLY: the host build of the TPSA system assembly
// (porepy_b200/csrc/tpsa_system.cuh, run on the device by face.cu's pb_tpsa_system / pb_tpsa_rhs): the per-face routine
// of tpsa_face.cuh over all faces, the row pattern and the block / right-hand-side gathers, one loop step where the device
// runs one thread, so the arithmetic and the layout can be checked on a box without a GPU.  Built by
// tests/emu_tpsa_system.py with g++ into tests/emu/_emu_tpsa_system.so; the product never builds, links or loads it.
#include <cstdint>
#include <vector>

#include "../../porepy_b200/csrc/tpsa_face.cuh"
#include "../../porepy_b200/csrc/tpsa_system.cuh"

using namespace pb;

namespace {
struct System {
    int nd = 0;
    int64_t nrows = 0;
    std::vector<int32_t> ip, ix;
    std::vector<double> a, b;
};

template <int ND>
int assemble(System &S, int64_t nc, int64_t nf, const int32_t *cf_ip, const int32_t *cf_ix, const int32_t *fc,
             const GeoView &G, const double *mu, const double *lam, const double *vol, const uint8_t *codes,
             const double *robw, const uint8_t *flags, const double *g, const double *f, const double *sr,
             const double *sp) {
    using D = TpsaDims<ND>;
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
    S.nrows = nc * B;
    S.ip.assign(S.nrows + 1, 0);
    S.ix.assign((size_t)D::NZ * cc_ptr[nc], 0);
    S.a.assign(S.ix.size(), 0.0);
    S.b.assign(S.nrows, 0.0);
    for (int64_t c = 0; c < nc; ++c) {
        const int n = tpsa_cell_neighbours(c, t, nb.data());
        for (int j = 0; j < n; ++j) cc_ix[cc_ptr[c] + j] = nb[j];
        tpsa_pattern_rows<ND>(c, n, nb.data(), cc_ptr[c], S.ip.data(), S.ix.data());
    }
    S.ip[S.nrows] = (int32_t)S.ix.size();
    for (int64_t c = 0; c < nc; ++c)
        for (int j = 0; j < cc_ptr[c + 1] - cc_ptr[c]; ++j)
            tpsa_system_block<ND>(c, j, t, cc_ptr.data(), cc_ix.data(), T, mu, lam, vol, S.a.data());
    for (int64_t c = 0; c < nc; ++c)
        for (int l = 0; l < B; ++l) {
            const double src = l < ND ? (f ? f[c * ND + l] : 0.0)
                                       : (l < ND + NR ? (sr ? sr[c * NR + l - ND] : 0.0) : (sp ? sp[c] : 0.0));
            S.b[c * B + l] = tpsa_rhs_row<ND>(c, l, t, T, g, src);
        }
    return 0;
}
}  // namespace

extern "C" {

// A and b of the TPSA system on the grid given by cell_faces (CSC, +-1 data) and its geometry ((3, n) row-major
// arrays); the arguments of pb_tpsa_system / pb_tpsa_rhs otherwise.  *out: a handle for emu_tpsa_system_get.
int emu_tpsa_system(int64_t nc, int64_t nf, const int32_t *cf_ip, const int32_t *cf_ix, const int8_t *cf_da,
                    const double *fnorm, const double *fcent, const double *farea, const double *ccent, int nd,
                    const double *mu, const double *lam, const double *vol, const uint8_t *codes, const double *robw,
                    const uint8_t *flags, const double *g, const double *f, const double *sr, const double *sp,
                    void **out, int64_t *nrows, int64_t *nnz) {
    std::vector<int32_t> fc(2 * nf, -1);
    for (int64_t c = 0; c < nc; ++c)
        for (int q = cf_ip[c]; q < cf_ip[c + 1]; ++q) {
            const int32_t k = cf_ix[q];
            const int32_t enc = (int32_t)((c << 1) | (cf_da[q] < 0 ? 1 : 0));
            if (fc[2 * k] < 0) fc[2 * k] = enc;
            else if (fc[2 * k + 1] < 0) fc[2 * k + 1] = enc;
            else return 1;   // a face with more than two cells
        }
    GeoView G{nullptr, fnorm, fcent, farea, ccent, nullptr, 0, 1, nf, 1, nc, 1};
    System *S = new System;
    S->nd = nd;
    const int rc = nd == 3 ? assemble<3>(*S, nc, nf, cf_ip, cf_ix, fc.data(), G, mu, lam, vol, codes, robw, flags, g,
                                         f, sr, sp)
                           : assemble<2>(*S, nc, nf, cf_ip, cf_ix, fc.data(), G, mu, lam, vol, codes, robw, flags, g,
                                         f, sr, sp);
    if (rc) { delete S; return rc; }
    *out = S;
    *nrows = S->nrows;
    *nnz = (int64_t)S->ix.size();
    return 0;
}

// copy the system out (indptr nrows + 1, indices / data nnz, rhs nrows) and free the handle
void emu_tpsa_system_get(void *h, int32_t *ip, int32_t *ix, double *a, double *b) {
    System *S = (System *)h;
    for (size_t q = 0; q < S->ip.size(); ++q) ip[q] = S->ip[q];
    for (size_t q = 0; q < S->ix.size(); ++q) { ix[q] = S->ix[q]; a[q] = S->a[q]; }
    for (size_t q = 0; q < S->b.size(); ++q) b[q] = S->b[q];
    delete S;
}
}
