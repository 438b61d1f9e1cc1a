// emu_tpsa_contact.cpp -- TEST INFRASTRUCTURE ONLY: the host build of the TPSA contact system
// (porepy_b200/csrc/tpsa_system.cuh, run on the device by face.cu's pb_tpsa_contact_system / pb_tpsa_contact_rhs /
// pb_tpsa_contact_rows): the per-face routine of tpsa_face.cuh over all faces, the row pattern, the balance blocks, the
// interface rows, the right-hand side and the contact rows, one loop step where the device runs one thread, so the
// arithmetic and the layout can be checked on a box without a GPU.  Built by tests/emu_tpsa_contact.py with g++ into
// tests/emu/_emu_tpsa_contact.so; the product never builds, links or loads it.
#include <algorithm>
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

template <int ND>
int assemble(System &S, int64_t nc, int64_t nf, const int32_t *cf_ip, const int32_t *cf_ix, const int32_t *fc,
             const GeoView &G, const double *mu, const double *lam, const double *vol, const uint8_t *codes,
             const double *robw, const uint8_t *flags, TpsaMortars I, const double *g, const double *f,
             const double *sr, const double *sp) {
    using D = TpsaContactDims<ND>;
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
    // face -> mortar cell and the two mortar cells of every fracture cell, as pb_tpsa_contact_system checks them
    std::vector<int32_t> fm(nf, -1), pair(2 * I.nk, -1);
    for (int64_t m = 0; m < I.nm; ++m) {
        const int32_t fa = I.face[m], k = I.cell[m];
        if (fm[fa] >= 0 || fc[2 * fa + 1] >= 0) return 3;
        fm[fa] = (int32_t)m;
        if (pair[2 * k] < 0) pair[2 * k] = (int32_t)m;
        else if (pair[2 * k + 1] < 0) pair[2 * k + 1] = (int32_t)m;
        else return 3;
    }
    for (int64_t k = 0; k < I.nk; ++k) {
        if (pair[2 * k + 1] < 0) return 3;
        if (pair[2 * k] > pair[2 * k + 1]) std::swap(pair[2 * k], pair[2 * k + 1]);
    }
    I.face_mortar = fm.data();
    I.pair = pair.data();
    std::vector<int32_t> cc_ptr(nc + 1, 0), nb(kTpsaMaxNb);
    for (int64_t c = 0; c < nc; ++c) {
        const int n = tpsa_cell_neighbours(c, t, nb.data());
        if (n < 0) return 2;
        cc_ptr[c + 1] = cc_ptr[c] + n;
    }
    std::vector<int32_t> cc_ix(cc_ptr[nc]);
    std::vector<int64_t> blk_ptr(nc + 1, 0);
    for (int64_t c = 0; c < nc; ++c)
        blk_ptr[c + 1] = blk_ptr[c] + (int64_t)D::M::NZ * (cc_ptr[c + 1] - cc_ptr[c]) +
                         (int64_t)D::EXT * tpsa_contact_nfrac(c, t, fm.data());
    const int64_t ni = (int64_t)ND * (I.nm + I.nk);
    S.nrows = nc * B + ni;
    S.ip.assign(S.nrows + 1, 0);
    S.ix.assign((size_t)(blk_ptr[nc] + (int64_t)ND * I.nm * D::LF + (int64_t)ND * I.nk * D::LC), 0);
    S.a.assign(S.ix.size(), 0.0);
    S.b.assign(S.nrows, 0.0);
    for (int64_t c = 0; c < nc; ++c) {
        const int n = tpsa_cell_neighbours(c, t, nb.data());
        for (int j = 0; j < n; ++j) cc_ix[cc_ptr[c] + j] = nb[j];
        tpsa_contact_pattern_rows<ND>(c, n, nb.data(), blk_ptr[c], t, I, S.ip.data(), S.ix.data());
    }
    for (int64_t q = 0; q < ni; ++q) tpsa_contact_iface_pattern<ND>(q, nc, blk_ptr[nc], t, I, S.ip.data(), S.ix.data());
    S.ip[S.nrows] = (int32_t)S.ix.size();
    for (int64_t c = 0; c < nc; ++c)
        for (int j = 0; j < cc_ptr[c + 1] - cc_ptr[c]; ++j)
            tpsa_contact_block<ND>(c, j, t, cc_ptr.data(), cc_ix.data(), blk_ptr.data(), I, T, mu, lam, vol, S.a.data());
    for (int64_t q = 0; q < ni; ++q) tpsa_contact_iface_row<ND>(q, blk_ptr[nc], t, I, T, S.a.data());
    for (int64_t c = 0; c < nc; ++c)
        for (int l = 0; l < B; ++l) {
            const double src = l < ND ? (f ? f[c * ND + l] : 0.0)
                                       : (l < ND + NR ? (sr ? sr[c * NR + l - ND] : 0.0) : (sp ? sp[c] : 0.0));
            S.b[c * B + l] = tpsa_rhs_row<ND>(c, l, t, T, g, src);
        }
    for (int64_t q = 0; q < ni; ++q) S.b[nc * B + q] = tpsa_contact_iface_rhs<ND>(q, t, I, T, g);
    return 0;
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

// The contact system of pb_tpsa_contact_system (contact rows 0) and b0 of pb_tpsa_contact_rhs.  w: m2p, p2m, sign,
// volume, nm each.  *out: a handle for emu_tpsa_contact_get.  Returns 1 / 2 / 3 for a face with three cells, too many
// face neighbours, an interface pb_tpsa_contact_system refuses.
int emu_tpsa_contact_system(int64_t nc, int64_t nf, const int32_t *cf_ip, const int32_t *cf_ix, const int8_t *cf_da,
                            const double *fnorm, const double *fcent, const double *farea, const double *ccent, int nd,
                            const double *mu, const double *lam, const double *vol, const uint8_t *codes,
                            const double *robw, const uint8_t *flags, int64_t nm, int64_t nk, const int32_t *mface,
                            const int32_t *mcell, const double *w, const double *frames, double ct, const double *g,
                            const double *f, const double *sr, const double *sp, void **out, int64_t *nrows,
                            int64_t *nnz) {
    std::vector<int32_t> fc;
    if (face_cells(nc, nf, cf_ip, cf_ix, cf_da, fc)) return 1;
    if (nm != 2 * nk) return 3;
    for (int64_t m = 0; m < nm; ++m)
        if (mface[m] < 0 || mface[m] >= nf || mcell[m] < 0 || mcell[m] >= nk) return 3;
    GeoView G{nullptr, fnorm, fcent, farea, ccent, nullptr, 0, 1, nf, 1, nc, 1};
    const TpsaMortars I{nm, nk, mface, mcell, nullptr, nullptr, w, w + nm, w + 2 * nm, w + 3 * nm, frames, ct};
    System *S = new System;
    const int rc = nd == 3 ? assemble<3>(*S, nc, nf, cf_ip, cf_ix, fc.data(), G, mu, lam, vol, codes, robw, flags, I,
                                         g, f, sr, sp)
                           : assemble<2>(*S, nc, nf, cf_ip, cf_ix, fc.data(), G, mu, lam, vol, codes, robw, flags, I,
                                         g, f, sr, sp);
    if (rc) { delete S; return rc; }
    *out = S;
    *nrows = S->nrows;
    *nnz = (int64_t)S->ix.size();
    return 0;
}

// The contact rows of pb_tpsa_contact_rows on host arrays (ix / a: the system, b: its right-hand side; c0 = B nc, e0:
// the first entry of the contact rows, row0: their first row); returns the number of Jacobian entries outside the
// pattern.
int emu_tpsa_contact_rows(int nd, int64_t nrows, int64_t c0, int64_t e0, int64_t row0, const int32_t *ix,
                          const int32_t *jc_ip, const int32_t *jc_ix, const double *jc_a, const double *neg_res,
                          double *a, double *b) {
    int missing = 0;
    for (int64_t r = 0; r < nrows; ++r)
        missing += nd == 3 ? tpsa_contact_law_row<3>(r, c0, e0, row0 + r, ix, jc_ip, jc_ix, jc_a, neg_res, a, b)
                           : tpsa_contact_law_row<2>(r, c0, e0, row0 + r, ix, jc_ip, jc_ix, jc_a, neg_res, a, b);
    return missing;
}

// copy the system out (indptr nrows + 1, indices / data nnz, rhs nrows) and free the handle
void emu_tpsa_contact_get(void *h, int32_t *ip, int32_t *ix, double *a, double *b) {
    System *S = (System *)h;
    for (size_t q = 0; q < S->ip.size(); ++q) ip[q] = S->ip[q];
    for (size_t q = 0; q < S->ix.size(); ++q) { ix[q] = S->ix[q]; a[q] = S->a[q]; }
    for (size_t q = 0; q < S->b.size(); ++q) b[q] = S->b[q];
    delete S;
}
}
