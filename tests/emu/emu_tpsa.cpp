// emu_tpsa.cpp -- TEST INFRASTRUCTURE ONLY: the host build of the TPSA family (porepy_b200/csrc/tpsa_face.cuh and
// tpsa_system.cuh, run on the device by face.cu): the per-face routine of pb_tpsa, and the three-field, poromechanics /
// thermo-poromechanics and contact systems with their right-hand sides and row writers, one loop step where the device
// runs one thread, so the arithmetic and the layouts can be checked on a box without a GPU.  Built by tests/emu_tpsa.py
// with g++ into tests/emu/_emu_tpsa.so; the product never builds, links or loads it.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../porepy_b200/csrc/tpsa_face.cuh"
#include "../../porepy_b200/csrc/tpsa_system.cuh"

using namespace pb;

namespace {
// face -> cell table as face.cu builds it on the device: 2 per face, (cell << 1) | (sign < 0), -1 = none, slot 0 = the
// smaller cell index
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

struct System {
    int64_t nrows = 0;
    std::vector<int32_t> ip, ix;
    std::vector<double> a, b;
};

// The arguments of a system call besides the grid; fp_*: the sorted flux pattern (NS > 0), I: the interfaces (contact).
struct Inputs {
    const double *mu, *lam, *alpha, *vol;
    const uint8_t *codes;
    const double *robw;
    const uint8_t *flags;
    const int32_t *fp_ip, *fp_ix;
    TpsaMortars I;
    const double *g, *f, *sr, *sp;
};

// A and b of the three-field (NS = 0), poromechanics / thermo-poromechanics (NS = 1 / 2) or contact (NS = 0, contact)
// system, as face.cu assembles them: scalar rows and contact rows 0.  Returns 2 / 3 for too many face neighbours / an
// interface pb_tpsa_contact_system refuses.
template <int ND, int NS>
int assemble(System &S, bool contact, int64_t nc, int64_t nf, const int32_t *cf_ip, const int32_t *cf_ix,
             const int32_t *fc, const GeoView &G, Inputs in) {
    using D = TpsaDims<ND>;
    using K = TpsaContactDims<ND>;
    constexpr int NR = D::NR, B = D::B + NS;
    // stage 1: the face terms
    std::vector<int32_t> fc_ptr(nf + 1, 0);
    for (int64_t k = 0; k < nf; ++k) fc_ptr[k + 1] = fc_ptr[k] + (fc[2 * k] >= 0) + (fc[2 * k + 1] >= 0);
    std::vector<std::vector<double>> buf(14);
    TpsaOut o{};
    TpsaTerms T{};
    for (int k = 0; k < 14; ++k) {
        buf[k].assign(tpsa_term_size(k, ND, (size_t)fc_ptr[nf], (size_t)nf), 0.0);
        o.t[k] = buf[k].data();
        T.t[k] = buf[k].data();
    }
    for (int64_t k = 0; k < nf; ++k) tpsa_face<ND>(k, G, in.mu, in.codes, in.robw, in.flags, fc, fc_ptr.data(), o);
    const TpsaTopo t{nc, cf_ip, cf_ix, fc, fc_ptr.data()};
    // face -> mortar cell and the two mortar cells of every fracture cell, as pb_tpsa_contact_system checks them
    TpsaMortars &I = in.I;
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
    // the neighbour lists and the first entry of every block row
    std::vector<int32_t> cc_ptr(nc + 1, 0), nb(kTpsaMaxNb);
    for (int64_t c = 0; c < nc; ++c) {
        const int n = tpsa_cell_neighbours(c, t, nb.data());
        if (n < 0) return 2;
        cc_ptr[c + 1] = cc_ptr[c] + n;
    }
    std::vector<int32_t> cc_ix(cc_ptr[nc]);
    std::vector<int64_t> blk(nc + 1, 0);
    for (int64_t c = 0; c < nc; ++c) {
        const int n = tpsa_cell_neighbours(c, t, cc_ix.data() + cc_ptr[c]);
        if constexpr (NS > 0) blk[c + 1] = blk[c] + tpsa_poro_row_count<ND, NS>(c, n, in.fp_ip, in.fp_ix);
        else blk[c + 1] = blk[c] + (int64_t)D::NZ * n + (contact ? (int64_t)K::EXT * tpsa_contact_nfrac(c, t, fm.data()) : 0);
    }
    // the pattern and the values
    const int64_t ni = contact ? (int64_t)ND * (I.nm + I.nk) : 0;
    S.nrows = nc * B + ni;
    S.ip.assign(S.nrows + 1, 0);
    S.ix.assign((size_t)(blk[nc] + (int64_t)ND * I.nm * K::LF + (int64_t)ND * I.nk * K::LC), 0);
    S.a.assign(S.ix.size(), 0.0);
    S.b.assign(S.nrows, 0.0);
    for (int64_t c = 0; c < nc; ++c) {
        const int n = cc_ptr[c + 1] - cc_ptr[c];
        const int32_t *nbs = cc_ix.data() + cc_ptr[c];
        if constexpr (NS > 0)
            tpsa_poro_pattern_rows<ND, NS>(c, n, nbs, blk[c], in.fp_ip, in.fp_ix, S.ip.data(), S.ix.data());
        else if (contact) tpsa_contact_pattern_rows<ND>(c, n, nbs, blk[c], t, I, S.ip.data(), S.ix.data());
        else tpsa_pattern_rows<ND>(c, n, nbs, cc_ptr[c], S.ip.data(), S.ix.data());
    }
    for (int64_t q = 0; q < ni; ++q) tpsa_contact_iface_pattern<ND>(q, nc, blk[nc], t, I, S.ip.data(), S.ix.data());
    S.ip[S.nrows] = (int32_t)S.ix.size();
    for (int64_t c = 0; c < nc; ++c)
        for (int j = 0; j < cc_ptr[c + 1] - cc_ptr[c]; ++j) {
            if constexpr (NS > 0)
                tpsa_poro_block<ND, NS>(c, j, t, cc_ptr.data(), cc_ix.data(), blk.data(), T, in.mu, in.lam, in.alpha,
                                        in.vol, S.a.data());
            else if (contact)
                tpsa_contact_block<ND>(c, j, t, cc_ptr.data(), cc_ix.data(), blk.data(), I, T, in.mu, in.lam, in.vol,
                                       S.a.data());
            else tpsa_system_block<ND>(c, j, t, cc_ptr.data(), cc_ix.data(), T, in.mu, in.lam, in.vol, S.a.data());
        }
    for (int64_t q = 0; q < ni; ++q) tpsa_contact_iface_row<ND>(q, blk[nc], t, I, T, S.a.data());
    // stage 3: b, as tpsa_rhs_kernel
    for (int64_t c = 0; c < nc; ++c)
        for (int l = 0; l < D::B; ++l) {
            const double src = l < ND ? (in.f ? in.f[c * ND + l] : 0.0)
                                       : (l < ND + NR ? (in.sr ? in.sr[c * NR + l - ND] : 0.0) : (in.sp ? in.sp[c] : 0.0));
            S.b[c * B + l] = tpsa_rhs_row<ND>(c, l, t, T, in.g, src);
        }
    for (int64_t q = 0; q < ni; ++q) S.b[nc * B + q] = tpsa_contact_iface_rhs<ND>(q, t, I, T, in.g);
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
}  // namespace

extern "C" {

// The 14 value arrays of pb_tpsa; out = 14 pointers in PB_TPSA_* order, each may be NULL.
int emu_facegrid_tpsa(int64_t nc, int64_t nf, const int32_t *cf_ip, const int32_t *cf_ix, const int8_t *cf_da,
                      const double *fnorm, const double *fcent, const double *farea, const double *ccent, int nd,
                      const double *mu, const uint8_t *codes, const double *robw, const uint8_t *flags,
                      const int32_t *fc_ptr, double **out) {
    std::vector<int32_t> fc;
    if (face_cells(nc, nf, cf_ip, cf_ix, cf_da, fc)) return 1;
    GeoView G{nullptr, fnorm, fcent, farea, ccent, nullptr, 0, 1, nf, 1, nc, 1};
    TpsaOut o{};
    for (int k = 0; k < 14; ++k) o.t[k] = out[k];
    for (int64_t f = 0; f < nf; ++f) {
        if (nd == 3) tpsa_face<3>(f, G, mu, codes, robw, flags, fc.data(), fc_ptr, o);
        else tpsa_face<2>(f, G, mu, codes, robw, flags, fc.data(), fc_ptr, o);
    }
    return 0;
}

// A and b0 of one TPSA system on the grid given by cell_faces (CSC, +-1 data) and its geometry ((3, n) row-major
// arrays): ns = 0 and contact = 0 the three-field system, ns = 1 / 2 the poromechanics / thermo-poromechanics system
// (alpha, fp_ip / fp_ix: the sorted CSR pattern of div @ flux), contact = 1 the contact system (w: m2p, p2m, sign,
// volume, nm each).  The other arguments as for the pb_tpsa*_system / _rhs calls.  *out: a handle for emu_tpsa_get.
// Returns 1 / 2 / 3 for a face with three cells, too many face neighbours, an interface pb_tpsa_contact_system refuses.
int emu_tpsa_assemble(int contact, int ns, int64_t nc, int64_t nf, const int32_t *cf_ip, const int32_t *cf_ix,
                      const int8_t *cf_da, const double *fnorm, const double *fcent, const double *farea,
                      const double *ccent, int nd, const double *mu, const double *lam, const double *alpha,
                      const double *vol, const uint8_t *codes, const double *robw, const uint8_t *flags,
                      const int32_t *fp_ip, const int32_t *fp_ix, int64_t nm, int64_t nk, const int32_t *mface,
                      const int32_t *mcell, const double *w, const double *frames, double ct, const double *g,
                      const double *f, const double *sr, const double *sp, void **out, int64_t *nrows, int64_t *nnz) {
    std::vector<int32_t> fc;
    if (face_cells(nc, nf, cf_ip, cf_ix, cf_da, fc)) return 1;
    if (nm != 2 * nk) return 3;
    for (int64_t m = 0; m < nm; ++m)
        if (mface[m] < 0 || mface[m] >= nf || mcell[m] < 0 || mcell[m] >= nk) return 3;
    GeoView G{nullptr, fnorm, fcent, farea, ccent, nullptr, 0, 1, nf, 1, nc, 1};
    const TpsaMortars I{nm, nk, mface, mcell, nullptr, nullptr, w, w + nm, w + 2 * nm, w + 3 * nm, frames, ct};
    const Inputs in{mu, lam, alpha, vol, codes, robw, flags, fp_ip, fp_ix, I, g, f, sr, sp};
    System *S = new System;
    const int32_t *fcd = fc.data();
    const int rc = nd == 3 ? (ns == 2 ? assemble<3, 2>(*S, false, nc, nf, cf_ip, cf_ix, fcd, G, in)
                              : ns == 1 ? assemble<3, 1>(*S, false, nc, nf, cf_ip, cf_ix, fcd, G, in)
                                        : assemble<3, 0>(*S, contact, nc, nf, cf_ip, cf_ix, fcd, G, in))
                           : (ns == 2 ? assemble<2, 2>(*S, false, nc, nf, cf_ip, cf_ix, fcd, G, in)
                              : ns == 1 ? assemble<2, 1>(*S, false, nc, nf, cf_ip, cf_ix, fcd, G, in)
                                        : assemble<2, 0>(*S, contact, nc, nf, cf_ip, cf_ix, fcd, G, in));
    if (rc) { delete S; return rc; }
    *out = S;
    *nrows = S->nrows;
    *nnz = (int64_t)S->ix.size();
    return 0;
}

// The ns scalar rows of pb_tpsa_poro_fluid_rows (ns = 1) / pb_tpsa_thm_balance_rows (ns = 2) on host arrays (ip / ix /
// a: the system, b: its right-hand side); returns the number of Jacobian entries outside the pattern.
int emu_tpsa_balance_rows(int nd, int ns, int64_t nc, const int32_t *ip, const int32_t *ix, const int32_t *jf_ip,
                          const int32_t *jf_ix, const double *jf_a, const double *neg_res, double *a, double *b) {
    if (ns == 2)
        return nd == 3 ? balance_rows<3, 2>(nc, ip, ix, jf_ip, jf_ix, jf_a, neg_res, a, b)
                       : balance_rows<2, 2>(nc, ip, ix, jf_ip, jf_ix, jf_a, neg_res, a, b);
    return nd == 3 ? balance_rows<3, 1>(nc, ip, ix, jf_ip, jf_ix, jf_a, neg_res, a, b)
                   : balance_rows<2, 1>(nc, ip, ix, jf_ip, jf_ix, jf_a, neg_res, a, b);
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
void emu_tpsa_get(void *h, int32_t *ip, int32_t *ix, double *a, double *b) {
    System *S = (System *)h;
    std::copy(S->ip.begin(), S->ip.end(), ip);
    std::copy(S->ix.begin(), S->ix.end(), ix);
    std::copy(S->a.begin(), S->a.end(), a);
    std::copy(S->b.begin(), S->b.end(), b);
    delete S;
}
}
