// emu_tpsa.cpp -- TEST INFRASTRUCTURE ONLY: runs the per-face routine of the two-point stress approximation
// (porepy_b200/csrc/tpsa_face.cuh), which face.cu's tpsa_kernel runs one thread per face, on the host one face
// after the other, so the arithmetic and the value layout can be checked against the golden fixtures on a box
// without a GPU.  Built by tests/emu_tpsa.py with g++ into tests/emu/_emu_tpsa.so; the product never builds, links
// or loads it.
#include <cstdint>
#include <vector>

#include "../../porepy_b200/csrc/tpsa_face.cuh"

using namespace pb;

extern "C" {

// face -> cell table as face.cu builds it on the device: 2 per face, (cell << 1) | (sign < 0), -1 = none, slot 0 =
// the smaller cell index; out = 14 pointers in PB_TPSA_* order, each may be NULL
int emu_facegrid_tpsa(int64_t nc, int64_t nf, const int32_t *cf_ip, const int32_t *cf_ix, const int8_t *cf_da,
                      const double *fnorm, const double *fcent, const double *farea, const double *ccent, int nd,
                      const double *mu, const uint8_t *codes, const double *robw, const uint8_t *flags,
                      const int32_t *fc_ptr, double **out) {
    std::vector<int32_t> fc(2 * nf, -1);
    for (int64_t c = 0; c < nc; ++c)
        for (int q = cf_ip[c]; q < cf_ip[c + 1]; ++q) {
            const int32_t f = cf_ix[q];
            const int32_t enc = (int32_t)((c << 1) | (cf_da[q] < 0 ? 1 : 0));
            if (fc[2 * f] < 0) fc[2 * f] = enc;
            else if (fc[2 * f + 1] < 0) fc[2 * f + 1] = enc;
            else return 1;   // a face with more than two cells
        }
    GeoView G{nullptr, fnorm, fcent, farea, ccent, nullptr, 0, 1, nf, 1, nc, 1};
    TpsaOut o{};
    for (int k = 0; k < 14; ++k) o.t[k] = out[k];
    for (int64_t f = 0; f < nf; ++f) {
        if (nd == 3) tpsa_face<3>(f, G, mu, codes, robw, flags, fc.data(), fc_ptr, o);
        else tpsa_face<2>(f, G, mu, codes, robw, flags, fc.data(), fc_ptr, o);
    }
    return 0;
}
}
