// emu_group.cpp -- TEST INFRASTRUCTURE ONLY: the host build of the grouped block-Jacobi inverse of gmres.cu
// (porepy_b200/csrc/group_block.cuh): the same gather and Gauss-Jordan routines that group_inv_kernel runs with one lane
// per row, here in a loop, so their arithmetic can be checked on a box without a GPU.  Built by tests/emu_group.py with
// g++ into tests/emu/_emu_group.so; the product never builds, links or loads it.
#include <cstdint>
#include <vector>

#include "../../porepy_b200/csrc/group_block.cuh"

// inv_out at inv_off[g] (row-major s_g x s_g); returns the lowest group with a zero or non-finite pivot, or -1
extern "C" int64_t emu_group_inv(const int32_t *ip, const int32_t *ix, const double *data, int64_t ngroups,
                                 const int64_t *gptr, const int32_t *grows, const int32_t *gcols, const int64_t *inv_off,
                                 double *inv_out) {
    std::vector<double> A(pb::kGroupMax * pb::kGroupMax), E(pb::kGroupMax * pb::kGroupMax);
    for (int64_t g = 0; g < ngroups; ++g) {
        const int64_t base = gptr[g];
        const int s = (int)(gptr[g + 1] - base);
        for (int i = 0; i < s; ++i) pb::group_gather_row(ip, ix, data, grows[base + i], gcols + base, s, &A[i * s]);
        if (pb::group_invert_serial(A.data(), E.data(), s) >= 0) return g;
        for (int q = 0; q < s * s; ++q) {
            if (!std::isfinite(E[q])) return g;
            inv_out[inv_off[g] + q] = E[q];
        }
    }
    return -1;
}
