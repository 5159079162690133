// gauss_newton_case.h -- TEST-ONLY: one Gauss-Newton system in the Stage-II workspace, shared by the GPU harness
// (tests/tc/gauss_newton_test.cu) and its host twin (mosh2_emu_gauss_newton in tests/emu/mosh2_emu.cpp).
//
// The workspace is laid out by the library's own layout (mosh2_host::layout) of a Model that carries only the dimensions of a
// mosh2_model_desc (mosh2_host::model_dims), with the tile choice of the library's plan_workspace, so that ld, lda, ldp, npad
// and the offsets of A, Lm, Linv, Pn, g, tmp and ds are the ones a solve of that model uses.  Include after mosh2_device.cuh.
#pragma once
#include <cstddef>

#include "../../moshpp_b200/csrc/mosh2_host.h"

namespace gn_case {

using mosh2_host::kMaxSmem;                  // the library's shared-memory budget per block
constexpr unsigned char kNaN = 0xff;         // every byte 0xff: a NaN in float32 and in float64

// The layout plan_workspace would choose with the workspace in shared memory (BIG = false: 20-marker tiles, else 10)
// or in the per-block global workspace (BIG = true: 10-marker tiles).  False if its shared part exceeds the budget.
template <class real, bool BIG>
bool layout(mosh2::Model<real> &m, mosh2::Dims &d, mosh2::Work<real, BIG> &w, size_t &smem, size_t &gws) {
    for (int tile : {20, 10}) {
        if (BIG && tile == 20) continue;
        m.tile_markers = tile;
        const mosh2_host::Layout<real, BIG> L = mosh2_host::layout<real, BIG>(m);
        d = L.d;
        w = L.w;
        smem = (L.smem + 15) & ~size_t(15);
        gws = (L.gws + 255) & ~size_t(255);
        if (L.smem <= kMaxSmem) return true;
    }
    return false;
}

}  // namespace gn_case
