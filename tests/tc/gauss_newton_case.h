// gauss_newton_case.h -- TEST-ONLY: one Gauss-Newton system in the Stage-II workspace, shared by the GPU harness
// (tests/tc/gauss_newton_test.cu) and its host twin (mosh2_emu_gauss_newton in tests/emu/mosh2_emu.cpp).
//
// The workspace is laid out by the product's own make_dims / carve from a Model that carries only the dimensions of a
// mosh2_model_desc, with the tile choice of the library's plan_workspace, so that ld, lda, ldp, npad and the offsets of
// A, Lm, Linv, Pn, g, tmp and ds are the ones a solve of that model uses.  Include after mosh2_device.cuh.
#pragma once
#include <cstddef>
#include <cstring>
#include <vector>

#include "../../include/mosh2.h"
#include "../../moshpp_b200/csrc/mosh2_host.h"

namespace gn_case {

using mosh2_host::kMaxSmem;                  // the library's shared-memory budget per block
constexpr unsigned char kNaN = 0xff;         // every byte 0xff: a NaN in float32 and in float64

template <class real>
mosh2::Model<real> dims_model(const mosh2_model_desc &desc) {
    mosh2::Model<real> m{};
    m.nJ = desc.n_joints; m.M = desc.n_markers; m.body_dof = desc.body_dof; m.p_red = desc.p_red;
    m.n_hand_red = desc.n_hand_red; m.n_hand_full = desc.n_hand_full; m.nd = desc.n_dmpl; m.kw = desc.kw;
    m.prior_k = desc.prior_k; m.prior_d = desc.prior_d; m.prior_d4 = (desc.prior_d + 3) & ~3;
    m.n1 = desc.n_free1; m.n2 = desc.n_free2;
    std::vector<double> hct;
    mosh2::HandBlock blocks[mosh2::kMaxHandBlocks];
    m.hb_n = mosh2_host::hand_blocks(desc.hand_comps, desc.n_hand_red, desc.n_hand_full, blocks, hct);
    m.hct_size = int(hct.size());
    return m;
}

// The layout plan_workspace would choose with the workspace in shared memory (BIG = false: 20-marker tiles, else 10)
// or in the per-block global workspace (BIG = true: 10-marker tiles).  False if its shared part exceeds the budget.
template <class real, bool BIG>
bool layout(mosh2::Model<real> &m, mosh2::Dims &d, mosh2::Work<real, BIG> &w, size_t &smem, size_t &gws) {
    for (int tile : {20, 10}) {
        if (BIG && tile == 20) continue;
        m.tile_markers = tile;
        d = mosh2::make_dims(m);
        w = mosh2::Work<real, BIG>{};
        mosh2::Arena S{mosh2::kSmemHeader}, G{0};
        mosh2::carve<real, BIG>(w, d, m, S, G);
        smem = (S.off + 15) & ~size_t(15);
        gws = (G.off + 255) & ~size_t(255);
        if (S.off <= kMaxSmem) return true;
    }
    return false;
}

}  // namespace gn_case
