// mosh2_host.h -- host-side layout helpers shared by libmosh2.so and the test-only host build.
#pragma once
#include <vector>

#include "mosh2_device.cuh"

namespace mosh2_host {

// Splits the hand-PCA matrix C (n_red x n_full, row-major) into dense blocks of consecutive rows that
// share one non-zero column range (SMPL-H / SMPL-X: left and right hand; MANO: one block) and stores each
// block transposed, rows padded to a multiple of four: hct[ct_off + (q-q0)*rw4 + (r-r0)] = C[r][q].
// Falls back to a single dense block when the structure is irregular.
inline int hand_blocks(const double *C, int n_red, int n_full, mosh2::HandBlock *out, std::vector<double> &hct) {
    hct.clear();
    if (n_red == 0) return 0;
    std::vector<int> lo(n_red), hi(n_red);
    for (int r = 0; r < n_red; ++r) {
        int a = n_full, b = 0;
        for (int c = 0; c < n_full; ++c)
            if (C[size_t(r) * n_full + c] != 0.0) { if (c < a) a = c; b = c + 1; }
        if (b <= a) { a = 0; b = 0; }
        lo[r] = a; hi[r] = b;
    }
    int nb = 0;
    bool regular = true;
    for (int r = 0; r < n_red && regular;) {
        int e = r + 1;
        while (e < n_red && lo[e] == lo[r] && hi[e] == hi[r]) ++e;
        if (nb == mosh2::kMaxHandBlocks) { regular = false; break; }
        out[nb].r0 = r; out[nb].r1 = e; out[nb].q0 = lo[r]; out[nb].q1 = hi[r];
        ++nb;
        r = e;
    }
    for (int a = 0; a < nb && regular; ++a)          // column ranges of different blocks must not overlap
        for (int b = a + 1; b < nb; ++b)
            if (out[a].q0 < out[b].q1 && out[b].q0 < out[a].q1) regular = false;
    if (!regular) { nb = 1; out[0].r0 = 0; out[0].r1 = n_red; out[0].q0 = 0; out[0].q1 = n_full; }
    for (int b = 0; b < nb; ++b) {
        mosh2::HandBlock &h = out[b];
        h.rw4 = ((h.r1 - h.r0) + 3) & ~3;
        h.ct_off = int(hct.size());
        hct.resize(hct.size() + size_t(h.q1 - h.q0) * h.rw4, 0.0);
        for (int q = h.q0; q < h.q1; ++q)
            for (int r = h.r0; r < h.r1; ++r) hct[h.ct_off + size_t(q - h.q0) * h.rw4 + (r - h.r0)] = C[size_t(r) * n_full + q];
    }
    return nb;
}

// Chunk table of a job that holds n_seq sequences back to back on its frame axis: kChunkRec ints per chunk -- first
// emitted frame, end of the emitted range, first frame of the chunk's sequence, warm-up length (solved frames), number of
// fully solved warm-up frames.  chunk_len <= 0: one chunk per sequence (the reference's sequential pass).  Chunks never
// straddle a sequence boundary.  first_extra > 0: the FIRST chunk of every sequence emits chunk_len + first_extra frames --
// it has no warm-up to solve, so with first_extra = the cost of a warm-up every chunk of the sequence finishes at the same
// time, and no later chunk starts so close to the sequence start that its walk-back is cut short.
inline std::vector<int> chunk_table(const int *frame_counts, int n_seq, int chunk_len, int warmup, int warm_full, int first_extra = 0) {
    std::vector<int> tab;
    int s0 = 0;
    for (int q = 0; q < n_seq; ++q) {
        const int F = frame_counts[q];
        const int L = (chunk_len > 0 && chunk_len < F) ? chunk_len : F;
        const int E = (first_extra > 0 && L < F) ? first_extra : 0;
        for (int f = 0; f < F;) {
            long long e = (long long)f + L + (f == 0 ? E : 0);
            if (e > F) e = F;
            const int rec[mosh2::kChunkRec] = {s0 + f, s0 + int(e), s0, warmup, warm_full};
            tab.insert(tab.end(), rec, rec + mosh2::kChunkRec);
            f = int(e);
        }
        s0 += F;
    }
    return tab;
}

// ---- multi-model jobs (mosh2_job_create_multi) ------------------------------------------------------------------------------
// The chunks of one launch may belong to sequences of different subjects.  Each thread block copies the Model record of its
// chunk's subject into the shared-memory header, behind the base of the per-CTA global workspace, so the workspace of a
// multi-model launch starts this many bytes into the dynamic shared memory.
template <class real>
constexpr unsigned multi_smem_header() { return mosh2::kSmemHeader + ((unsigned(sizeof(mosh2::Model<real>)) + 15u) & ~15u); }

// Model index of every chunk of `tab` (chunk_table): the chunk's sequence is found from the first frame of its sequence.
inline std::vector<int> model_of_chunks(const std::vector<int> &tab, const int *frame_counts, int n_seq, const int *model_of_seq) {
    std::vector<int> out(tab.size() / mosh2::kChunkRec);
    int q = 0, s0 = 0;
    for (size_t c = 0; c < out.size(); ++c) {
        const int first = tab[c * mosh2::kChunkRec + 2];
        while (q + 1 < n_seq && s0 + frame_counts[q] <= first) s0 += frame_counts[q++];
        out[c] = model_of_seq[q];
    }
    return out;
}

// One workspace plan serves several models when they have the same kernel shape: equal sizes, free-variable counts, finger /
// face / joint-angle ranges, prior size and hand-block structure.  Returns the name of the first field (as in mosh2_model_desc)
// in which `b` differs from `a`, or nullptr.  Their tables (shape, latent markers, attachment, prior, ...) may differ.
template <class real>
const char *kernel_shape_mismatch(const mosh2::Model<real> &a, const mosh2::Model<real> &b) {
    const struct { const char *name; int a, b; } f[] = {
        {"n_joints", a.nJ, b.nJ}, {"n_markers", a.M, b.M}, {"body_dof", a.body_dof, b.body_dof}, {"p_red", a.p_red, b.p_red},
        {"n_hand_red", a.n_hand_red, b.n_hand_red}, {"n_hand_full", a.n_hand_full, b.n_hand_full}, {"n_dmpl", a.nd, b.nd},
        {"kw", a.kw, b.kw}, {"n_free1", a.n1, b.n1}, {"n_free2", a.n2, b.n2}, {"finger_lo", a.finger_lo, b.finger_lo},
        {"finger_hi", a.finger_hi, b.finger_hi}, {"n_expr", a.n_expr, b.n_expr}, {"face_lo", a.face_lo, b.face_lo},
        {"face_hi", a.face_hi, b.face_hi}, {"n_jangles", a.n_jang, b.n_jang}, {"prior_k", a.prior_k, b.prior_k},
        {"prior_d", a.prior_d, b.prior_d}, {"hand_comps (hand blocks)", a.hb_n, b.hb_n},
        {"hand_comps (hand-block table size)", a.hct_size, b.hct_size}};
    for (const auto &e : f)
        if (e.a != e.b) return e.name;
    for (int k = 0; k < a.hb_n; ++k) {
        const mosh2::HandBlock &x = a.hb[k], &y = b.hb[k];
        if (x.r0 != y.r0 || x.r1 != y.r1 || x.q0 != y.q0 || x.q1 != y.q1 || x.ct_off != y.ct_off || x.rw4 != y.rw4)
            return "hand_comps (hand-block structure)";
    }
    return nullptr;
}

}  // namespace mosh2_host
