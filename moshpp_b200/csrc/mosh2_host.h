// mosh2_host.h -- job preparation shared by libmosh2.so and the test-only host build: model checks and tables, options,
// schedule, workspace layout and plan, linearise-mode buffer layout, argument checks of the marker upload.
#pragma once
#include <algorithm>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/mosh2.h"
#include "mosh2_device.cuh"

namespace mosh2_host {

// Formats a rejection into *msg and returns `code`.
inline int reject(std::string *msg, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    *msg = buf;
    return code;
}

// ---- model description ---------------------------------------------------------------------------------------------------------
// The checks of mosh2_model_create that need no device: 0, or MOSH2_E_INVALID / MOSH2_E_TOO_LARGE with the reason in *msg.
inline int check_model_desc(const mosh2_model_desc &d, std::string *msg) {
    if (d.n_joints < 1 || d.n_markers < 1 || d.kw < 1 || d.kw > 8 || d.n_free1 < 1 || d.n_free2 < d.n_free1)
        return reject(msg, MOSH2_E_INVALID, "inconsistent model sizes");
    if (d.n_expr < 0 || d.n_expr > d.n_dmpl || d.face_lo < 0 || d.face_hi < d.face_lo || d.face_hi > d.p_red)
        return reject(msg, MOSH2_E_INVALID, "inconsistent face description: n_expr=%d of %d linear coefficients, jaw ids [%d, %d)",
                      d.n_expr, d.n_dmpl, d.face_lo, d.face_hi);
    if (d.n_joints > 254) return reject(msg, MOSH2_E_TOO_LARGE, "%d joints (max 254)", d.n_joints);
    if (d.n_jangles < 0 || d.n_jangles > mosh2::kMaxJangles || (d.n_jangles > 0 && (!d.jangles_ids || !d.jangles_signs)))
        return reject(msg, MOSH2_E_INVALID, "joint-angle term: %d entries (max %d)", d.n_jangles, mosh2::kMaxJangles);
    for (int i = 0; i < d.n_jangles; ++i)
        if (d.jangles_ids[i] < 0 || d.jangles_ids[i] >= d.p_red)
            return reject(msg, MOSH2_E_INVALID, "joint-angle entry %d refers to pose id %d of %d", i, d.jangles_ids[i], d.p_red);
    for (int i = 0; i < d.prior_d; ++i) {
        const int id = d.prior_ids ? d.prior_ids[i] : d.prior_off + i;
        if (id < 0 || id >= d.p_red) return reject(msg, MOSH2_E_INVALID, "prior dimension %d refers to pose id %d of %d", i, id, d.p_red);
    }
    for (int j = 0; j < d.n_joints; ++j) {
        int depth = 1;
        for (int a = d.parents[j]; a >= 0; a = d.parents[a])
            if (a >= d.n_joints || ++depth > d.n_joints) return reject(msg, MOSH2_E_INVALID, "parents[] is not a forest (joint %d)", j);
        if (depth > mosh2::kMaxDepth)
            return reject(msg, MOSH2_E_TOO_LARGE, "kinematic chain of joint %d is %d levels deep (max %d)", j, depth, mosh2::kMaxDepth);
    }
    if (d.body_dof + d.n_hand_full != 3 * d.n_joints || d.body_dof + d.n_hand_red != d.p_red)
        return reject(msg, MOSH2_E_INVALID, "pose layout mismatch: body_dof=%d hand_full=%d hand_red=%d p_red=%d joints=%d",
                      d.body_dof, d.n_hand_full, d.n_hand_red, d.p_red, d.n_joints);
    return 0;
}

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

// The scalar part of a Model: sizes, free-variable counts, finger / face / joint-angle terms, prior size and hand-block
// structure; `hct`, if given, receives the hand-block table.  No table pointer is set.
template <class real>
mosh2::Model<real> model_dims(const mosh2_model_desc &d, std::vector<double> *hct = nullptr) {
    std::vector<double> own;
    if (!hct) hct = &own;
    mosh2::Model<real> m{};
    m.nJ = d.n_joints; m.M = d.n_markers; m.body_dof = d.body_dof; m.p_red = d.p_red;
    m.n_hand_red = d.n_hand_red; m.n_hand_full = d.n_hand_full; m.nd = d.n_dmpl; m.kw = d.kw;
    m.prior_k = d.prior_k; m.prior_d = d.prior_d; m.prior_d4 = (d.prior_d + 3) & ~3;
    m.n1 = d.n_free1; m.n2 = d.n_free2; m.finger_lo = d.finger_lo; m.finger_hi = d.finger_hi;
    m.n_expr = d.n_expr; m.face_lo = d.face_lo; m.face_hi = d.face_hi;
    m.n_jang = d.n_jangles;
    for (int i = 0; i < d.n_jangles && i < mosh2::kMaxJangles; ++i) { m.jang_id[i] = d.jangles_ids[i]; m.jang_sign[i] = real(d.jangles_signs[i]); }
    mosh2::HandBlock blocks[mosh2::kMaxHandBlocks];
    m.hb_n = hand_blocks(d.hand_comps, d.n_hand_red, d.n_hand_full, blocks, *hct);
    for (int b = 0; b < m.hb_n; ++b) m.hb[b] = blocks[b];
    m.hct_size = int(hct->size());
    return m;
}

// ---- workspace layout ------------------------------------------------------------------------------------------------------------
// The workspace of model `m` carved behind `header` bytes of shared memory (mosh2::carve).  smem / gws: the ends of the shared
// and the global arena, in bytes.
template <class real, bool BIG>
struct Layout {
    mosh2::Dims d;
    mosh2::Work<real, BIG> w;
    size_t smem, gws;
};

template <class real, bool BIG>
Layout<real, BIG> layout(const mosh2::Model<real> &m, unsigned header = mosh2::kSmemHeader) {
    Layout<real, BIG> L{};
    L.d = mosh2::make_dims(m);
    mosh2::Arena S{header}, G{0};
    mosh2::carve<real, BIG>(L.w, L.d, m, S, G);
    L.smem = S.off;
    L.gws = G.off;
    return L;
}

// ---- model tables ------------------------------------------------------------------------------------------------------------------
// Model `d` in precision `real`: the scalar part (model_dims) and every table, converted and derived on the host -- joints in
// depth order, the transposed hand blocks, both layouts of the pose-blend table, the prior's Q4 / Qt, the prior ids and the
// staged-table image.  Each table goes to `place(const T *host, size_t n)`, which returns where the table now lives, or nullptr
// on failure; build_model then stops and returns false.  The tile choice (plan_workspace) is left to the caller.
template <class real, class Place>
bool build_model(const mosh2_model_desc &d, mosh2::Model<real> &m, Place &&place) {
    std::vector<double> hct;
    m = model_dims<real>(d, &hct);
    const size_t nJ = d.n_joints, S = size_t(3) * d.n_markers, nd = d.n_dmpl, K = d.prior_k, D = d.prior_d, D4 = m.prior_d4;
    std::vector<int> order(nJ), depth(nJ, 0), ids(D);
    for (size_t j = 0; j < nJ; ++j) { int dj = 0; for (int a = d.parents[j]; a >= 0; a = d.parents[a]) ++dj; depth[j] = dj; }
    for (size_t j = 0; j < nJ; ++j) order[j] = int(j);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return depth[a] < depth[b]; });   // parents before children
    for (size_t i = 0; i < D; ++i) ids[i] = d.prior_ids ? d.prior_ids[i] : d.prior_off + int(i);
    // pose-blend table twice: [(nJ-1)][9 e][3 c][Sp] (eval: four slots per 16-byte load, no padding) and
    // [(nJ-1)][9 e][3M slots][x y z -] (build: one slot per 16-byte load)
    const size_t Sp = (S + 3) & ~size_t(3);
    std::vector<double> pdc((nJ - 1) * 27 * Sp, 0.0), pd4((nJ - 1) * 9 * S * 4, 0.0);
    for (size_t j = 0; j + 1 < nJ; ++j)
        for (size_t sl = 0; sl < S; ++sl)
            for (int c = 0; c < 3; ++c)
                for (int e = 0; e < 9; ++e) {
                    const double v = d.pd[(j * 3 * S + 3 * sl + c) * 9 + e];
                    pdc[((j * 9 + e) * 3 + c) * Sp + sl] = v;
                    pd4[((j * 9 + e) * S + sl) * 4 + c] = v;
                }
    // prior precision matrices per component, rows padded to D4: Q4 [K][D i][D4 l] and transposed, Qt [K][D l][D4 i]
    std::vector<double> q4(K * D * D4, 0.0), qt(K * D * D4, 0.0);
    for (size_t k = 0; k < K; ++k)
        for (size_t i = 0; i < D; ++i)
            for (size_t l = 0; l < D; ++l) q4[(k * D + i) * D4 + l] = qt[(k * D + l) * D4 + i] = d.prior_Q[(k * D + i) * D + l];
    // image of the staged shared-memory tables: what a chunk fetches with one bulk copy (its layout does not depend on the tile)
    const Layout<real, false> L = layout<real, false>(m);
    std::vector<unsigned char> img(L.w.stage_bytes, 0);
    const int *isrc[6] = {d.parents, order.data(), d.w_joint, d.free1, d.free2, ids.data()};
    const double *rsrc[9] = {d.w_val, d.v0, d.coefs, d.j0, d.hands_mean, d.prior_means, d.prior_neglogw, d.jd, hct.data()};
    mosh2::stage_image(L.w, L.d, m.hct_size, m.n_hand_full, [&](uint32_t ofs, int id, size_t n) {
        if (id < 6) { int *o = reinterpret_cast<int *>(img.data() + ofs); for (size_t i = 0; i < n; ++i) o[i] = isrc[id][i]; }
        else { real *o = reinterpret_cast<real *>(img.data() + ofs); for (size_t i = 0; i < n; ++i) o[i] = real(rsrc[id - 6][i]); }
    });

    bool ok = true;
    auto put = [&](auto &dst, const auto *src, size_t n) {      // dst: `const T *` member of m
        using T = std::remove_const_t<std::remove_pointer_t<std::remove_reference_t<decltype(dst)>>>;
        if (!ok) return;
        const std::vector<T> host(src, src + n);
        dst = place(host.data(), n);
        ok = dst != nullptr;
    };
    put(m.parents, d.parents, nJ); put(m.fk_order, order.data(), nJ); put(m.w_joint, d.w_joint, S * d.kw);
    put(m.hct, hct.data(), hct.size()); put(m.hands_mean, d.hands_mean, size_t(d.n_hand_full));
    put(m.v0, d.v0, S * 3); put(m.sd, d.sd, S * 3 * nd); put(m.pdc, pdc.data(), pdc.size()); put(m.pd4, pd4.data(), pd4.size());
    put(m.w_val, d.w_val, S * d.kw); put(m.j0, d.j0, nJ * 3); put(m.jd, d.jd, nJ * 3 * nd); put(m.coefs, d.coefs, S);
    put(m.prior_means, d.prior_means, K * D); put(m.prior_Q4, q4.data(), q4.size()); put(m.prior_Qt, qt.data(), qt.size());
    put(m.prior_nlw, d.prior_neglogw, K); put(m.prior_ids, ids.data(), D);
    put(m.free1, d.free1, size_t(d.n_free1)); put(m.free2, d.free2, size_t(d.n_free2));
    put(m.stage_blob, img.data(), img.size());
    return ok;
}

// ---- options and schedule ----------------------------------------------------------------------------------------------------------
inline mosh2::Options to_options(const mosh2_options &o) {
    mosh2::Options q{};
    q.wt_data = o.wt_data; q.wt_poseB = o.wt_poseB; q.wt_poseH = o.wt_poseH; q.wt_velo = o.wt_velo;
    q.wt_dmpl = o.wt_dmpl; q.wt_annealing = o.wt_annealing; q.wt_extrap = o.wt_extrap_dmpl;
    q.num_train_markers = o.num_train_markers; q.delta_0 = o.delta_0; q.e3_first = o.e3_first; q.e3 = o.e3;
    q.maxiter = o.maxiter; q.optimize_fingers = o.optimize_fingers; q.optimize_dynamics = o.optimize_dynamics;
    q.wt_poseF = o.wt_poseF; q.wt_expr = o.wt_expr; q.optimize_face = o.optimize_face;
    q.robust_sigma = o.robust_sigma;
    return q;
}

// robust_sigma: 0 (off) or a finite sigma > 0
inline bool robust_sigma_ok(const mosh2_options &o) {
    return o.robust_sigma == 0 || (o.robust_sigma > 0 && o.robust_sigma < 1e300);
}

// The options a linearisation takes from its call (mosh2_job_linearize: Stage I anneals these weights between minimisations,
// and leaves robust_sigma at 0); every other option stays as the job was created.
inline void apply_call_weights(mosh2::Options &q, const mosh2_options &o) {
    q.wt_data = o.wt_data; q.wt_poseB = o.wt_poseB; q.wt_poseH = o.wt_poseH; q.wt_poseF = o.wt_poseF; q.wt_expr = o.wt_expr;
    q.optimize_fingers = o.optimize_fingers; q.robust_sigma = o.robust_sigma;
}

// Chunk table of a job that holds n_seq sequences back to back on its frame axis: kChunkRec ints per chunk -- first
// emitted frame, end of the emitted range, first frame of the chunk's sequence, warm-up length (solved frames), number of
// fully solved warm-up frames, full turns added to the root of the chunk's cold start (0; mosh2_job_relaunch_chunks sets it).  chunk_len <= 0: one chunk per sequence (the reference's sequential pass).  Chunks never
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
            const int rec[mosh2::kChunkRec] = {s0 + f, s0 + int(e), s0, warmup, warm_full, 0};
            tab.insert(tab.end(), rec, rec + mosh2::kChunkRec);
            f = int(e);
        }
        s0 += F;
    }
    return tab;
}

// The chunk table of a job created with schedule `s` (NULL: the sequential pass).  Negative lengths count as zero, a
// warmup_full outside [0, chunk_warmup] as chunk_warmup, and first_extra only applies to chunked schedules with a warm-up.
inline std::vector<int> schedule_table(const mosh2_schedule *s, const int *frame_counts, int n_seq) {
    const int chunk_len = s && s->chunk_len > 0 ? s->chunk_len : 0, warmup = s && s->chunk_warmup > 0 ? s->chunk_warmup : 0;
    const int warm_full = (!s || s->warmup_full < 0 || s->warmup_full > warmup) ? warmup : s->warmup_full;
    const int first_extra = (s && s->first_extra > 0 && chunk_len > 0 && warmup > 0) ? s->first_extra : 0;
    return chunk_table(frame_counts, n_seq, chunk_len, warmup, warm_full, first_extra);
}

// ---- multi-model jobs (mosh2_job_create_multi) ------------------------------------------------------------------------------
// The chunks of one launch may belong to sequences of different subjects.  Each thread block copies the Model record of its
// chunk's subject into the shared-memory header, behind the base of the per-CTA global workspace, so the workspace of a
// multi-model launch starts this many bytes into the dynamic shared memory.
template <class real>
constexpr unsigned multi_smem_header() { return mosh2::kSmemHeader + ((unsigned(sizeof(mosh2::Model<real>)) + 15u) & ~15u); }

// ---- the workspace plan of a job ----------------------------------------------------------------------------------------------
constexpr size_t kMaxSmem = 227 * 1024;      // dynamic shared memory per block on sm_90

// Chooses the layout of `m`'s workspace and sets m.tile_markers.  Preference order, while the workspace fits the shared-memory
// budget: in float32 every marker in one tile (one pass: the Jacobian is built once and A written once per linearisation),
// then the fewest tiles of more than 20 markers; 20-marker tiles, then 10-marker tiles; then (*big = 1) the layout that moves
// A, its factor, the Jacobian tiles and the linear-block scratch to a per-CTA global workspace of *gws bytes.  *smem >
// kMaxSmem: the model does not fit at all.  `header`: bytes in front of the workspace (a multi-model job keeps the chunk's
// Model record there).
template <class real>
void plan_workspace(mosh2::Model<real> &m, size_t *smem, size_t *gws, int *big, unsigned header = mosh2::kSmemHeader) {
    std::vector<std::pair<int, int>> tries;                  // markers per tile, big
    const char *dev_tile = getenv("MOSH2_DEV_TILE");      // development aid: 10 = only the 10-marker tile in shared memory
    const bool dev_big = getenv("MOSH2_DEV_BIG") != nullptr;   // development aid: force the global-workspace layout
    if (!dev_big && !(dev_tile && atoi(dev_tile) == 10)) {
        if (sizeof(real) == 4)
            for (int k = 1; (m.M + k - 1) / k > 20; ++k) tries.push_back({(m.M + k - 1) / k, 0});
        tries.push_back({20, 0});
    }
    if (!dev_big) tries.push_back({10, 0});
    tries.push_back({10, 1});
    for (const auto &t : tries) {
        m.tile_markers = t.first;
        *big = t.second;
        size_t s, g;
        if (*big) { const Layout<real, true> L = layout<real, true>(m, header); s = L.smem; g = L.gws; }
        else { const Layout<real, false> L = layout<real, false>(m, header); s = L.smem; g = L.gws; }
        *smem = (s + 15) & ~size_t(15);
        *gws = (g + 255) & ~size_t(255);
        if (s <= kMaxSmem) return;
    }
}

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

// ---- linearise mode (mosh2_job_linearize) -------------------------------------------------------------------------------------
// One buffer of reals for F frames with n free variables: x [F][NX] | A [F][n][n] | g [F][n] | J [F][3M][n] | r [F][3M] | vp [F][9M].
struct LinLayout {
    size_t x, A, g, J, r, vp, words;      // element offsets, and the size
};

inline LinLayout lin_layout(size_t F, size_t M, size_t NX, size_t n) {
    LinLayout L;
    size_t o = 0;
    L.x = o; o += F * NX;
    L.A = o; o += F * n * n;
    L.g = o; o += F * n;
    L.J = o; o += F * 3 * M * n;
    L.r = o; o += F * 3 * M;
    L.vp = o; o += F * 9 * M;
    L.words = o;
    return L;
}

// Points the linearise-mode arrays of `job` into the buffer `p` of layout `L`.
template <class real>
void bind_lin(mosh2::Job<real> &job, real *p, const LinLayout &L) {
    job.lin_x = p + L.x; job.lin_A = p + L.A; job.lin_g = p + L.g; job.lin_J = p + L.J; job.lin_r = p + L.r; job.lin_vp = p + L.vp;
}

// ---- sequence sweep (mosh2_job_sequence_sweep) ----------------------------------------------------------------------------------
// The processed frames of a job (status has MOSH2_ST_SOLVED: at least one visible marker) in the processed order of their own
// sequence, from the status of the last launch and the chunk table `tab` (chunk_table; field 2 of a record is the first frame of
// the chunk's sequence).  nbr [F][4]: the two processed frames before and the two after each frame, -1 where the sequence ends
// first (skipped frames are passed over, sequences never neighbour each other).  colour[c]: the processed frames with processed
// index k = c (mod 3) within their sequence -- frames of one colour share no temporal residual.
inline void sequence_tables(const int *status, int n_frames, const std::vector<int> &tab, std::vector<int> &nbr,
                            std::vector<int> colour[3]) {
    std::vector<int> seq_start(n_frames, 0);
    for (size_t c = 0; c < tab.size() / mosh2::kChunkRec; ++c)
        for (int f = tab[c * mosh2::kChunkRec]; f < tab[c * mosh2::kChunkRec + 1]; ++f) seq_start[f] = tab[c * mosh2::kChunkRec + 2];
    nbr.assign(size_t(n_frames) * 4, -1);
    for (int c = 0; c < 3; ++c) colour[c].clear();
    std::vector<int> run;                                   // processed frames of the current sequence
    for (int f = 0; f <= n_frames; ++f) {
        if (f == n_frames || (f > 0 && seq_start[f] != seq_start[f - 1])) {
            const int n = int(run.size());
            for (int k = 0; k < n; ++k) {
                int *q = &nbr[size_t(run[k]) * 4];
                q[0] = k >= 2 ? run[k - 2] : -1; q[1] = k >= 1 ? run[k - 1] : -1;
                q[2] = k + 1 < n ? run[k + 1] : -1; q[3] = k + 2 < n ? run[k + 2] : -1;
                colour[k % 3].push_back(run[k]);
            }
            run.clear();
        }
        if (f < n_frames && (status[f] & MOSH2_ST_SOLVED)) run.push_back(f);
    }
}

// ---- mosh2_job_upload_markers_range ---------------------------------------------------------------------------------------------
// Argument checks of an upload of frames [frame0, frame0 + n) of a job of n_frames frames and M markers: 0, or MOSH2_E_INVALID
// with the reason in *msg.
inline int check_marker_range(int n_frames, int M, int frame0, int n, const double *markers, int n_file_frames, int n_cols,
                              const int *col_of_marker, int frame_start, int frame_step, double unit_per_metre, std::string *msg) {
    if (!markers || !col_of_marker) return reject(msg, MOSH2_E_INVALID, "null argument");
    if (frame0 < 0 || n < 1 || frame0 > n_frames - n)
        return reject(msg, MOSH2_E_INVALID, "frame range [%d, %d) outside the job's %d frames", frame0, frame0 + n, n_frames);
    if (n_cols < 1 || frame_step < 1 || frame_start < 0 || !(unit_per_metre > 0) ||
        size_t(frame_start) + size_t(n - 1) * frame_step >= size_t(n_file_frames))
        return reject(msg, MOSH2_E_INVALID, "frames %d + k*%d (k < %d) do not fit a file of %d frames", frame_start, frame_step, n,
                      n_file_frames);
    for (int i = 0; i < M; ++i)
        if (col_of_marker[i] >= n_cols) return reject(msg, MOSH2_E_INVALID, "marker %d: column %d of %d", i, col_of_marker[i], n_cols);
    return 0;
}

// ---- mosh2_job_upload_markers_folds -----------------------------------------------------------------------------------------------
// Argument checks of a fold upload into sequences [seq0, seq0 + n_folds) of a job whose sequences have `counts` frames: the folds'
// sequences exist and have one frame count, every hide mask is 0 / 1 and hides at least one marker, and the capture fits the first
// fold's range (check_marker_range).  0, or MOSH2_E_INVALID with the reason in *msg.
inline int check_marker_folds(const std::vector<int> &counts, int M, int seq0, int n_folds, const uint8_t *hide, const double *markers,
                              int n_file_frames, int n_cols, const int *col_of_marker, int frame_start, int frame_step,
                              double unit_per_metre, std::string *msg) {
    if (!hide) return reject(msg, MOSH2_E_INVALID, "null argument");
    if (seq0 < 0 || n_folds < 1 || size_t(seq0) + size_t(n_folds) > counts.size())
        return reject(msg, MOSH2_E_INVALID, "folds [%d, %d) outside the job's %d sequences", seq0, seq0 + n_folds, int(counts.size()));
    for (int k = 1; k < n_folds; ++k)
        if (counts[seq0 + k] != counts[seq0])
            return reject(msg, MOSH2_E_INVALID, "fold %d has %d frames, fold 0 %d: every fold is the same capture", k, counts[seq0 + k],
                          counts[seq0]);
    for (int k = 0; k < n_folds; ++k) {
        int n = 0;
        for (int i = 0; i < M; ++i) {
            const uint8_t h = hide[size_t(k) * M + i];
            if (h > 1) return reject(msg, MOSH2_E_INVALID, "hide[%d][%d] = %d (0 or 1)", k, i, int(h));
            n += h;
        }
        if (!n) return reject(msg, MOSH2_E_INVALID, "fold %d hides no marker", k);
    }
    int frame0 = 0, total = 0;
    for (int q = 0; q < seq0; ++q) frame0 += counts[q];
    for (int c : counts) total += c;
    return check_marker_range(total, M, frame0, counts[seq0], markers, n_file_frames, n_cols, col_of_marker, frame_start, frame_step,
                              unit_per_metre, msg);
}

// Side-buffer layout of a fold upload: slot[k * M + i] = rank of marker i among the markers fold k hides (-1: not hidden);
// idx[k * K + r] = the r-th marker fold k hides (-1 past its count).  Returns K, the most markers one fold hides.
inline int fold_slots(const uint8_t *hide, int n_folds, int M, std::vector<int> &slot, std::vector<int> &idx) {
    int K = 0;
    slot.assign(size_t(n_folds) * M, -1);
    for (int k = 0; k < n_folds; ++k) {
        int r = 0;
        for (int i = 0; i < M; ++i)
            if (hide[size_t(k) * M + i]) slot[size_t(k) * M + i] = r++;
        K = std::max(K, r);
    }
    idx.assign(size_t(n_folds) * K, -1);
    for (int k = 0; k < n_folds; ++k)
        for (int i = 0; i < M; ++i)
            if (slot[size_t(k) * M + i] >= 0) idx[size_t(k) * K + slot[size_t(k) * M + i]] = i;
    return K;
}

}  // namespace mosh2_host
