// mosh2_emu_sequence.cpp -- TEST-ONLY host build of the sequence sweep (mosh2_job_sequence_sweep), linked into the same library
// as mosh2_emu.cpp (moshpp_b200/build.py build_emu).  Never part of libmosh2.so.
//
// A batch job of one model is solved with its schedule, chunk after chunk, then swept: per sweep one pass per colour over the
// colour's frames, each through the sweep instantiation of Solver::run_chunk (Job::lin_mode == 3), with the neighbour table and
// colours of the library (mosh2_host::sequence_tables).
#define MOSH2_EMU 1
#include "../../moshpp_b200/csrc/mosh2_host.h"

#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

namespace {

template <class T>
T *align32_seq(char *raw) { return reinterpret_cast<T *>(raw + ((32 - (reinterpret_cast<uintptr_t>(raw) & 31)) & 31)); }

template <class real>
int solve_sequence(const mosh2_model_desc &desc, const mosh2_options &opt, int n_seq, const int *counts, const double *obs_in,
                   const uint8_t *vis, const mosh2_schedule *sched, int max_sweeps, const double *tol, const mosh2_result &res,
                   int *sweeps_out, double *deltas_out) {
    std::string msg;
    if (const int rc = mosh2_host::check_model_desc(desc, &msg)) return rc;
    std::vector<std::vector<char>> store;
    mosh2::Model<real> m{};
    mosh2_host::build_model<real>(desc, m, [&store](const auto *src, size_t n) {
        store.emplace_back((n + 1) * sizeof(*src) + 32);
        auto *p = align32_seq<std::remove_const_t<std::remove_pointer_t<decltype(src)>>>(store.back().data());
        std::copy(src, src + n, p);
        return static_cast<decltype(src)>(p);
    });
    m.tile_markers = 20;
    m.dev_no_tc = 1;
    int F = 0;
    for (int q = 0; q < n_seq; ++q) F += counts[q];
    const size_t M = desc.n_markers, PF = size_t(3) * desc.n_joints, PR = desc.p_red, nd = desc.n_dmpl;
    std::vector<real> obs(obs_in, obs_in + size_t(F) * M * 3), fullpose(F * PF), pose(F * PR), trans(F * 3), dmpls(F * nd + 1),
        mk(F * M * 3), errs(F * mosh2::N_ERR);
    std::vector<int> status(F), counters(F * 4, 0), nbr, colour[3];
    std::vector<double> delta(size_t(F) * 4);
    int totals[8] = {};
    const std::vector<int> tab = mosh2_host::schedule_table(sched, counts, n_seq);
    mosh2::Job<real> job{};
    job.n_frames = F;
    job.n_chunks = int(tab.size() / mosh2::kChunkRec);
    job.chunk_tab = tab.data();
    job.obs = obs.data(); job.vis = vis;
    job.fullpose = fullpose.data(); job.pose = pose.data(); job.trans = trans.data(); job.dmpls = nd ? dmpls.data() : nullptr;
    job.markers_sim = mk.data(); job.errs = errs.data(); job.status = status.data(); job.counters = counters.data();
    job.totals = totals;
    job.opt = mosh2_host::to_options(opt);
    const mosh2_host::Layout<real, false> L = mosh2_host::layout<real, false>(m, mosh2::kSmemHeader);
    std::vector<char> smem_raw(L.smem + 128);
    auto run = [&](int c, auto sweep) {
        unsigned char *smem = align32_seq<unsigned char>(smem_raw.data());
        std::memset(smem, 0, L.smem + 64);
        mosh2::m2_smem_ref() = smem;
        mosh2::Solver<real, false, decltype(sweep)::value> s(m, job, L.w, L.d, mosh2::Cta{0, 1});
        s.run_chunk(c);
    };
    for (int c = 0; c < job.n_chunks; ++c) run(c, std::false_type{});
    mosh2_host::sequence_tables(status.data(), F, tab, nbr, colour);
    job.lin_mode = 3;
    job.seq_nbr = nbr.data();
    job.seq_delta = delta.data();
    int sweeps = 0;
    while (sweeps < max_sweeps) {
        std::fill(delta.begin(), delta.end(), 0.0);
        for (int c = 0; c < 3; ++c)
            for (int f : colour[c]) run(f, std::true_type{});
        double md[4] = {0, 0, 0, 0};
        for (int f = 0; f < F; ++f)
            for (int q = 0; q < 4; ++q) md[q] = std::max(md[q], delta[size_t(f) * 4 + q]);
        if (deltas_out) for (int q = 0; q < 4; ++q) deltas_out[4 * sweeps + q] = md[q];
        ++sweeps;
        bool within = true;
        for (int q = 0; q < 4; ++q) within = within && md[q] <= tol[q];
        if (within) break;
    }
    *sweeps_out = sweeps;
    auto widen = [](double *dst, const std::vector<real> &src, size_t n) { if (dst) for (size_t i = 0; i < n; ++i) dst[i] = double(src[i]); };
    widen(res.fullpose, fullpose, F * PF);
    widen(res.pose, pose, F * PR);
    widen(res.trans, trans, F * 3);
    if (nd) widen(res.dmpls, dmpls, F * nd);
    widen(res.markers_sim, mk, F * M * 3);
    widen(res.errs, errs, F * mosh2::N_ERR);
    if (res.status) std::copy(status.begin(), status.end(), res.status);
    if (res.counters) std::copy(counters.begin(), counters.end(), res.counters);
    return 0;
}

}  // namespace

// The causal solve of a batch job (schedule `sched`; sequences back to back) followed by at most `max_sweeps` sequence sweeps,
// stopped after the first sweep whose largest row change is within tol[4] per group (root + body pose, other pose coefficients,
// translation, linear block).  *sweeps_out: sweeps run; deltas_out [max_sweeps][4] (or NULL): each sweep's largest changes.
// The result holds the rows after the last sweep; its velo / extrap_dmpl errs columns hold each frame's coupled temporal SSE.
extern "C" int mosh2_emu_solve_sequence(const mosh2_model_desc *desc, const mosh2_options *opt, int32_t n_seq, const int32_t *frame_counts,
                                        const double *obs, const uint8_t *vis, const mosh2_schedule *sched, int32_t precision,
                                        int32_t max_sweeps, const double *tol, const mosh2_result *res, int32_t *sweeps_out,
                                        double *deltas_out) {
    if (precision == MOSH2_F64)
        return solve_sequence<double>(*desc, *opt, n_seq, frame_counts, obs, vis, sched, max_sweeps, tol, *res, sweeps_out, deltas_out);
    return solve_sequence<float>(*desc, *opt, n_seq, frame_counts, obs, vis, sched, max_sweeps, tol, *res, sweeps_out, deltas_out);
}
