// mosh2_emu.cpp -- TEST-ONLY host build of the CTA program (moshpp_b200/csrc/mosh2_device.cuh).
//
// Compiles the device source with MOSH2_EMU: one "thread" (tid 0 of 1), barriers are no-ops.  The CPU
// test-suite runs it against the oracle to validate index math and control flow of the exact code that
// nvcc compiles for sm_90a.  The model tables, options, chunk table, workspace layout and argument checks come from the
// library's own job preparation (moshpp_b200/csrc/mosh2_host.h).  It is never linked into libmosh2.so and never loaded
// by moshpp_b200.
#define MOSH2_EMU 1
#include "../../moshpp_b200/csrc/mosh2_host.h"
#include "../tc/gauss_newton_case.h"

#include <cstring>
#include <memory>
#include <string>
#include <vector>

namespace {

template <class T>
T *align32(char *raw) { return reinterpret_cast<T *>(raw + ((32 - (reinterpret_cast<uintptr_t>(raw) & 31)) & 31)); }

template <class real>
void widen(double *dst, const real *src, size_t n) {
    if (dst) for (size_t i = 0; i < n; ++i) dst[i] = double(src[i]);
}

// mosh2_host::build_model with every table in a 32-byte aligned host buffer, laid out for 20-marker tiles and the CUDA-core
// J^T J (the host build has no tensor cores)
template <class real>
struct HostModel {
    mosh2::Model<real> m{};
    std::vector<std::vector<char>> store;
    explicit HostModel(const mosh2_model_desc &d) {
        mosh2_host::build_model<real>(d, m, [this](const auto *src, size_t n) {
            store.emplace_back((n + 1) * sizeof(*src) + 32);
            auto *p = align32<std::remove_const_t<std::remove_pointer_t<decltype(src)>>>(store.back().data());
            std::copy(src, src + n, p);
            return static_cast<decltype(src)>(p);
        });
        m.tile_markers = 20;
        m.dev_no_tc = 1;
    }
};

// One job on the host build: its outputs in the compute type, the Job record, and the shared memory of the workspace of `m`
// behind `header` bytes.  Chunks run one after the other.
template <class real>
struct HostJob {
    size_t F, M, PF, PR, nd;
    std::vector<real> obs, fullpose, pose, trans, dmpls, mk, errs;
    std::vector<int> status, counters, tab;
    int totals[8] = {};
    mosh2::Job<real> job{};
    mosh2_host::Layout<real, false> L;
    std::vector<char> smem_raw;

    HostJob(const mosh2_model_desc &desc, const mosh2_options &opt, int n_frames, const double *o, const uint8_t *vis,
            const mosh2::Model<real> &m, unsigned header)
        : F(n_frames), M(desc.n_markers), PF(size_t(3) * desc.n_joints), PR(desc.p_red), nd(desc.n_dmpl), obs(o, o + F * M * 3),
          fullpose(F * PF), pose(F * PR), trans(F * 3), dmpls(F * nd + 1), mk(F * M * 3), errs(F * mosh2::N_ERR), status(F),
          counters(F * 4), L(mosh2_host::layout<real, false>(m, header)), smem_raw(L.smem + 128) {
        job.n_frames = job.n_chunks = n_frames;
        job.obs = obs.data(); job.vis = vis;
        job.fullpose = fullpose.data(); job.pose = pose.data(); job.trans = trans.data(); job.dmpls = nd ? dmpls.data() : nullptr;
        job.markers_sim = mk.data(); job.errs = errs.data(); job.status = status.data(); job.counters = counters.data();
        job.totals = totals;
        job.opt = mosh2_host::to_options(opt);
    }
    void set_chunks(std::vector<int> t) {
        tab = std::move(t);
        job.chunk_tab = tab.data();
        job.n_chunks = int(tab.size() / mosh2::kChunkRec);
    }
    // chunk c with the Model record `m`, or (in_header) with a copy of it in the shared-memory header, as the multi-model kernel
    // binds it
    void run_chunk(int c, const mosh2::Model<real> &m, bool in_header = false) {
        unsigned char *smem = align32<unsigned char>(smem_raw.data());
        std::memset(smem, 0, L.smem + 64);
        mosh2::m2_smem_ref() = smem;
        const void *rec = in_header ? std::memcpy(smem + mosh2::kSmemHeader, &m, sizeof m) : &m;
        mosh2::Solver<real, false> s(*static_cast<const mosh2::Model<real> *>(rec), job, L.w, L.d, mosh2::Cta{0, 1});
        s.run_chunk(c);
    }
    void widen_result(const mosh2_result &r) const {
        widen(r.fullpose, fullpose.data(), F * PF);
        widen(r.pose, pose.data(), F * PR);
        widen(r.trans, trans.data(), F * 3);
        if (nd) widen(r.dmpls, dmpls.data(), F * nd);
        widen(r.markers_sim, mk.data(), F * M * 3);
        widen(r.errs, errs.data(), F * mosh2::N_ERR);
        if (r.status) std::copy(status.begin(), status.end(), r.status);
        if (r.counters) std::copy(counters.begin(), counters.end(), r.counters);
    }
};

// Sequences back to back on one frame axis, chunked as mosh2_job_create_batch chunks them.  model_of_seq == nullptr: one model
// (a batch job); else sequence q is solved with descs[model_of_seq[q]] and every chunk binds a copy of its model's record in the
// multi-model shared-memory header (a multi-model job).  resume_all: then a boundary repair of every chunk, in order -- chunk c
// continues from the rows chunk c-1 emitted.  root_turns (or nullptr): per chunk, full turns added to the root of its cold
// start (what mosh2_job_relaunch_chunks writes into the chunk record; the chunks of a launch are independent, so setting them
// before the one pass over the chunks gives the rows of a launch followed by a relaunch of the chunks with turns).
template <class real>
int solve(const mosh2_model_desc *const *descs, int n_models, const int *model_of_seq, const mosh2_options &opt, int n_seq,
          const int *counts, const double *obs, const uint8_t *vis, const mosh2_schedule *sched, const mosh2_result &res,
          bool resume_all = false, const int *root_turns = nullptr) {
    std::vector<std::unique_ptr<HostModel<real>>> hms;
    for (int k = 0; k < n_models; ++k) {
        std::string msg;
        if (const int rc = mosh2_host::check_model_desc(*descs[k], &msg)) return rc;
        hms.emplace_back(new HostModel<real>(*descs[k]));
        if (mosh2_host::kernel_shape_mismatch(hms[0]->m, hms[k]->m)) return MOSH2_E_INVALID;
    }
    int n_frames = 0;
    for (int q = 0; q < n_seq; ++q) n_frames += counts[q];
    const unsigned header = model_of_seq ? mosh2_host::multi_smem_header<real>() : mosh2::kSmemHeader;
    HostJob<real> hj(*descs[0], opt, n_frames, obs, vis, hms[0]->m, header);
    hj.set_chunks(mosh2_host::schedule_table(sched, counts, n_seq));
    if (root_turns)
        for (int c = 0; c < hj.job.n_chunks; ++c) hj.tab[size_t(c) * mosh2::kChunkRec + 5] = root_turns[c];
    const std::vector<int> moc = model_of_seq ? mosh2_host::model_of_chunks(hj.tab, counts, n_seq, model_of_seq)
                                              : std::vector<int>(size_t(hj.job.n_chunks), 0);
    for (int c = 0; c < hj.job.n_chunks; ++c) hj.run_chunk(c, hms[moc[c]]->m, model_of_seq != nullptr);
    if (resume_all)
        for (int c = 1; c < hj.job.n_chunks; ++c) {
            hj.tab[size_t(c) * mosh2::kChunkRec + 3] = -1;
            hj.run_chunk(c, hms[moc[c]]->m, model_of_seq != nullptr);
        }
    hj.widen_result(res);
    return 0;
}

// linearise mode (mosh2_job_linearize): every frame evaluated / linearised at the caller's state; observations and states
// rounded to `real` and the outputs widened to float64, as the library does
template <class real>
int linearize(const mosh2_model_desc &desc, const mosh2_options &opt, int n_frames, const double *obs, const uint8_t *vis,
              int step, int build, const double *x, const mosh2_lin_out &out) {
    std::string msg;
    if (const int rc = mosh2_host::check_model_desc(desc, &msg)) return rc;
    const HostModel<real> hm(desc);
    HostJob<real> hj(desc, opt, n_frames, obs, vis, hm.m, mosh2::kSmemHeader);
    const size_t F = n_frames, M = desc.n_markers, NX = 3 + desc.p_red + desc.n_dmpl;
    const size_t n = step == 2 ? desc.n_free2 : desc.n_free1;
    const mosh2_host::LinLayout L = mosh2_host::lin_layout(F, M, NX, n);
    std::vector<real> lin(L.words);
    for (size_t i = 0; i < F * NX; ++i) lin[L.x + i] = real(x[i]);
    mosh2_host::bind_lin(hj.job, lin.data(), L);
    hj.job.lin_mode = build ? 2 : 1;
    hj.job.lin_step = step;
    for (int f = 0; f < n_frames; ++f) hj.run_chunk(f, hm.m);
    widen(out.errs, hj.errs.data(), hj.errs.size());
    widen(out.markers_sim, hj.mk.data(), hj.mk.size());
    widen(out.r, lin.data() + L.r, F * 3 * M);
    widen(out.vp, lin.data() + L.vp, F * 9 * M);
    if (build) {
        widen(out.A, lin.data() + L.A, F * n * n);
        widen(out.g, lin.data() + L.g, F * n);
        widen(out.J, lin.data() + L.J, F * 3 * M * n);
    }
    return 0;
}

// one Gauss-Newton solve and A g in the workspace of a model with the dimensions of `desc`: the host twin of gn_run
// (tests/tc/gauss_newton_test.cu), with the same layout and the same NaN fill
template <class real, bool BIG>
int run_gn(const mosh2_model_desc *desc, int n, const double *A, const double *g, double *dgn_out, double *Ag_out, int *ok_out) {
    mosh2::Model<real> m = mosh2_host::model_dims<real>(*desc);
    mosh2::Dims d;
    mosh2::Work<real, BIG> w;
    size_t smem = 0, gws_bytes = 0;
    if (n < 1 || n > m.n2 || !gn_case::layout<real, BIG>(m, d, w, smem, gws_bytes)) return -1;
    std::vector<char> smem_raw(smem + 32, char(gn_case::kNaN)), gws_raw(gws_bytes + 32, char(gn_case::kNaN));
    unsigned char *smem_base = align32<unsigned char>(smem_raw.data());
    char *gws = align32<char>(gws_raw.data());
    mosh2::m2_smem_ref() = smem_base;
    if (BIG) *reinterpret_cast<char **>(smem_base) = gws;
    real *wA = w.A, *wg = w.g;
    for (int i = 0; i < n; ++i) {
        for (int j = 0; j < n; ++j) wA[i * d.lda + j] = real(A[size_t(i) * n + j]);
        wg[i] = real(g[i]);
    }
    const mosh2::Job<real> job{};
    mosh2::Solver<real, BIG> s(m, job, w, d, mosh2::Cta{0, 1});
    const bool solved = s.gauss_newton(n);
    s.symv(w.g, w.Ag, n);
    for (int i = 0; i < n; ++i) { dgn_out[i] = double(w.dgn[i]); Ag_out[i] = double(w.Ag[i]); }
    *ok_out = solved ? 1 : 0;
    return 0;
}

template <class real>
int run_plan(const mosh2_model_desc *desc, int multi, int64_t *out) {
    mosh2::Model<real> m = mosh2_host::model_dims<real>(*desc);
    size_t smem = 0, gws = 0;
    int big = 0;
    mosh2_host::plan_workspace(m, &smem, &gws, &big, multi ? mosh2_host::multi_smem_header<real>() : mosh2::kSmemHeader);
    out[0] = int64_t(smem); out[1] = int64_t(gws); out[2] = big; out[3] = m.tile_markers; out[4] = int64_t(mosh2_host::kMaxSmem);
    return 0;
}

}  // namespace

// The library's workspace plan (mosh2_host::plan_workspace) for a model with the dimensions of `desc`, as mosh2_job_create
// (multi = 0) or mosh2_job_create_multi (multi = 1) makes it.  out[5]: shared-memory bytes per block, global-workspace bytes
// per block, 1 if the global-workspace layout was chosen, markers per Jacobian tile, the shared-memory budget.  The job fits
// iff out[0] <= out[4].
extern "C" int mosh2_emu_plan(const mosh2_model_desc *desc, int32_t precision, int32_t multi, int64_t *out) {
    if (precision == MOSH2_F64) return run_plan<double>(desc, multi, out);
    return run_plan<float>(desc, multi, out);
}

// `threads` is accepted for the signature of gn_run and ignored: the host build is one thread
extern "C" int mosh2_emu_gauss_newton(int32_t precision, int32_t big, int32_t threads, const mosh2_model_desc *desc, int32_t n,
                                      const double *A, const double *g, double *dgn_out, double *Ag_out, int32_t *ok_out) {
    (void)threads;
    if (precision == MOSH2_F64)
        return big ? run_gn<double, true>(desc, n, A, g, dgn_out, Ag_out, ok_out) : run_gn<double, false>(desc, n, A, g, dgn_out, Ag_out, ok_out);
    return big ? run_gn<float, true>(desc, n, A, g, dgn_out, Ag_out, ok_out) : run_gn<float, false>(desc, n, A, g, dgn_out, Ag_out, ok_out);
}

extern "C" int mosh2_emu_linearize_precision(const mosh2_model_desc *desc, const mosh2_options *opt, int32_t n_frames, const double *obs,
                                             const uint8_t *vis, int32_t step, int32_t build, const double *x, int32_t precision,
                                             const mosh2_lin_out *out) {
    if (precision == MOSH2_F64) return linearize<double>(*desc, *opt, n_frames, obs, vis, step, build, x, *out);
    return linearize<float>(*desc, *opt, n_frames, obs, vis, step, build, x, *out);
}

// float64, the Stage-I back end of the tests (conftest.EmuStageIBackend)
extern "C" int mosh2_emu_linearize(const mosh2_model_desc *desc, const mosh2_options *opt, int32_t n_frames, const double *obs,
                                   const uint8_t *vis, int32_t step, int32_t build, const double *x, const mosh2_lin_out *out) {
    return linearize<double>(*desc, *opt, n_frames, obs, vis, step, build, x, *out);
}

// several sequences of one subject back to back on the frame axis (mosh2_job_create_batch)
extern "C" int mosh2_emu_solve_batch(const mosh2_model_desc *desc, const mosh2_options *opt, int32_t n_seq, const int32_t *frame_counts,
                                     const double *obs, const uint8_t *vis, const mosh2_schedule *sched,
                                     int32_t precision, const mosh2_result *res) {
    if (precision == MOSH2_F64) return solve<double>(&desc, 1, nullptr, *opt, n_seq, frame_counts, obs, vis, sched, *res);
    return solve<float>(&desc, 1, nullptr, *opt, n_seq, frame_counts, obs, vis, sched, *res);
}

extern "C" int mosh2_emu_solve(const mosh2_model_desc *desc, const mosh2_options *opt, int32_t n_frames,
                               const double *obs, const uint8_t *vis, const mosh2_schedule *sched,
                               int32_t precision, const mosh2_result *res) {
    return mosh2_emu_solve_batch(desc, opt, 1, &n_frames, obs, vis, sched, precision, res);
}

// chunked solve followed by a resume (mosh2_job_relaunch_chunks with chunk_warmup < 0) of every chunk in order
extern "C" int mosh2_emu_solve_resumed(const mosh2_model_desc *desc, const mosh2_options *opt, int32_t n_frames,
                                       const double *obs, const uint8_t *vis, const mosh2_schedule *sched,
                                       int32_t precision, const mosh2_result *res) {
    if (precision == MOSH2_F64) return solve<double>(&desc, 1, nullptr, *opt, 1, &n_frames, obs, vis, sched, *res, true);
    return solve<float>(&desc, 1, nullptr, *opt, 1, &n_frames, obs, vis, sched, *res, true);
}

// the chunked schedule with the chunk records' root turns (one per chunk of the schedule)
extern "C" int mosh2_emu_solve_root_turns(const mosh2_model_desc *desc, const mosh2_options *opt, int32_t n_frames,
                                          const double *obs, const uint8_t *vis, const mosh2_schedule *sched, const int32_t *root_turns,
                                          int32_t precision, const mosh2_result *res) {
    if (precision == MOSH2_F64) return solve<double>(&desc, 1, nullptr, *opt, 1, &n_frames, obs, vis, sched, *res, false, root_turns);
    return solve<float>(&desc, 1, nullptr, *opt, 1, &n_frames, obs, vis, sched, *res, false, root_turns);
}
