// mosh2_emu_multi.cpp -- TEST-ONLY host build of the multi-model job (mosh2_job_create_multi).
//
// The host build proper (mosh2_emu.cpp) is compiled as part of this translation unit, so that its model tables (HostModel)
// serve here too.  mosh2_emu_solve_multi runs the sequences of several subjects back to back on one frame axis, as
// mosh2_stageii_multi_kernel does on the GPU: one workspace layout behind the multi-model shared-memory header
// (mosh2_host::multi_smem_header), and every chunk bound to a copy of its subject's Model record in that header.
#include "mosh2_emu.cpp"

namespace {

template <class real>
int run_multi(const mosh2_model_desc *const *descs, int n_models, const mosh2_options *opt, int n_seq, const int *counts,
              const int *model_of_seq, const double *obs, const uint8_t *vis, const mosh2_schedule *sched, const mosh2_result *res) {
    std::vector<HostModel<real>> hms(n_models);
    for (int k = 0; k < n_models; ++k) {
        hms[k].build(*descs[k]);
        hms[k].m.tile_markers = 20;
        hms[k].m.dev_no_tc = 1;                  // the host build runs the CUDA-core formulation
        if (k > 0 && mosh2_host::kernel_shape_mismatch(hms[0].m, hms[k].m)) return -1;
    }
    const mosh2_model_desc *desc = descs[0];
    int n_frames = 0;
    for (int q = 0; q < n_seq; ++q) n_frames += counts[q];
    const int chunk_len = sched ? sched->chunk_len : 0, warmup = sched ? sched->chunk_warmup : 0;
    const size_t F = n_frames, M = desc->n_markers, PF = size_t(3) * desc->n_joints, PR = desc->p_red, nd = desc->n_dmpl;
    std::vector<real> o(F * M * 3);
    for (size_t i = 0; i < o.size(); ++i) o[i] = real(obs[i]);
    std::vector<real> fullpose(F * PF), pose(F * PR), trans(F * 3), dmpls(F * nd + 1), mk(F * M * 3), errs(F * mosh2::N_ERR);
    mosh2::Job<real> job{};
    job.n_frames = n_frames;
    const int wu = warmup > 0 ? warmup : 0;
    const int wf = (!sched || sched->warmup_full < 0 || sched->warmup_full > wu) ? wu : sched->warmup_full;
    const int first_extra = (sched && sched->first_extra > 0 && chunk_len > 0 && wu > 0) ? sched->first_extra : 0;
    const std::vector<int> tab = mosh2_host::chunk_table(counts, n_seq, chunk_len, wu, wf, first_extra);
    const std::vector<int> moc = mosh2_host::model_of_chunks(tab, counts, n_seq, model_of_seq);
    job.n_chunks = int(tab.size() / mosh2::kChunkRec);
    job.chunk_tab = tab.data();
    job.obs = o.data(); job.vis = vis;
    job.fullpose = fullpose.data(); job.pose = pose.data(); job.trans = trans.data();
    job.dmpls = nd ? dmpls.data() : nullptr; job.markers_sim = mk.data(); job.errs = errs.data();
    std::vector<int> status(F, 0), counters(F * 4, 0);
    job.status = status.data(); job.counters = counters.data();
    int totals[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    job.totals = totals;
    mosh2::Options &q = job.opt;
    q.wt_data = opt->wt_data; q.wt_poseB = opt->wt_poseB; q.wt_poseH = opt->wt_poseH; q.wt_velo = opt->wt_velo;
    q.wt_dmpl = opt->wt_dmpl; q.wt_annealing = opt->wt_annealing; q.wt_extrap = opt->wt_extrap_dmpl;
    q.num_train_markers = opt->num_train_markers; q.delta_0 = opt->delta_0; q.e3_first = opt->e3_first; q.e3 = opt->e3;
    q.maxiter = opt->maxiter; q.optimize_fingers = opt->optimize_fingers; q.optimize_dynamics = opt->optimize_dynamics;
    q.wt_poseF = opt->wt_poseF; q.wt_expr = opt->wt_expr; q.optimize_face = opt->optimize_face;

    const mosh2::Dims d = mosh2::make_dims(hms[0].m);
    mosh2::Work<real, false> w{};
    mosh2::Arena S0{mosh2_host::multi_smem_header<real>()}, G0{0};
    mosh2::carve<real, false>(w, d, hms[0].m, S0, G0);
    std::vector<char> smem_raw(S0.off + 128);
    char *smem_base = smem_raw.data() + ((32 - (reinterpret_cast<uintptr_t>(smem_raw.data()) & 31)) & 31);
    mosh2::m2_smem_ref() = reinterpret_cast<unsigned char *>(smem_base);
    for (int c = 0; c < job.n_chunks; ++c) {
        std::memset(smem_base, 0, S0.off + 64);
        mosh2::Model<real> *rec = reinterpret_cast<mosh2::Model<real> *>(smem_base + mosh2::kSmemHeader);
        std::memcpy(static_cast<void *>(rec), &hms[moc[c]].m, sizeof(mosh2::Model<real>));
        mosh2::Solver<real, false> s(*rec, job, w, d, mosh2::Cta{0, 1});
        s.run_chunk(c);
    }
    auto conv = [](double *dst, const std::vector<real> &src, size_t n) {
        if (dst) for (size_t i = 0; i < n; ++i) dst[i] = double(src[i]);
    };
    conv(res->fullpose, fullpose, F * PF);
    conv(res->pose, pose, F * PR);
    conv(res->trans, trans, F * 3);
    if (nd) conv(res->dmpls, dmpls, F * nd);
    conv(res->markers_sim, mk, F * M * 3);
    conv(res->errs, errs, F * mosh2::N_ERR);
    if (res->status) std::memcpy(res->status, status.data(), F * sizeof(int));
    if (res->counters) std::memcpy(res->counters, counters.data(), F * 4 * sizeof(int));
    return 0;
}

}  // namespace

// sequences of several subjects back to back on the frame axis (mosh2_job_create_multi): sequence q solved with
// descs[model_of_seq[q]]; -1 when the models do not have one kernel shape or an index is out of range
extern "C" int mosh2_emu_solve_multi(const mosh2_model_desc *const *descs, int32_t n_models, const mosh2_options *opt, int32_t n_seq,
                                     const int32_t *frame_counts, const int32_t *model_of_seq, const double *obs, const uint8_t *vis,
                                     const mosh2_schedule *sched, int32_t precision, const mosh2_result *res) {
    if (!descs || n_models < 1 || n_seq < 1 || !frame_counts || !model_of_seq) return -1;
    for (int q = 0; q < n_seq; ++q)
        if (model_of_seq[q] < 0 || model_of_seq[q] >= n_models || frame_counts[q] < 1) return -1;
    if (precision == MOSH2_F64) return run_multi<double>(descs, n_models, opt, n_seq, frame_counts, model_of_seq, obs, vis, sched, res);
    return run_multi<float>(descs, n_models, opt, n_seq, frame_counts, model_of_seq, obs, vis, sched, res);
}
