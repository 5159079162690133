// mosh2_emu_multi.cpp -- TEST-ONLY host build of the multi-model job (mosh2_job_create_multi).
//
// The host build proper (mosh2_emu.cpp) is compiled as part of this translation unit: its solve() runs a multi-model job
// as mosh2_stageii_multi_kernel does on the GPU -- one workspace layout behind the multi-model shared-memory header
// (mosh2_host::multi_smem_header), and every chunk bound to a copy of its subject's Model record in that header.
#include "mosh2_emu.cpp"

// sequences of several subjects back to back on the frame axis (mosh2_job_create_multi): sequence q solved with
// descs[model_of_seq[q]]; -1 when the models do not have one kernel shape or an index is out of range
extern "C" int mosh2_emu_solve_multi(const mosh2_model_desc *const *descs, int32_t n_models, const mosh2_options *opt, int32_t n_seq,
                                     const int32_t *frame_counts, const int32_t *model_of_seq, const double *obs, const uint8_t *vis,
                                     const mosh2_schedule *sched, int32_t precision, const mosh2_result *res) {
    if (!descs || n_models < 1 || n_seq < 1 || !frame_counts || !model_of_seq) return -1;
    for (int q = 0; q < n_seq; ++q)
        if (model_of_seq[q] < 0 || model_of_seq[q] >= n_models || frame_counts[q] < 1) return -1;
    if (precision == MOSH2_F64) return solve<double>(descs, n_models, model_of_seq, *opt, n_seq, frame_counts, obs, vis, sched, *res);
    return solve<float>(descs, n_models, model_of_seq, *opt, n_seq, frame_counts, obs, vis, sched, *res);
}
