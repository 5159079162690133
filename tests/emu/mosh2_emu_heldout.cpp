// mosh2_emu_heldout.cpp -- TEST-ONLY host build of the held-out marker folds (mosh2_job_upload_markers_folds,
// mosh2_job_heldout_errors), linked into the same library as mosh2_emu.cpp (moshpp_b200/build.py build_emu).  Never part of
// libmosh2.so.
#define MOSH2_EMU 1
#include "../../moshpp_b200/csrc/mosh2_host.h"

#include <cstddef>
#include <string>
#include <vector>

// mosh2_job_upload_markers_folds on the host: with the library's argument checks, the folds' observations obs [n_frames][M][3]
// (rounded to the job's precision, returned as float64) and visibility vis [n_frames][M] of a batch job with sequences of
// `counts` frames, and the side buffer side [n_folds][n][K][3], per sample through mosh2::fold_marker_sample.  *K_out: K.
extern "C" int mosh2_emu_upload_markers_folds(int32_t precision, int32_t M, int32_t n_seq, const int32_t *counts, double *obs, uint8_t *vis,
                                              double *side, int32_t *K_out, int32_t seq0, int32_t n_folds, const double *markers,
                                              int32_t n_file_frames, int32_t n_cols, const int32_t *col_of_marker, const uint8_t *hide,
                                              int32_t frame_start, int32_t frame_step, double unit_per_metre, const double *rot3x3) {
    const std::vector<int> cnt(counts, counts + n_seq);
    std::string msg;
    if (const int rc = mosh2_host::check_marker_folds(cnt, M, seq0, n_folds, hide, markers, n_file_frames, n_cols, col_of_marker,
                                                      frame_start, frame_step, unit_per_metre, &msg))
        return rc;
    std::vector<int> slot, idx;
    const int K = mosh2_host::fold_slots(hide, n_folds, M, slot, idx);
    *K_out = K;
    size_t frame0 = 0;
    for (int q = 0; q < seq0; ++q) frame0 += size_t(counts[q]);
    const int n = counts[seq0];
    for (int k = 0; k < n_folds; ++k)
        for (int t = 0; t < n; ++t)
            for (int mk = 0; mk < M; ++mk) {
                const int col = col_of_marker[mk], r = slot[size_t(k) * M + mk];
                const double *p = col >= 0 ? markers + ((size_t(frame_start) + size_t(t) * frame_step) * n_cols + col) * 3 : nullptr;
                double o[3], sd[3];
                const bool ok = mosh2::fold_marker_sample(p, unit_per_metre, rot3x3, r >= 0, o, sd);
                const size_t i = (frame0 + size_t(k) * n + t) * M + mk;
                for (int c = 0; c < 3; ++c) obs[3 * i + c] = precision == MOSH2_F64 ? o[c] : double(float(o[c]));
                vis[i] = ok ? 1 : 0;
                if (r >= 0)
                    for (int c = 0; c < 3; ++c) side[((size_t(k) * n + t) * K + r) * 3 + c] = sd[c];
            }
    return 0;
}

// mosh2_job_heldout_errors on the host: err [n_folds][n][K] and status [n_folds][n] of folds that start at frame0 of a job's rows
// markers_sim [F][M][3] (float64: the rows of a float32 job widened) and status [F], per sample through mosh2::heldout_error
extern "C" int mosh2_emu_heldout_errors(int32_t M, int32_t n_folds, int32_t n, const uint8_t *hide, int32_t frame0, const double *markers_sim,
                                        const int32_t *status, const double *side, double *err, int32_t *fold_status) {
    std::vector<int> slot, idx;
    const int K = mosh2_host::fold_slots(hide, n_folds, M, slot, idx);
    for (int k = 0; k < n_folds; ++k)
        for (int t = 0; t < n; ++t) {
            const size_t f = size_t(frame0) + size_t(k) * n + t, ft = size_t(k) * n + t;
            fold_status[ft] = status[f];
            for (int r = 0; r < K; ++r) {
                const int mk = idx[size_t(k) * K + r];
                err[ft * K + r] = mk < 0 ? NAN : mosh2::heldout_error(markers_sim + (f * M + mk) * 3, side + (ft * K + r) * 3,
                                                                      (status[f] & mosh2::ST_SOLVED) != 0);
            }
        }
    return 0;
}
