// mosh2_emu_adapter.cpp -- TEST-ONLY host build of the mocap input adapter of the device source, linked into the same
// library as mosh2_emu.cpp (moshpp_b200/build.py build_emu).  Never part of libmosh2.so.
#define MOSH2_EMU 1
#include "../../moshpp_b200/csrc/mosh2_host.h"

#include <cstddef>
#include <string>

// mosh2_job_upload_markers_range on the host: frames [frame0, frame0 + n) of a batch job's observations obs [n_frames][M][3]
// (rounded to the job's precision, returned as float64) and visibility vis [n_frames][M], per sample through the device source's
// mosh2::gather_marker_sample, with the library's argument checks
extern "C" int mosh2_emu_upload_markers_range(int32_t precision, int32_t M, int32_t n_frames, double *obs, uint8_t *vis, int32_t frame0,
                                              int32_t n, const double *markers, int32_t n_file_frames, int32_t n_cols,
                                              const int32_t *col_of_marker, int32_t frame_start, int32_t frame_step,
                                              double unit_per_metre, const double *rot3x3) {
    std::string msg;
    if (const int rc = mosh2_host::check_marker_range(n_frames, M, frame0, n, markers, n_file_frames, n_cols, col_of_marker, frame_start,
                                                      frame_step, unit_per_metre, &msg))
        return rc;
    for (int f = 0; f < n; ++f)
        for (int mk = 0; mk < M; ++mk) {
            const int col = col_of_marker[mk];
            const double *p = col >= 0 ? markers + ((size_t(frame_start) + size_t(f) * frame_step) * n_cols + col) * 3 : nullptr;
            double v[3];
            const bool ok = mosh2::gather_marker_sample(p, unit_per_metre, rot3x3, v);
            const size_t i = size_t(frame0 + f) * M + mk;
            for (int c = 0; c < 3; ++c) obs[3 * i + c] = precision == MOSH2_F64 ? v[c] : double(float(v[c]));
            vis[i] = ok ? 1 : 0;
        }
    return 0;
}
