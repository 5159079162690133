// mosh2_emu_adapter.cpp -- TEST-ONLY host build of the mocap input adapter of the device source, linked into the same
// library as mosh2_emu.cpp (moshpp_b200/build.py build_emu).  Never part of libmosh2.so.
#define MOSH2_EMU 1
#include "../../include/mosh2.h"
#include "../../moshpp_b200/csrc/mosh2_device.cuh"

#include <cstddef>

// mosh2_job_upload_markers_range on the host: frames [frame0, frame0 + n) of a batch job's observations obs [n_frames][M][3]
// (rounded to the job's precision, returned as float64) and visibility vis [n_frames][M], per sample through the device source's
// mosh2::gather_marker_sample, with the library's argument checks
extern "C" int mosh2_emu_upload_markers_range(int32_t precision, int32_t M, int32_t n_frames, double *obs, uint8_t *vis, int32_t frame0,
                                              int32_t n, const double *markers, int32_t n_file_frames, int32_t n_cols,
                                              const int32_t *col_of_marker, int32_t frame_start, int32_t frame_step,
                                              double unit_per_metre, const double *rot3x3) {
    if (frame0 < 0 || n < 1 || frame0 > n_frames - n) return MOSH2_E_INVALID;
    if (n_cols < 1 || frame_step < 1 || frame_start < 0 || !(unit_per_metre > 0) ||
        size_t(frame_start) + size_t(n - 1) * frame_step >= size_t(n_file_frames))
        return MOSH2_E_INVALID;
    for (int i = 0; i < M; ++i)
        if (col_of_marker[i] >= n_cols) return MOSH2_E_INVALID;
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
