// mosh2.cu -- libmosh2.so: kernels and the C-ABI declared in include/mosh2.h.
//
// One CUDA thread block per chunk of frames runs the whole Stage-II schedule of
// src/moshpp/chmosh.py:584-724 on device (mosh2_device.cuh).  Built for sm_90a (H100) only.
#include "../../include/mosh2.h"

#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <map>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "mesh_distance.cuh"
#include "mosh2_device.cuh"
#include "mosh2_host.h"

namespace {

thread_local std::string g_err;

int fail(int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define CU(expr)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (expr);                                                                   \
        if (e_ != cudaSuccess) return fail(MOSH2_E_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

// ---------------------------------------------------------------------------------------------------------------------
// Caching allocator for job buffers.  A Stage-II call creates a job, runs it and destroys it; cudaMallocHost / cudaMalloc /
// cudaFree(Host) of its few tens of megabytes cost more wall clock than the solve itself and vary by 10x between calls.
// Freed blocks are therefore kept (per device, pinned host memory apart) and handed to the next job that fits; the cache
// is bounded and mosh2_release_cached_memory() empties it.
// ---------------------------------------------------------------------------------------------------------------------
class BlockCache {
  public:
    // dev >= 0: device memory of that device; dev == -1: pinned host memory
    cudaError_t get(int dev, size_t bytes, void **out) {
        const size_t need = round_up(bytes);
        {
            std::lock_guard<std::mutex> lock(mu_);
            auto &pool = pools_[dev];
            auto it = pool.lower_bound(need);
            if (it != pool.end() && it->first <= 2 * need + (1u << 20)) {
                *out = it->second;
                sizes_[*out] = it->first;
                cached_ -= it->first;
                pool.erase(it);
                return cudaSuccess;
            }
        }
        cudaError_t e = dev < 0 ? cudaMallocHost(out, need) : cudaMalloc(out, need);
        if (e != cudaSuccess) {             // make room and try once more
            release_all();
            cudaGetLastError();
            e = dev < 0 ? cudaMallocHost(out, need) : cudaMalloc(out, need);
        }
        if (e == cudaSuccess) { std::lock_guard<std::mutex> lock(mu_); sizes_[*out] = need; }
        return e;
    }
    void put(int dev, void *p) {
        if (!p) return;
        size_t bytes = 0;
        {
            std::lock_guard<std::mutex> lock(mu_);
            auto it = sizes_.find(p);
            if (it == sizes_.end()) { lock_free(dev, p); return; }
            bytes = it->second;
            sizes_.erase(it);
            if (cached_ + bytes <= kLimit) { pools_[dev].emplace(bytes, p); cached_ += bytes; return; }
        }
        lock_free(dev, p);
    }
    void release_all() {
        std::map<int, std::multimap<size_t, void *>> pools;
        { std::lock_guard<std::mutex> lock(mu_); pools.swap(pools_); cached_ = 0; }
        for (auto &dp : pools)
            for (auto &b : dp.second) lock_free(dp.first, b.second);
    }

  private:
    static constexpr size_t kLimit = size_t(1) << 30;      // cached bytes, all pools together
    static size_t round_up(size_t b) { const size_t g = b < (1u << 20) ? 4096 : (1u << 18); return (b + g - 1) / g * g; }
    static void lock_free(int dev, void *p) {
        if (dev < 0) cudaFreeHost(p);
        else { int cur = 0; cudaGetDevice(&cur); cudaSetDevice(dev); cudaFree(p); cudaSetDevice(cur); }
    }
    std::mutex mu_;
    std::map<int, std::multimap<size_t, void *>> pools_;
    std::map<void *, size_t> sizes_;
    size_t cached_ = 0;
};
BlockCache g_blocks;

using mosh2_host::kMaxSmem;
using mosh2_host::plan_workspace;
#ifndef MOSH2_F32_THREADS
#define MOSH2_F32_THREADS 384      // 168 registers per thread: measured best of 256 / 320 / 384 / 512 (profiles/)
#endif
template <class real> constexpr int threads_for() { return sizeof(real) == 4 ? MOSH2_F32_THREADS : 256; }

template <class real, bool BIG, bool SWEEP = false>
__global__ void __launch_bounds__(threads_for<real>(), 1)
mosh2_stageii_kernel(const __grid_constant__ mosh2::Model<real> m, const __grid_constant__ mosh2::Job<real> job,
                     const __grid_constant__ mosh2::Work<real, BIG> w, const __grid_constant__ mosh2::Dims d) {
    // The workspace layout `w` was computed on the host (mosh2::carve) and arrives in the constant bank: every array
    // is shared-memory base + a parameter word.  BIG = true (f64 / oversized models): A, its factor and the Jacobian
    // tiles live in a per-CTA global workspace whose base is parked in the shared-memory header.
    if (BIG) {
        if (threadIdx.x == 0) *reinterpret_cast<char **>(mosh2::m2_smem()) = job.gws + size_t(blockIdx.x) * job.gws_stride;   // (per block, not per chunk)
        __syncthreads();
    }
    mosh2::Cta c{int(threadIdx.x), int(blockDim.x)};
    mosh2::Solver<real, BIG, SWEEP> s(m, job, w, d, c);
    s.run_chunk(job.chunk_ids ? job.chunk_ids[blockIdx.x] : int(blockIdx.x));
}

// The same for a multi-model job (mosh2_job_create_multi): the sequences of the launch belong to subjects with models of one
// kernel shape, so `w` and `d` serve every chunk.  The block copies its chunk's Model record from the device array `models`
// into the shared-memory header (mosh2_host::multi_smem_header, behind the global-workspace base) and binds its Solver to
// that copy; the Solver stages that model's tables (Model::stage_blob) as in the single-model kernel.
template <class real, bool BIG, bool SWEEP = false>
__global__ void __launch_bounds__(threads_for<real>(), 1)
mosh2_stageii_multi_kernel(const mosh2::Model<real> *__restrict__ models, const int *__restrict__ model_of_chunk,
                           const __grid_constant__ mosh2::Job<real> job, const __grid_constant__ mosh2::Work<real, BIG> w,
                           const __grid_constant__ mosh2::Dims d) {
    static_assert(sizeof(mosh2::Model<real>) % 8 == 0, "the Model record is copied in 8-byte words");
    const int chunk = job.chunk_ids ? job.chunk_ids[blockIdx.x] : int(blockIdx.x);
    mosh2::Model<real> *rec = reinterpret_cast<mosh2::Model<real> *>(mosh2::m2_smem() + mosh2::kSmemHeader);
    {
        const unsigned long long *src = reinterpret_cast<const unsigned long long *>(models + model_of_chunk[chunk]);
        unsigned long long *dst = reinterpret_cast<unsigned long long *>(rec);
        for (int i = threadIdx.x; i < int(sizeof(mosh2::Model<real>) / 8); i += blockDim.x) dst[i] = src[i];
    }
    if (BIG && threadIdx.x == 0) *reinterpret_cast<char **>(mosh2::m2_smem()) = job.gws + size_t(blockIdx.x) * job.gws_stride;
    __syncthreads();
    mosh2::Cta c{int(threadIdx.x), int(blockDim.x)};
    mosh2::Solver<real, BIG, SWEEP> s(*rec, job, w, d, c);
    s.run_chunk(chunk);
}

// device copy of every model array in one precision
template <class real>
struct DevModel {
    mosh2::Model<real> m{};
    std::vector<void *> owned;
    int device = 0;
    ~DevModel() {
        for (void *p : owned) g_blocks.put(device, p);
    }
    // the tables of mosh2_host::build_model, each copied to a block of the cache
    int build(const mosh2_model_desc &d) {
        int rc = 0;
        auto place = [&](const auto *host, size_t n) -> decltype(host) {
            void *p = nullptr;
            cudaError_t e = g_blocks.get(device, n ? n * sizeof(*host) : 16, &p);   // (n = 0: still a valid address for the kernels)
            if (e == cudaSuccess) {
                owned.push_back(p);
                if (n) e = cudaMemcpy(p, host, n * sizeof(*host), cudaMemcpyHostToDevice);
            }
            if (e != cudaSuccess) { rc = fail(MOSH2_E_CUDA, "model upload: %s", cudaGetErrorString(e)); return nullptr; }
            return static_cast<decltype(host)>(p);
        };
        return mosh2_host::build_model<real>(d, m, place) ? 0 : rc;
    }
};

}  // namespace

template <class S, class D>
__global__ void convert_kernel(const S *__restrict__ src, D *__restrict__ dst, size_t n) {
    const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = D(src[i]);
}

// one packed float32 row per frame: [fullpose PF | trans 3 | dmpls nd | errs N_ERR | status | jacobian builds]
template <class real>
__global__ void pack_rows_kernel(const real *__restrict__ fullpose, const real *__restrict__ trans, const real *__restrict__ dmpls,
                                 const real *__restrict__ errs, const int *__restrict__ status, const int *__restrict__ counters,
                                 float *__restrict__ rows, int n_frames, int PF, int nd) {
    const int width = PF + 3 + nd + mosh2::N_ERR + 2;
    const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= size_t(n_frames) * width) return;
    const int f = int(i / width);
    int c = int(i - size_t(f) * width);
    float v;
    if (c < PF) v = float(fullpose[size_t(f) * PF + c]);
    else if ((c -= PF) < 3) v = float(trans[size_t(f) * 3 + c]);
    else if ((c -= 3) < nd) v = float(dmpls[size_t(f) * nd + c]);
    else if ((c -= nd) < mosh2::N_ERR) v = float(errs[size_t(f) * mosh2::N_ERR + c]);
    else if ((c -= mosh2::N_ERR) == 0) v = float(status[f]);
    else v = float(counters[4 * f + 2]);
    rows[i] = v;
}

// boundary check on the device: per chunk max |state on the last warm-up frame - emitted row of that frame| over
// (root+body pose, other pose coefficients, translation, linear coefficients); one warp per chunk
template <class real>
__global__ void boundary_delta_kernel(const real *__restrict__ warm_x, const int *__restrict__ warm_f, const real *__restrict__ pose,
                                      const real *__restrict__ trans, const real *__restrict__ dmpls, float *__restrict__ out,
                                      int n_chunks, int PR, int nd, int body) {
    const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (c >= n_chunks) return;
    const int f = warm_f[c];
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (f >= 0) {
        const real *x = warm_x + size_t(c) * (3 + PR + nd);
        for (int i = lane; i < PR; i += 32) {
            const float d = fabsf(float(x[3 + i] - pose[size_t(f) * PR + i]));
            if (i < body) v[0] = fmaxf(v[0], d); else v[1] = fmaxf(v[1], d);
        }
        if (lane < 3) v[2] = fabsf(float(x[lane] - trans[size_t(f) * 3 + lane]));
        for (int i = lane; i < nd; i += 32) v[3] = fmaxf(v[3], fabsf(float(x[3 + PR + i] - dmpls[size_t(f) * nd + i])));
    }
    for (int q = 0; q < 4; ++q) {
        for (int o = 16; o > 0; o >>= 1) v[q] = fmaxf(v[q], __shfl_xor_sync(0xffffffffu, v[q], o));
        if (lane == 0) out[4 * c + q] = v[q];
    }
}

// Mocap input adapter on the device (tools/mocap_interface.py:186,223-225,254-279; chmosh.py:582-594): from the raw marker
// table of a capture file [file frame][file column][xyz] (file units, float64) to the job's observations [frame][marker][xyz]
// (metres, compute precision) and visibility, per sample by mosh2::gather_marker_sample; markers whose label the file does
// not have (col < 0) are invisible and stored as zero.  `obs` / `vis` point at the first frame the call writes.
template <class real>
__global__ void gather_markers_kernel(const double *__restrict__ raw, int n_cols, const int *__restrict__ col_of_marker, int M,
                                      int n_frames, int frame_step, double unit_per_metre, const double *__restrict__ rot,
                                      real *__restrict__ obs, uint8_t *__restrict__ vis) {
    const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= size_t(n_frames) * M) return;
    const int f = int(i / M), mk = int(i - size_t(f) * M), col = col_of_marker[mk];
    double v[3];
    const bool ok = mosh2::gather_marker_sample(col >= 0 ? raw + (size_t(f) * frame_step * n_cols + col) * 3 : nullptr,
                                                unit_per_metre, rot, v);
    obs[3 * i] = real(v[0]); obs[3 * i + 1] = real(v[1]); obs[3 * i + 2] = real(v[2]);
    vis[i] = ok ? 1 : 0;
}

// Held-out folds (mosh2_job_upload_markers_folds): one thread per (fold, frame, marker) over the capture's raw table, staged once;
// per sample mosh2::fold_marker_sample.  `obs` / `vis` point at the first frame of fold 0, fold k starts k * n_frames frames later;
// side [n_folds][n_frames][K][3] (metres, float64) takes the samples of the markers a fold hides (slot [n_folds][M]: their rank).
template <class real>
__global__ void gather_folds_kernel(const double *__restrict__ raw, int n_cols, const int *__restrict__ col_of_marker, int M,
                                    int n_frames, int n_folds, int frame_step, double unit_per_metre, const double *__restrict__ rot,
                                    const int *__restrict__ slot, int K, real *__restrict__ obs, uint8_t *__restrict__ vis,
                                    double *__restrict__ side) {
    const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= size_t(n_folds) * n_frames * M) return;
    const int mk = int(i % M);
    const size_t ft = i / M;                     // fold * n_frames + frame
    const int t = int(ft % n_frames), k = int(ft / n_frames), col = col_of_marker[mk], r = slot[size_t(k) * M + mk];
    double o[3], sd[3];
    const bool ok = mosh2::fold_marker_sample(col >= 0 ? raw + (size_t(t) * frame_step * n_cols + col) * 3 : nullptr, unit_per_metre,
                                              rot, r >= 0, o, sd);
    obs[3 * i] = real(o[0]); obs[3 * i + 1] = real(o[1]); obs[3 * i + 2] = real(o[2]);
    vis[i] = ok ? 1 : 0;
    if (r >= 0) {
        double *p = side + (ft * K + r) * 3;
        p[0] = sd[0]; p[1] = sd[1]; p[2] = sd[2];
    }
}

// Held-out errors (mosh2_job_heldout_errors): one thread per (fold, frame, hidden marker), per sample mosh2::heldout_error from
// the fold's simulated marker and the side buffer; the thread of the first hidden marker also copies the frame's status.
template <class real>
__global__ void heldout_error_kernel(const real *__restrict__ markers_sim, const int *__restrict__ status, const double *__restrict__ side,
                                     const int *__restrict__ idx, int M, int n_frames, int n_folds, int K, int frame0,
                                     double *__restrict__ err, int *__restrict__ fold_status) {
    const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= size_t(n_folds) * n_frames * K) return;
    const int r = int(i % K);
    const size_t ft = i / K;
    const int k = int(ft / n_frames), mk = idx[size_t(k) * K + r];
    const size_t f = size_t(frame0) + ft;
    if (r == 0) fold_status[ft] = status[f];
    if (mk < 0) { err[i] = NAN; return; }
    const real *s = markers_sim + (f * M + mk) * 3;
    const double sim[3] = {double(s[0]), double(s[1]), double(s[2])};
    err[i] = mosh2::heldout_error(sim, side + 3 * i, (status[f] & mosh2::ST_SOLVED) != 0);
}

// Host copy of a model description: the caller's buffers need not outlive mosh2_model_create, and the device copy of a
// precision is only built when the first job of that precision is created.
struct HostDesc {
    mosh2_model_desc d{};
    std::vector<int32_t> parents, w_joint, free1, free2, prior_ids, jangles_ids;
    std::vector<double> jangles_signs;
    std::vector<double> hand_comps, hands_mean, v0, sd, pd, w_val, j0, jd, coefs, prior_means, prior_Q, prior_neglogw;
    template <class T> static const T *keep(std::vector<T> &dst, const T *src, size_t n) {
        dst.assign(src, src + n);
        if (dst.empty()) dst.resize(1);
        return dst.data();
    }
    void copy_from(const mosh2_model_desc &s) {
        d = s;
        const size_t nJ = s.n_joints, S = size_t(3) * s.n_markers, nd = s.n_dmpl, K = s.prior_k, D = s.prior_d;
        d.parents = keep(parents, s.parents, nJ);
        d.w_joint = keep(w_joint, s.w_joint, S * s.kw);
        d.free1 = keep(free1, s.free1, s.n_free1);
        d.free2 = keep(free2, s.free2, s.n_free2);
        if (s.prior_ids) d.prior_ids = keep(prior_ids, s.prior_ids, D);
        if (s.n_jangles > 0) { d.jangles_ids = keep(jangles_ids, s.jangles_ids, s.n_jangles); d.jangles_signs = keep(jangles_signs, s.jangles_signs, s.n_jangles); }
        d.hand_comps = keep(hand_comps, s.hand_comps, size_t(s.n_hand_red) * s.n_hand_full);
        d.hands_mean = keep(hands_mean, s.hands_mean, s.n_hand_full);
        d.v0 = keep(v0, s.v0, S * 3);
        d.sd = keep(sd, s.sd, S * 3 * nd);
        d.pd = keep(pd, s.pd, (nJ - 1) * 3 * S * 9);
        d.w_val = keep(w_val, s.w_val, S * s.kw);
        d.j0 = keep(j0, s.j0, nJ * 3);
        d.jd = keep(jd, s.jd, nJ * 3 * nd);
        d.coefs = keep(coefs, s.coefs, size_t(s.n_markers) * 3);
        d.prior_means = keep(prior_means, s.prior_means, K * D);
        d.prior_Q = keep(prior_Q, s.prior_Q, K * D * D);
        d.prior_neglogw = keep(prior_neglogw, s.prior_neglogw, K);
    }
};

struct mosh2_model {
    int device = 0;
    HostDesc host;
    DevModel<float> f32;
    DevModel<double> f64;
    bool have_f32 = false, have_f64 = false;
    int n_joints = 0, n_markers = 0, p_red = 0, n_dmpl = 0;
    int ensure(int precision) {
        if (precision == MOSH2_F64) {
            if (!have_f64) { f64.device = device; const int rc = f64.build(host.d); if (rc) return rc; have_f64 = true; }
        } else if (!have_f32) { f32.device = device; const int rc = f32.build(host.d); if (rc) return rc; have_f32 = true; }
        return 0;
    }
};

struct mosh2_job {
    mosh2_model *model = nullptr;
    int precision = MOSH2_F32;
    int n_frames = 0, n_chunks = 1;
    int *d_chunk_tab = nullptr, *d_chunk_ids = nullptr, *d_warm_f = nullptr;
    void *d_warm_x = nullptr;
    float *d_delta = nullptr;
    std::vector<int> tab, tab0;       // host copy of the chunk table (tab0: as created; repairs edit tab)
    bool tab_dirty = false;
    double merge_tol = 0;
    int launch_blocks = 0;            // blocks of the next launch (all chunks, or the subset in d_chunk_ids)
    bool subset = false;
    mosh2::Options opt{};
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_in = nullptr;
    size_t esz = 4;                 // element size of the compute type
    size_t smem = 0, gws_stride = 0;
    int big_in_global = 0;
    // device buffers
    void *d_obs = nullptr, *d_out = nullptr, *d_gws = nullptr;
    uint8_t *d_vis = nullptr;
    int *d_status = nullptr, *d_counters = nullptr, *d_totals = nullptr;
    long long *d_prof = nullptr;
    // pinned staging
    void *h_obs = nullptr, *h_out = nullptr;
    uint8_t *h_vis = nullptr;
    void *d_lin = nullptr;                       // linearise mode: states in, normal equations / Jacobian rows / residuals out
    size_t lin_bytes = 0;
    int lin_mode = 0, lin_step = 1;
    mosh2_host::LinLayout lin{};                 // layout of d_lin for the current call
    // mosh2_job_upload_markers[_range]: one staging slot per upload in flight.  A slot holds the table rows, the rotation and
    // the column map (pinned, and their device copy); `done` is recorded behind the gather kernel that reads them, and a
    // slot is only refilled once its event has completed, so uploads of several captures can be queued back to back.
    struct RangeSlot { void *h = nullptr, *d = nullptr; size_t bytes = 0; cudaEvent_t done = nullptr; };
    std::vector<RangeSlot> range_slots;
    std::vector<int> counts;                     // frames of every sequence of the job
    // the last mosh2_job_upload_markers_folds: its folds (first frame, frames per fold, count, most hidden markers K), the side
    // buffer [n_folds][n][K][3] (float64), the hidden markers [n_folds][K], and the errors and status of mosh2_job_heldout_errors
    int fold_frame0 = 0, fold_n = 0, fold_count = 0, fold_K = 0;
    double *d_fold_side = nullptr, *d_fold_err = nullptr;
    int *d_fold_idx = nullptr, *d_fold_status = nullptr;
    int *h_status = nullptr, *h_counters = nullptr;
    // multi-model job (mosh2_job_create_multi; `model` is models[0]): the Model records of the job's precision as the kernel
    // reads them (host copy, whose first record also carries the job's workspace plan, and device array), and the model
    // index of every chunk -- an array of its own, the chunk records are rewritten in place by mosh2_job_relaunch_chunks
    std::vector<mosh2_model *> models;
    std::vector<unsigned char> h_models;
    void *d_models = nullptr;
    int *d_model_of_chunk = nullptr;
    std::vector<int> model_of_frame;             // multi-model job: model index of every frame (sequence sweeps)
    int *d_model_of_frame = nullptr;
    // sequence sweep (mosh2_job_sequence_sweep): neighbour table, the frames of the three colours back to back, per-frame deltas;
    // `seq_ids` points at the frames of the current launch.  gws_slots: per-CTA global workspaces allocated (BIG layout).
    int *d_seq_nbr = nullptr, *d_seq_ids = nullptr;
    const int *seq_ids = nullptr;
    double *d_seq_delta = nullptr;
    size_t gws_slots = 0;
    bool ev0_held = false;                       // a sweep times its three launches as one
    bool launched = false;                       // mosh2_job_launch has run: status and rows hold a solve (a sweep needs them)
    size_t n_obs = 0, n_out = 0;
    size_t o_fullpose = 0, o_pose = 0, o_trans = 0, o_dmpls = 0, o_mk = 0, o_errs = 0;   // element offsets in d_out
};

namespace {

template <class real, bool BIG, bool SWEEP>
cudaError_t launch_kernel(mosh2_job *j, const mosh2::Model<real> &m, const mosh2::Job<real> &job, int threads) {
    const mosh2_host::Layout<real, BIG> L = mosh2_host::layout<real, BIG>(m, mosh2::kSmemHeader);
    const cudaError_t e = cudaFuncSetAttribute(mosh2_stageii_kernel<real, BIG, SWEEP>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(j->smem));
    if (e != cudaSuccess) return e;
    mosh2_stageii_kernel<real, BIG, SWEEP><<<j->launch_blocks, threads, j->smem, j->stream>>>(m, job, L.w, L.d);
    return cudaGetLastError();
}

template <class real, bool BIG, bool SWEEP>
cudaError_t launch_multi_kernel(mosh2_job *j, const mosh2::Job<real> &job, int threads) {
    const mosh2::Model<real> &m = *reinterpret_cast<const mosh2::Model<real> *>(j->h_models.data());
    const mosh2_host::Layout<real, BIG> L = mosh2_host::layout<real, BIG>(m, mosh2_host::multi_smem_header<real>());
    const cudaError_t e = cudaFuncSetAttribute(mosh2_stageii_multi_kernel<real, BIG, SWEEP>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(j->smem));
    if (e != cudaSuccess) return e;
    mosh2_stageii_multi_kernel<real, BIG, SWEEP><<<j->launch_blocks, threads, j->smem, j->stream>>>(
        static_cast<const mosh2::Model<real> *>(j->d_models), j->lin_mode == 3 ? j->d_model_of_frame : j->d_model_of_chunk, job, L.w, L.d);
    return cudaGetLastError();
}

template <class real>
int launch(mosh2_job *j, const mosh2::Model<real> &m) {
    mosh2::Job<real> job{};
    job.n_frames = j->n_frames; job.n_chunks = j->n_chunks;
    job.chunk_tab = j->d_chunk_tab; job.chunk_ids = j->subset ? j->d_chunk_ids : nullptr;
    job.warm_x = static_cast<real *>(j->d_warm_x); job.warm_f = j->d_warm_f; job.merge_tol = j->merge_tol;
    job.obs = static_cast<const real *>(j->d_obs);
    job.vis = j->d_vis;
    real *out = static_cast<real *>(j->d_out);
    job.fullpose = out + j->o_fullpose; job.pose = out + j->o_pose; job.trans = out + j->o_trans;
    job.dmpls = j->model->n_dmpl ? out + j->o_dmpls : nullptr;
    job.markers_sim = out + j->o_mk; job.errs = out + j->o_errs;
    job.status = j->d_status; job.counters = j->d_counters; job.totals = j->d_totals; job.prof = j->d_prof;
    job.gws = static_cast<char *>(j->d_gws); job.gws_stride = j->gws_stride;
    job.lin_mode = j->lin_mode; job.lin_step = j->lin_step;
    if (j->lin_mode == 1 || j->lin_mode == 2) mosh2_host::bind_lin(job, static_cast<real *>(j->d_lin), j->lin);
    if (j->lin_mode == 3) {                      // sequence sweep: one block per frame of the colour; no chunk records
        job.chunk_ids = j->seq_ids;
        job.seq_nbr = j->d_seq_nbr; job.seq_delta = j->d_seq_delta;
        job.warm_x = nullptr; job.warm_f = nullptr;
    }
    job.opt = j->opt;
    int threads = threads_for<real>();
    if (const char *e = getenv("MOSH2_DEV_THREADS")) {      // development aid: any multiple of 32 from 128 up to the launch bound
        const int t = atoi(e);
        if (t >= 128 && t <= threads && t % 32 == 0) threads = t;
    }
    if (!j->ev0_held) CU(cudaEventRecord(j->ev0, j->stream));
    const bool sweep = j->lin_mode == 3;         // (the sequence sweep is a kernel of its own: the causal one is compiled without it)
    if (j->d_models) {
        if (sweep) CU(j->big_in_global ? (launch_multi_kernel<real, true, true>(j, job, threads)) : (launch_multi_kernel<real, false, true>(j, job, threads)));
        else if (j->big_in_global) CU((launch_multi_kernel<real, true, false>(j, job, threads)));
        else CU((launch_multi_kernel<real, false, false>(j, job, threads)));
    } else if (sweep) CU(j->big_in_global ? (launch_kernel<real, true, true>(j, m, job, threads)) : (launch_kernel<real, false, true>(j, m, job, threads)));
    else if (j->big_in_global) CU((launch_kernel<real, true, false>(j, m, job, threads)));
    else CU((launch_kernel<real, false, false>(j, m, job, threads)));
    CU(cudaGetLastError());
    CU(cudaEventRecord(j->ev1, j->stream));
    return 0;
}

// mosh2_job_linearize in the job's compute type: the caller's float64 states are rounded to `real` on the way in, every
// output is widened to the float64 buffers of mosh2_lin_out on the way out
template <class real>
int linearize(mosh2_job *j, const mosh2::Model<real> &m, int32_t step, int32_t build, const double *x, const mosh2_lin_out *out) {
    const size_t F = j->n_frames, M = j->model->n_markers, NX = 3 + j->model->p_red + j->model->n_dmpl;
    const size_t n = step == 2 ? m.n2 : m.n1;
    const size_t words = mosh2_host::lin_layout(F, M, NX, std::max(m.n1, m.n2)).words;      // room for either step
    if (words * sizeof(real) > j->lin_bytes) {
        g_blocks.put(j->model->device, j->d_lin);
        j->d_lin = nullptr; j->lin_bytes = 0;
        CU(g_blocks.get(j->model->device, words * sizeof(real), &j->d_lin));
        j->lin_bytes = words * sizeof(real);
    }
    const std::vector<real> xr(x, x + F * NX);      // (alive until the stream is synchronised below)
    CU(cudaMemcpyAsync(j->d_lin, xr.data(), F * NX * sizeof(real), cudaMemcpyHostToDevice, j->stream));
    CU(cudaMemsetAsync(j->d_out, 0, j->n_out * j->esz, j->stream));
    j->lin_mode = build ? 2 : 1;
    j->lin_step = step;
    j->lin = mosh2_host::lin_layout(F, M, NX, n);
    j->subset = false;
    j->launch_blocks = int(F);
    const int rc = launch<real>(j, m);
    j->lin_mode = 0;
    j->launch_blocks = j->n_chunks;
    if (rc) return rc;
    const real *p = static_cast<const real *>(j->d_lin), *dA = p + j->lin.A, *dg = p + j->lin.g, *dJ = p + j->lin.J;
    const real *dr = p + j->lin.r, *dvp = p + j->lin.vp;
    const real *dout = static_cast<const real *>(j->d_out);
    struct Back { double *dst; const real *src; size_t cnt; std::vector<real> h; };
    Back b[7] = {{out->r, dr, F * 3 * M, {}}, {out->vp, dvp, F * 9 * M, {}}, {out->errs, dout + j->o_errs, F * mosh2::N_ERR, {}},
                 {out->markers_sim, dout + j->o_mk, F * 3 * M, {}}, {build ? out->A : nullptr, dA, F * n * n, {}},
                 {build ? out->g : nullptr, dg, F * n, {}}, {build ? out->J : nullptr, dJ, F * 3 * M * n, {}}};
    for (Back &e : b) {
        if (!e.dst) continue;
        e.h.resize(e.cnt);
        CU(cudaMemcpyAsync(e.h.data(), e.src, e.cnt * sizeof(real), cudaMemcpyDeviceToHost, j->stream));
    }
    CU(cudaStreamSynchronize(j->stream));
    for (const Back &e : b)
        if (e.dst) for (size_t i = 0; i < e.cnt; ++i) e.dst[i] = double(e.h[i]);
    return 0;
}

// A staging slot of at least `total` bytes (pinned host memory and its device twin) whose last copy and kernel have finished.
int staging_slot(mosh2_job *j, size_t total, mosh2_job::RangeSlot **out) {
    const int dv = j->model->device;
    mosh2_job::RangeSlot *slot = nullptr, *idle = nullptr;
    for (auto &s : j->range_slots) {
        const cudaError_t q = cudaEventQuery(s.done);
        if (q == cudaErrorNotReady) continue;
        CU(q);
        if (s.bytes >= total) { slot = &s; break; }
        if (!idle) idle = &s;
    }
    if (!slot) {
        if (!idle) {
            j->range_slots.emplace_back();
            idle = &j->range_slots.back();
            CU(cudaEventCreateWithFlags(&idle->done, cudaEventDisableTiming));
        }
        slot = idle;
        g_blocks.put(-1, slot->h); g_blocks.put(dv, slot->d);
        slot->h = slot->d = nullptr; slot->bytes = 0;
        CU(g_blocks.get(-1, total, &slot->h));
        CU(g_blocks.get(dv, total, &slot->d));
        slot->bytes = total;
    }
    *out = slot;
    return 0;
}

// Per-CTA global workspaces a BIG-layout sweep launch may use: two thread blocks per SM of an H100 SXM (132 SMs).  A colour with
// more frames runs in launches of this many blocks; the job's own workspaces (one per chunk) are used if there are more of them.
constexpr size_t kSweepGwsSlots = 2 * 132;

// mosh2_job_sequence_sweep in the job's compute type: the neighbour table and the colours from the status of the last launch,
// then one launch per colour (in batches of the per-CTA global workspaces there are, in the BIG layout), then the deltas
template <class real>
int sequence_sweep(mosh2_job *j, const mosh2::Model<real> &m, double *max_delta) {
    const int F = j->n_frames, dv = j->model->device;
    if (!j->d_seq_nbr) {
        CU(g_blocks.get(dv, size_t(F) * 4 * sizeof(int), reinterpret_cast<void **>(&j->d_seq_nbr)));
        CU(g_blocks.get(dv, size_t(F) * sizeof(int), reinterpret_cast<void **>(&j->d_seq_ids)));
        CU(g_blocks.get(dv, size_t(F) * 4 * sizeof(double), reinterpret_cast<void **>(&j->d_seq_delta)));
    }
    CU(cudaMemcpyAsync(j->h_status, j->d_status, size_t(F) * sizeof(int), cudaMemcpyDeviceToHost, j->stream));
    CU(cudaStreamSynchronize(j->stream));
    std::vector<int> nbr, colour[3];
    mosh2_host::sequence_tables(j->h_status, F, j->tab0, nbr, colour);
    std::vector<int> ids;
    size_t widest = 0;
    for (const auto &c : colour) { ids.insert(ids.end(), c.begin(), c.end()); widest = std::max(widest, c.size()); }
    CU(cudaMemcpy(j->d_seq_nbr, nbr.data(), nbr.size() * sizeof(int), cudaMemcpyHostToDevice));
    if (!ids.empty()) CU(cudaMemcpy(j->d_seq_ids, ids.data(), ids.size() * sizeof(int), cudaMemcpyHostToDevice));
    CU(cudaMemsetAsync(j->d_seq_delta, 0, size_t(F) * 4 * sizeof(double), j->stream));
    size_t slots = widest;
    if (j->gws_stride) {                         // BIG layout: one global workspace per block of a launch
        slots = std::max(j->gws_slots, std::min(widest, kSweepGwsSlots));
        if (slots > j->gws_slots) {
            g_blocks.put(dv, j->d_gws);
            j->d_gws = nullptr; j->gws_slots = 0;
            CU(g_blocks.get(dv, j->gws_stride * slots, &j->d_gws));
            j->gws_slots = slots;
        }
    }
    j->lin_mode = 3;
    int rc = 0;
    size_t off = 0;
    for (int c = 0; c < 3 && !rc; ++c) {
        for (size_t b = 0; b < colour[c].size() && !rc; b += slots) {
            j->seq_ids = j->d_seq_ids + off + b;
            j->launch_blocks = int(std::min(slots, colour[c].size() - b));
            rc = launch<real>(j, m);
            j->ev0_held = true;
        }
        off += colour[c].size();
    }
    j->lin_mode = 0; j->ev0_held = false; j->seq_ids = nullptr; j->launch_blocks = j->n_chunks;
    if (rc) return rc;
    std::vector<double> dl(size_t(F) * 4);
    CU(cudaMemcpyAsync(dl.data(), j->d_seq_delta, dl.size() * sizeof(double), cudaMemcpyDeviceToHost, j->stream));
    CU(cudaStreamSynchronize(j->stream));
    if (max_delta) {
        for (int q = 0; q < 4; ++q) max_delta[q] = 0;
        for (int f = 0; f < F; ++f)
            for (int q = 0; q < 4; ++q) max_delta[q] = std::max(max_delta[q], dl[size_t(f) * 4 + q]);
    }
    return 0;
}

}  // namespace

extern "C" {

int mosh2_version(void) { return MOSH2_VERSION; }
const char *mosh2_last_error(void) { return g_err.c_str(); }

int mosh2_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

void mosh2_default_options(mosh2_options *o) {
    if (!o) return;
    // support_data/conf/moshpp_conf.yaml:99,118-125; chmosh.py:460,653,671,697
    o->wt_data = 400; o->wt_poseB = 1.6; o->wt_poseH = 1.0; o->wt_velo = 2.5; o->wt_dmpl = 1.0;
    o->wt_annealing = 2.5; o->wt_extrap_dmpl = 6.0; o->num_train_markers = 46;
    o->delta_0 = 0.5; o->e3_first = 1e-3; o->e3 = 1e-2; o->maxiter = 100;
    o->optimize_fingers = 0; o->optimize_dynamics = 0;
    o->wt_poseF = 1.0; o->wt_expr = 1.0; o->optimize_face = 0;
    o->robust_sigma = 0;       // the reference's least-squares data term
}

int mosh2_model_create(const mosh2_model_desc *d, int device, mosh2_model **out) {
    if (!d || !out) return fail(MOSH2_E_INVALID, "null argument");
    *out = nullptr;
    std::string msg;
    if (const int rc = mosh2_host::check_model_desc(*d, &msg)) return fail(rc, "%s", msg.c_str());
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(MOSH2_E_NO_DEVICE, "no CUDA device: libmosh2 has no CPU path");
    }
    if (device < 0 || device >= ndev) return fail(MOSH2_E_INVALID, "device %d out of range (%d devices)", device, ndev);
    CU(cudaSetDevice(device));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(MOSH2_E_NO_DEVICE, "device %d is sm_%d%d; libmosh2 is built for sm_90a only", device, prop.major, prop.minor);
    mosh2_model *m = new (std::nothrow) mosh2_model;
    if (!m) return fail(MOSH2_E_INVALID, "out of host memory");
    m->device = device; m->n_joints = d->n_joints; m->n_markers = d->n_markers; m->p_red = d->p_red; m->n_dmpl = d->n_dmpl;
    m->host.copy_from(*d);      // the device copy of a precision is built by the first job that asks for it
    *out = m;
    return 0;
}

void mosh2_model_destroy(mosh2_model *m) {
    if (!m) return;
    cudaSetDevice(m->device);
    delete m;
}

int mosh2_job_create(mosh2_model *m, const mosh2_options *opt, int32_t n_frames, const mosh2_schedule *sched,
                     int32_t precision, mosh2_job **out) {
    return mosh2_job_create_batch(m, opt, 1, &n_frames, sched, precision, out);
}

int mosh2_job_create_batch(mosh2_model *m, const mosh2_options *opt, int32_t n_seq, const int32_t *frame_counts,
                           const mosh2_schedule *sched, int32_t precision, mosh2_job **out) {
    if (!m || !opt || !out || n_seq < 1 || !frame_counts) return fail(MOSH2_E_INVALID, "bad argument");
    long long total = 0;
    for (int q = 0; q < n_seq; ++q) {
        if (frame_counts[q] < 1) return fail(MOSH2_E_INVALID, "sequence %d has %d frames", q, frame_counts[q]);
        total += frame_counts[q];
    }
    if (total > 0x3fffffff) return fail(MOSH2_E_TOO_LARGE, "%lld frames in one job", total);
    const int32_t n_frames = int32_t(total);
    if (precision != MOSH2_F32 && precision != MOSH2_F64) return fail(MOSH2_E_INVALID, "precision must be MOSH2_F32 or MOSH2_F64");
    if (!mosh2_host::robust_sigma_ok(*opt)) return fail(MOSH2_E_INVALID, "robust_sigma must be 0 (off) or a finite sigma > 0");
    *out = nullptr;
    CU(cudaSetDevice(m->device));
    if (const int rc = m->ensure(precision)) return rc;
    mosh2_job *j = new (std::nothrow) mosh2_job;
    if (!j) return fail(MOSH2_E_INVALID, "out of host memory");
    j->model = m; j->precision = precision; j->n_frames = n_frames;
    j->counts.assign(frame_counts, frame_counts + n_seq);
    j->tab = mosh2_host::schedule_table(sched, frame_counts, n_seq);
    j->tab0 = j->tab;
    const std::vector<int> &tab = j->tab;
    j->n_chunks = int(tab.size() / mosh2::kChunkRec);
    j->launch_blocks = j->n_chunks;
    j->esz = precision == MOSH2_F64 ? 8 : 4;
    j->opt = mosh2_host::to_options(*opt);

    size_t gws = 0;
    if (precision == MOSH2_F64) plan_workspace(m->f64.m, &j->smem, &gws, &j->big_in_global);
    else plan_workspace(m->f32.m, &j->smem, &gws, &j->big_in_global);
    if (j->smem > kMaxSmem) {
        const size_t need = j->smem;
        delete j;
        return fail(MOSH2_E_TOO_LARGE, "model needs %zu bytes of shared memory per block (max %zu)", need, kMaxSmem);
    }
    j->gws_stride = j->big_in_global ? gws : 0;

    const size_t F = n_frames, M = m->n_markers, PF = size_t(3) * m->n_joints, PR = m->p_red, nd = m->n_dmpl;
    j->n_obs = F * M * 3;
    size_t off = 0;
    j->o_fullpose = off; off += F * PF;
    j->o_pose = off; off += F * PR;
    j->o_trans = off; off += F * 3;
    j->o_dmpls = off; off += F * nd;
    j->o_mk = off; off += F * M * 3;
    j->o_errs = off; off += F * mosh2::N_ERR;
    j->n_out = off;
    cudaError_t e = cudaSuccess;
    auto chk = [&](cudaError_t r) { if (e == cudaSuccess) e = r; };
    chk(cudaStreamCreateWithFlags(&j->stream, cudaStreamNonBlocking));
    chk(cudaEventCreate(&j->ev0));
    chk(cudaEventCreate(&j->ev1));
    chk(cudaEventCreateWithFlags(&j->ev_in, cudaEventDisableTiming));
    chk(g_blocks.get(m->device, j->n_obs * j->esz, reinterpret_cast<void **>(&j->d_obs)));
    chk(g_blocks.get(m->device, j->n_out * j->esz, reinterpret_cast<void **>(&j->d_out)));
    chk(g_blocks.get(m->device, F * M, reinterpret_cast<void **>(&j->d_vis)));
    chk(g_blocks.get(m->device, F * sizeof(int), reinterpret_cast<void **>(&j->d_status)));
    chk(g_blocks.get(m->device, F * 4 * sizeof(int), reinterpret_cast<void **>(&j->d_counters)));
    chk(g_blocks.get(m->device, 8 * sizeof(int), reinterpret_cast<void **>(&j->d_totals)));
    chk(g_blocks.get(m->device, tab.size() * sizeof(int), reinterpret_cast<void **>(&j->d_chunk_tab)));
    chk(g_blocks.get(m->device, size_t(j->n_chunks) * sizeof(int), reinterpret_cast<void **>(&j->d_chunk_ids)));
    chk(g_blocks.get(m->device, size_t(j->n_chunks) * sizeof(int), reinterpret_cast<void **>(&j->d_warm_f)));
    chk(g_blocks.get(m->device, size_t(j->n_chunks) * 4 * sizeof(float), reinterpret_cast<void **>(&j->d_delta)));
    chk(g_blocks.get(m->device, size_t(j->n_chunks) * (3 + m->p_red + m->n_dmpl) * j->esz, reinterpret_cast<void **>(&j->d_warm_x)));
    if (e == cudaSuccess) chk(cudaMemcpy(j->d_chunk_tab, tab.data(), tab.size() * sizeof(int), cudaMemcpyHostToDevice));
    chk(g_blocks.get(m->device, 32 * sizeof(long long), reinterpret_cast<void **>(&j->d_prof)));
    if (j->gws_stride) chk(g_blocks.get(m->device, j->gws_stride * j->n_chunks, reinterpret_cast<void **>(&j->d_gws)));
    j->gws_slots = size_t(j->n_chunks);
    chk(g_blocks.get(-1, j->n_obs * j->esz, reinterpret_cast<void **>(&j->h_obs)));
    chk(g_blocks.get(-1, j->n_out * j->esz, reinterpret_cast<void **>(&j->h_out)));
    chk(g_blocks.get(-1, F * M, reinterpret_cast<void **>(&j->h_vis)));
    chk(g_blocks.get(-1, F * sizeof(int), reinterpret_cast<void **>(&j->h_status)));
    chk(g_blocks.get(-1, F * 4 * sizeof(int), reinterpret_cast<void **>(&j->h_counters)));
    if (e != cudaSuccess) {
        mosh2_job_destroy(j);
        return fail(MOSH2_E_CUDA, "job allocation failed: %s", cudaGetErrorString(e));
    }
    *out = j;
    return 0;
}

}  // extern "C"

namespace {

// mosh2_job_create_multi in the job's compute type, on a batch job `j` of models[0]: the shape check, the workspace plan
// with the Model record in the shared-memory header, and the device arrays of Model records and chunk -> model indices
template <class real>
int make_multi(mosh2_job *j, mosh2_model *const *models, int32_t n_models, int32_t n_seq, const int32_t *frame_counts,
               const int32_t *model_of_seq) {
    auto dev_model = [](mosh2_model *mm) -> mosh2::Model<real> & {
        if constexpr (sizeof(real) == 8) return mm->f64.m; else return mm->f32.m;
    };
    mosh2::Model<real> plan = dev_model(models[0]);
    size_t smem = 0, gws = 0;
    int big = 0;
    plan_workspace(plan, &smem, &gws, &big, mosh2_host::multi_smem_header<real>());
    if (smem > kMaxSmem) return fail(MOSH2_E_TOO_LARGE, "model needs %zu bytes of shared memory per block (max %zu)", smem, kMaxSmem);
    const int dv = j->model->device;
    const size_t stride = big ? gws : 0;
    if (stride > j->gws_stride) {
        g_blocks.put(dv, j->d_gws);
        j->d_gws = nullptr;
        CU(g_blocks.get(dv, stride * j->n_chunks, &j->d_gws));
    }
    j->smem = smem; j->big_in_global = big; j->gws_stride = stride;
    j->gws_slots = size_t(j->n_chunks);
    std::vector<mosh2::Model<real>> recs(n_models);
    for (int k = 0; k < n_models; ++k) {
        recs[k] = dev_model(models[k]);
        recs[k].tile_markers = plan.tile_markers;
    }
    j->h_models.assign(reinterpret_cast<const unsigned char *>(recs.data()), reinterpret_cast<const unsigned char *>(recs.data() + n_models));
    const std::vector<int> moc = mosh2_host::model_of_chunks(j->tab0, frame_counts, n_seq, model_of_seq);
    CU(g_blocks.get(dv, j->h_models.size(), &j->d_models));
    CU(g_blocks.get(dv, moc.size() * sizeof(int), reinterpret_cast<void **>(&j->d_model_of_chunk)));
    CU(cudaMemcpy(j->d_models, j->h_models.data(), j->h_models.size(), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(j->d_model_of_chunk, moc.data(), moc.size() * sizeof(int), cudaMemcpyHostToDevice));
    j->model_of_frame.clear();
    for (int q = 0; q < n_seq; ++q) j->model_of_frame.insert(j->model_of_frame.end(), size_t(frame_counts[q]), model_of_seq[q]);
    CU(g_blocks.get(dv, j->model_of_frame.size() * sizeof(int), reinterpret_cast<void **>(&j->d_model_of_frame)));
    CU(cudaMemcpy(j->d_model_of_frame, j->model_of_frame.data(), j->model_of_frame.size() * sizeof(int), cudaMemcpyHostToDevice));
    j->models.assign(models, models + n_models);
    return 0;
}

}  // namespace

extern "C" {

int mosh2_job_create_multi(mosh2_model *const *models, int32_t n_models, const mosh2_options *opt, int32_t n_seq,
                           const int32_t *frame_counts, const int32_t *model_of_seq, const mosh2_schedule *sched,
                           int32_t precision, mosh2_job **out) {
    if (!models || n_models < 1 || !opt || !out || n_seq < 1 || !frame_counts || !model_of_seq) return fail(MOSH2_E_INVALID, "bad argument");
    if (precision != MOSH2_F32 && precision != MOSH2_F64) return fail(MOSH2_E_INVALID, "precision must be MOSH2_F32 or MOSH2_F64");
    *out = nullptr;
    for (int k = 0; k < n_models; ++k) {
        if (!models[k]) return fail(MOSH2_E_INVALID, "model %d is NULL", k);
        if (models[k]->device != models[0]->device)
            return fail(MOSH2_E_INVALID, "model %d is on device %d, model 0 on device %d", k, models[k]->device, models[0]->device);
    }
    for (int q = 0; q < n_seq; ++q)
        if (model_of_seq[q] < 0 || model_of_seq[q] >= n_models)
            return fail(MOSH2_E_INVALID, "sequence %d refers to model %d of %d", q, model_of_seq[q], n_models);
    CU(cudaSetDevice(models[0]->device));
    for (int k = 0; k < n_models; ++k)
        if (const int rc = models[k]->ensure(precision)) return rc;
    for (int k = 1; k < n_models; ++k) {
        const char *field = precision == MOSH2_F64 ? mosh2_host::kernel_shape_mismatch(models[0]->f64.m, models[k]->f64.m)
                                                   : mosh2_host::kernel_shape_mismatch(models[0]->f32.m, models[k]->f32.m);
        if (field) return fail(MOSH2_E_INVALID, "model %d does not have the kernel shape of model 0: %s differs", k, field);
    }
    mosh2_job *j = nullptr;
    if (const int rc = mosh2_job_create_batch(models[0], opt, n_seq, frame_counts, sched, precision, &j)) return rc;
    const int rc = precision == MOSH2_F64 ? make_multi<double>(j, models, n_models, n_seq, frame_counts, model_of_seq)
                                          : make_multi<float>(j, models, n_models, n_seq, frame_counts, model_of_seq);
    if (rc) {
        const std::string msg = g_err;
        mosh2_job_destroy(j);
        g_err = msg;
        return rc;
    }
    *out = j;
    return 0;
}

int mosh2_job_upload(mosh2_job *j, const double *obs, const uint8_t *vis) {
    if (!j || !obs || !vis) return fail(MOSH2_E_INVALID, "null argument");
    CU(cudaSetDevice(j->model->device));
    if (j->precision == MOSH2_F64) memcpy(j->h_obs, obs, j->n_obs * sizeof(double));
    else {
        float *h = static_cast<float *>(j->h_obs);
        for (size_t i = 0; i < j->n_obs; ++i) h[i] = float(obs[i]);
    }
    const size_t nv = size_t(j->n_frames) * j->model->n_markers;
    memcpy(j->h_vis, vis, nv);
    CU(cudaMemcpyAsync(j->d_obs, j->h_obs, j->n_obs * j->esz, cudaMemcpyHostToDevice, j->stream));
    CU(cudaMemcpyAsync(j->d_vis, j->h_vis, nv, cudaMemcpyHostToDevice, j->stream));
    return 0;
}

int mosh2_job_upload_markers(mosh2_job *j, const double *markers, int32_t n_file_frames, int32_t n_cols, const int32_t *col_of_marker,
                             int32_t frame_start, int32_t frame_step, double unit_per_metre, const double *rot3x3) {
    if (!j) return fail(MOSH2_E_INVALID, "null argument");
    return mosh2_job_upload_markers_range(j, 0, j->n_frames, markers, n_file_frames, n_cols, col_of_marker, frame_start, frame_step,
                                          unit_per_metre, rot3x3);
}

int mosh2_job_upload_markers_range(mosh2_job *j, int32_t frame0, int32_t nfr, const double *markers, int32_t n_file_frames, int32_t n_cols,
                                   const int32_t *col_of_marker, int32_t frame_start, int32_t frame_step, double unit_per_metre,
                                   const double *rot3x3) {
    if (!j) return fail(MOSH2_E_INVALID, "null argument");
    const int M = j->model->n_markers;
    std::string msg;
    if (const int rc = mosh2_host::check_marker_range(j->n_frames, M, frame0, nfr, markers, n_file_frames, n_cols, col_of_marker, frame_start,
                                                      frame_step, unit_per_metre, &msg))
        return fail(rc, "%s", msg.c_str());
    CU(cudaSetDevice(j->model->device));
    // slot layout: rows [frame_start, last used frame] of the table (all columns) | rotation (9) | column map (M int32)
    const size_t rows = size_t(nfr - 1) * frame_step + 1, bytes = rows * n_cols * 3 * sizeof(double);
    const size_t o_cols = bytes + 9 * sizeof(double), total = o_cols + size_t(M) * sizeof(int32_t);
    mosh2_job::RangeSlot *slot = nullptr;
    if (const int rc = staging_slot(j, total, &slot)) return rc;
    char *h = static_cast<char *>(slot->h);
    memcpy(h, markers + size_t(frame_start) * n_cols * 3, bytes);
    if (rot3x3) memcpy(h + bytes, rot3x3, 9 * sizeof(double));
    memcpy(h + o_cols, col_of_marker, size_t(M) * sizeof(int32_t));
    CU(cudaMemcpyAsync(slot->d, h, total, cudaMemcpyHostToDevice, j->stream));
    const char *d = static_cast<const char *>(slot->d);
    const double *d_table = reinterpret_cast<const double *>(d), *d_rot = rot3x3 ? reinterpret_cast<const double *>(d + bytes) : nullptr;
    const int *d_cols = reinterpret_cast<const int *>(d + o_cols);
    const size_t n = size_t(nfr) * M, o0 = size_t(frame0) * M;
    const int blocks = int((n + 255) / 256);
    if (j->precision == MOSH2_F64)
        gather_markers_kernel<double><<<blocks, 256, 0, j->stream>>>(d_table, n_cols, d_cols, M, nfr, frame_step, unit_per_metre, d_rot,
                                                                     static_cast<double *>(j->d_obs) + 3 * o0, j->d_vis + o0);
    else
        gather_markers_kernel<float><<<blocks, 256, 0, j->stream>>>(d_table, n_cols, d_cols, M, nfr, frame_step, unit_per_metre, d_rot,
                                                                    static_cast<float *>(j->d_obs) + 3 * o0, j->d_vis + o0);
    CU(cudaGetLastError());
    CU(cudaEventRecord(slot->done, j->stream));
    return 0;
}

int mosh2_job_upload_markers_folds(mosh2_job *j, int32_t seq0, int32_t n_folds, const double *markers, int32_t n_file_frames,
                                   int32_t n_cols, const int32_t *col_of_marker, const uint8_t *hide, int32_t frame_start,
                                   int32_t frame_step, double unit_per_metre, const double *rot3x3) {
    if (!j) return fail(MOSH2_E_INVALID, "null argument");
    const int M = j->model->n_markers;
    std::string msg;
    if (const int rc = mosh2_host::check_marker_folds(j->counts, M, seq0, n_folds, hide, markers, n_file_frames, n_cols, col_of_marker,
                                                      frame_start, frame_step, unit_per_metre, &msg))
        return fail(rc, "%s", msg.c_str());
    CU(cudaSetDevice(j->model->device));
    const int dv = j->model->device, n = j->counts[seq0];
    int frame0 = 0;
    for (int q = 0; q < seq0; ++q) frame0 += j->counts[q];
    std::vector<int> slot_of, idx;
    const int K = mosh2_host::fold_slots(hide, n_folds, M, slot_of, idx);
    // the fold buffers are replaced once the stream has finished with the previous ones
    CU(cudaStreamSynchronize(j->stream));
    for (void *p : {static_cast<void *>(j->d_fold_side), static_cast<void *>(j->d_fold_err), static_cast<void *>(j->d_fold_idx),
                    static_cast<void *>(j->d_fold_status)})
        g_blocks.put(dv, p);
    j->d_fold_side = j->d_fold_err = nullptr; j->d_fold_idx = j->d_fold_status = nullptr; j->fold_count = 0;
    const size_t nfk = size_t(n_folds) * n * K;
    CU(g_blocks.get(dv, nfk * 3 * sizeof(double), reinterpret_cast<void **>(&j->d_fold_side)));
    CU(g_blocks.get(dv, nfk * sizeof(double), reinterpret_cast<void **>(&j->d_fold_err)));
    CU(g_blocks.get(dv, idx.size() * sizeof(int), reinterpret_cast<void **>(&j->d_fold_idx)));
    CU(g_blocks.get(dv, size_t(n_folds) * n * sizeof(int), reinterpret_cast<void **>(&j->d_fold_status)));
    // slot layout: rows [frame_start, last used frame] of the table (all columns) | rotation (9) | column map (M) | hide ranks
    // [n_folds][M] | hidden markers [n_folds][K]
    const size_t rows = size_t(n - 1) * frame_step + 1, bytes = rows * n_cols * 3 * sizeof(double);
    const size_t o_cols = bytes + 9 * sizeof(double), o_slot = o_cols + size_t(M) * sizeof(int32_t);
    const size_t o_idx = o_slot + slot_of.size() * sizeof(int32_t), total = o_idx + idx.size() * sizeof(int32_t);
    mosh2_job::RangeSlot *slot = nullptr;
    if (const int rc = staging_slot(j, total, &slot)) return rc;
    char *h = static_cast<char *>(slot->h);
    memcpy(h, markers + size_t(frame_start) * n_cols * 3, bytes);
    if (rot3x3) memcpy(h + bytes, rot3x3, 9 * sizeof(double));
    memcpy(h + o_cols, col_of_marker, size_t(M) * sizeof(int32_t));
    memcpy(h + o_slot, slot_of.data(), slot_of.size() * sizeof(int32_t));
    memcpy(h + o_idx, idx.data(), idx.size() * sizeof(int32_t));
    CU(cudaMemcpyAsync(slot->d, h, total, cudaMemcpyHostToDevice, j->stream));
    CU(cudaMemcpyAsync(j->d_fold_idx, static_cast<char *>(slot->d) + o_idx, idx.size() * sizeof(int32_t), cudaMemcpyDeviceToDevice, j->stream));
    const char *d = static_cast<const char *>(slot->d);
    const double *d_table = reinterpret_cast<const double *>(d), *d_rot = rot3x3 ? reinterpret_cast<const double *>(d + bytes) : nullptr;
    const int *d_cols = reinterpret_cast<const int *>(d + o_cols), *d_slot = reinterpret_cast<const int *>(d + o_slot);
    const size_t cnt = size_t(n_folds) * n * M, o0 = size_t(frame0) * M;
    const int blocks = int((cnt + 255) / 256);
    if (j->precision == MOSH2_F64)
        gather_folds_kernel<double><<<blocks, 256, 0, j->stream>>>(d_table, n_cols, d_cols, M, n, n_folds, frame_step, unit_per_metre, d_rot,
                                                                   d_slot, K, static_cast<double *>(j->d_obs) + 3 * o0, j->d_vis + o0,
                                                                   j->d_fold_side);
    else
        gather_folds_kernel<float><<<blocks, 256, 0, j->stream>>>(d_table, n_cols, d_cols, M, n, n_folds, frame_step, unit_per_metre, d_rot,
                                                                  d_slot, K, static_cast<float *>(j->d_obs) + 3 * o0, j->d_vis + o0,
                                                                  j->d_fold_side);
    CU(cudaGetLastError());
    CU(cudaEventRecord(slot->done, j->stream));
    j->fold_frame0 = frame0; j->fold_n = n; j->fold_count = n_folds; j->fold_K = K;
    return 0;
}

int mosh2_job_heldout_errors(mosh2_job *j, double *err, int32_t *status) {
    if (!j || !err) return fail(MOSH2_E_INVALID, "null argument");
    if (!j->fold_count) return fail(MOSH2_E_INVALID, "mosh2_job_heldout_errors needs a fold upload (mosh2_job_upload_markers_folds)");
    if (!j->launched) return fail(MOSH2_E_INVALID, "mosh2_job_heldout_errors needs a solve of the job first (mosh2_job_launch)");
    CU(cudaSetDevice(j->model->device));
    const size_t nfk = size_t(j->fold_count) * j->fold_n * j->fold_K, nf = size_t(j->fold_count) * j->fold_n;
    const int blocks = int((nfk + 255) / 256), M = j->model->n_markers;
    if (j->precision == MOSH2_F64)
        heldout_error_kernel<double><<<blocks, 256, 0, j->stream>>>(static_cast<const double *>(j->d_out) + j->o_mk, j->d_status, j->d_fold_side,
                                                                    j->d_fold_idx, M, j->fold_n, j->fold_count, j->fold_K, j->fold_frame0,
                                                                    j->d_fold_err, j->d_fold_status);
    else
        heldout_error_kernel<float><<<blocks, 256, 0, j->stream>>>(static_cast<const float *>(j->d_out) + j->o_mk, j->d_status, j->d_fold_side,
                                                                   j->d_fold_idx, M, j->fold_n, j->fold_count, j->fold_K, j->fold_frame0,
                                                                   j->d_fold_err, j->d_fold_status);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(err, j->d_fold_err, nfk * sizeof(double), cudaMemcpyDeviceToHost, j->stream));
    if (status) CU(cudaMemcpyAsync(status, j->d_fold_status, nf * sizeof(int), cudaMemcpyDeviceToHost, j->stream));
    CU(cudaStreamSynchronize(j->stream));
    return 0;
}

int mosh2_job_linearize(mosh2_job *j, const mosh2_options *opt, int32_t step, int32_t build, const double *x, const mosh2_lin_out *out) {
    if (!j || !x || !out || (step != 1 && step != 2)) return fail(MOSH2_E_INVALID, "bad argument");
    if (j->n_chunks < j->n_frames) return fail(MOSH2_E_INVALID, "mosh2_job_linearize needs a job of one-frame chunks (chunk_len = 1)");
    if (j->d_models) return fail(MOSH2_E_INVALID, "mosh2_job_linearize does not take a multi-model job");
    if (opt && !mosh2_host::robust_sigma_ok(*opt)) return fail(MOSH2_E_INVALID, "robust_sigma must be 0 (off) or a finite sigma > 0");
    CU(cudaSetDevice(j->model->device));
    if (opt) mosh2_host::apply_call_weights(j->opt, *opt);
    j->launched = false;                          // (the linearisation clears the rows)
    if (j->precision == MOSH2_F64) return linearize<double>(j, j->model->f64.m, step, build, x, out);
    return linearize<float>(j, j->model->f32.m, step, build, x, out);
}

int mosh2_job_launch(mosh2_job *j) {
    if (!j) return fail(MOSH2_E_INVALID, "null job");
    CU(cudaSetDevice(j->model->device));
    CU(cudaMemsetAsync(j->d_out, 0, j->n_out * j->esz, j->stream));
    CU(cudaMemsetAsync(j->d_status, 0, size_t(j->n_frames) * sizeof(int), j->stream));
    CU(cudaMemsetAsync(j->d_counters, 0, size_t(j->n_frames) * 4 * sizeof(int), j->stream));
    CU(cudaMemsetAsync(j->d_totals, 0, 8 * sizeof(int), j->stream));
    CU(cudaMemsetAsync(j->d_prof, 0, 32 * sizeof(long long), j->stream));
    if (j->tab_dirty) {               // a full launch runs the schedule the job was created with
        j->tab = j->tab0;
        CU(cudaMemcpyAsync(j->d_chunk_tab, j->tab.data(), j->tab.size() * sizeof(int), cudaMemcpyHostToDevice, j->stream));
        j->tab_dirty = false;
    }
    j->subset = false;
    j->launch_blocks = j->n_chunks;
    j->launched = true;
    if (j->precision == MOSH2_F64) return launch<double>(j, j->model->f64.m);
    return launch<float>(j, j->model->f32.m);
}

int mosh2_job_relaunch_chunks(mosh2_job *j, int32_t n, const int32_t *chunk_ids, int32_t chunk_warmup, int32_t warmup_full, double merge_tol,
                              const int32_t *root_turns) {
    if (!j || n < 1 || !chunk_ids || !(merge_tol >= 0)) return fail(MOSH2_E_INVALID, "bad argument");
    j->merge_tol = merge_tol;
    CU(cudaSetDevice(j->model->device));
    const int wf = chunk_warmup < 0 ? 0 : ((warmup_full < 0 || warmup_full > chunk_warmup) ? chunk_warmup : warmup_full);
    for (int k = 0; k < n; ++k) {
        const int c = chunk_ids[k];
        if (c < 0 || c >= j->n_chunks) return fail(MOSH2_E_INVALID, "chunk %d out of range (%d chunks)", c, j->n_chunks);
        j->tab[size_t(c) * mosh2::kChunkRec + 3] = chunk_warmup;
        j->tab[size_t(c) * mosh2::kChunkRec + 4] = wf;
        j->tab[size_t(c) * mosh2::kChunkRec + 5] = root_turns ? root_turns[k] : 0;
    }
    j->tab_dirty = true;
    CU(cudaStreamSynchronize(j->stream));
    CU(cudaMemcpy(j->d_chunk_tab, j->tab.data(), j->tab.size() * sizeof(int), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(j->d_chunk_ids, chunk_ids, size_t(n) * sizeof(int), cudaMemcpyHostToDevice));
    // the rows of the frames these chunks emit are rewritten by the kernel; everything else of the last launch stays
    j->subset = true;
    j->launch_blocks = n;
    if (j->precision == MOSH2_F64) return launch<double>(j, j->model->f64.m);
    return launch<float>(j, j->model->f32.m);
}

int mosh2_job_sequence_sweep(mosh2_job *j, double *max_delta) {
    if (!j) return fail(MOSH2_E_INVALID, "null job");
    if (!j->launched) return fail(MOSH2_E_INVALID, "mosh2_job_sequence_sweep needs a solve of the job first (mosh2_job_launch)");
    CU(cudaSetDevice(j->model->device));
    if (j->precision == MOSH2_F64) return sequence_sweep<double>(j, j->model->f64.m, max_delta);
    return sequence_sweep<float>(j, j->model->f32.m, max_delta);
}

int mosh2_job_boundary_deltas(mosh2_job *j, int32_t body_ids, float *out) {
    if (!j || !out || body_ids < 0) return fail(MOSH2_E_INVALID, "bad argument");
    CU(cudaSetDevice(j->model->device));
    const int PR = j->model->p_red, nd = j->model->n_dmpl, blocks = (j->n_chunks + 3) / 4;
    if (j->precision == MOSH2_F64) {
        const double *o = static_cast<const double *>(j->d_out);
        boundary_delta_kernel<double><<<blocks, 128, 0, j->stream>>>(static_cast<const double *>(j->d_warm_x), j->d_warm_f, o + j->o_pose, o + j->o_trans, o + j->o_dmpls, j->d_delta, j->n_chunks, PR, nd, body_ids);
    } else {
        const float *o = static_cast<const float *>(j->d_out);
        boundary_delta_kernel<float><<<blocks, 128, 0, j->stream>>>(static_cast<const float *>(j->d_warm_x), j->d_warm_f, o + j->o_pose, o + j->o_trans, o + j->o_dmpls, j->d_delta, j->n_chunks, PR, nd, body_ids);
    }
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(out, j->d_delta, size_t(j->n_chunks) * 4 * sizeof(float), cudaMemcpyDeviceToHost, j->stream));
    CU(cudaStreamSynchronize(j->stream));
    return 0;
}

int mosh2_job_warm_states(mosh2_job *j, double *x, int32_t *frames) {
    if (!j || !x || !frames) return fail(MOSH2_E_INVALID, "null argument");
    CU(cudaSetDevice(j->model->device));
    CU(cudaStreamSynchronize(j->stream));
    const size_t nx = size_t(3) + j->model->p_red + j->model->n_dmpl, n = size_t(j->n_chunks) * nx;
    CU(cudaMemcpy(frames, j->d_warm_f, size_t(j->n_chunks) * sizeof(int), cudaMemcpyDeviceToHost));
    if (j->precision == MOSH2_F64) CU(cudaMemcpy(x, j->d_warm_x, n * sizeof(double), cudaMemcpyDeviceToHost));
    else {
        std::vector<float> tmp(n);
        CU(cudaMemcpy(tmp.data(), j->d_warm_x, n * sizeof(float), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < n; ++i) x[i] = double(tmp[i]);
    }
    return 0;
}

int mosh2_job_sync(mosh2_job *j) {
    if (!j) return fail(MOSH2_E_INVALID, "null job");
    CU(cudaSetDevice(j->model->device));
    CU(cudaStreamSynchronize(j->stream));
    return 0;
}

int mosh2_job_kernel_ms(mosh2_job *j, float *ms) {
    if (!j || !ms) return fail(MOSH2_E_INVALID, "null argument");
    CU(cudaSetDevice(j->model->device));
    CU(cudaEventElapsedTime(ms, j->ev0, j->ev1));
    return 0;
}

void mosh2_release_cached_memory(void) { g_blocks.release_all(); }

int mosh2_job_span_ms(mosh2_job *first, mosh2_job *last, float *ms) {
    if (!first || !last || !ms) return fail(MOSH2_E_INVALID, "null argument");
    if (first->model->device != last->model->device) return fail(MOSH2_E_INVALID, "jobs live on different devices");
    CU(cudaSetDevice(first->model->device));
    CU(cudaEventElapsedTime(ms, first->ev0, last->ev1));
    return 0;
}

int mosh2_job_num_chunks(mosh2_job *j) { return j ? j->n_chunks : 0; }

int mosh2_job_chunk_ranges(mosh2_job *j, int32_t *out) {
    if (!j || !out) return fail(MOSH2_E_INVALID, "null argument");
    for (int c = 0; c < j->n_chunks; ++c) {
        out[2 * c] = j->tab0[size_t(c) * mosh2::kChunkRec];
        out[2 * c + 1] = j->tab0[size_t(c) * mosh2::kChunkRec + 1];
    }
    return 0;
}

// development builds (-DMOSH2_PROFILE) only: 32 phase clock sums of the last launch; not part of mosh2.h
int mosh2_dev_phase_clocks(mosh2_job *j, long long *out32) {
    if (!j || !out32) return fail(MOSH2_E_INVALID, "null argument");
    CU(cudaSetDevice(j->model->device));
    CU(cudaStreamSynchronize(j->stream));
    CU(cudaMemcpy(out32, j->d_prof, 32 * sizeof(long long), cudaMemcpyDeviceToHost));
    return 0;
}

int mosh2_job_totals(mosh2_job *j, int32_t *out8) {
    if (!j || !out8) return fail(MOSH2_E_INVALID, "null argument");
    CU(cudaSetDevice(j->model->device));
    CU(cudaStreamSynchronize(j->stream));
    CU(cudaMemcpy(out8, j->d_totals, 8 * sizeof(int), cudaMemcpyDeviceToHost));
    return 0;
}

int mosh2_job_upload_device(mosh2_job *j, const void *d_obs, int32_t obs_f64, const uint8_t *d_vis, void *producer_stream) {
    if (!j) return fail(MOSH2_E_INVALID, "null argument");
    return mosh2_job_upload_device_range(j, 0, j->n_frames, d_obs, obs_f64, d_vis, producer_stream);
}

int mosh2_job_upload_device_range(mosh2_job *j, int32_t frame0, int32_t nfr, const void *d_obs, int32_t obs_f64,
                                  const uint8_t *d_vis, void *producer_stream) {
    if (!j || !d_obs || !d_vis) return fail(MOSH2_E_INVALID, "null argument");
    if (frame0 < 0 || nfr < 1 || frame0 + nfr > j->n_frames) return fail(MOSH2_E_INVALID, "frame range [%d, %d) outside the job's %d frames", frame0, frame0 + nfr, j->n_frames);
    CU(cudaSetDevice(j->model->device));
    CU(cudaEventRecord(j->ev_in, static_cast<cudaStream_t>(producer_stream)));
    CU(cudaStreamWaitEvent(j->stream, j->ev_in, 0));
    const size_t M = j->model->n_markers, n = size_t(nfr) * M * 3, nv = size_t(nfr) * M, o0 = size_t(frame0) * M * 3;
    const bool dst64 = j->precision == MOSH2_F64;
    char *dst = static_cast<char *>(j->d_obs) + o0 * j->esz;
    if (dst64 == (obs_f64 != 0)) CU(cudaMemcpyAsync(dst, d_obs, n * j->esz, cudaMemcpyDeviceToDevice, j->stream));
    else {
        const int blocks = int((n + 255) / 256);
        if (dst64) convert_kernel<float, double><<<blocks, 256, 0, j->stream>>>(static_cast<const float *>(d_obs), reinterpret_cast<double *>(dst), n);
        else convert_kernel<double, float><<<blocks, 256, 0, j->stream>>>(static_cast<const double *>(d_obs), reinterpret_cast<float *>(dst), n);
        CU(cudaGetLastError());
    }
    CU(cudaMemcpyAsync(j->d_vis + size_t(frame0) * M, d_vis, nv, cudaMemcpyDeviceToDevice, j->stream));
    return 0;
}

int mosh2_job_row_width(mosh2_job *j) { return j ? 3 * j->model->n_joints + 3 + j->model->n_dmpl + mosh2::N_ERR + 2 : 0; }

int mosh2_job_download_device(mosh2_job *j, float *d_rows) {
    if (!j || !d_rows) return fail(MOSH2_E_INVALID, "null argument");
    CU(cudaSetDevice(j->model->device));
    const int PF = 3 * j->model->n_joints, nd = j->model->n_dmpl, width = mosh2_job_row_width(j);
    const size_t total = size_t(j->n_frames) * width;
    const int blocks = int((total + 255) / 256);
    if (j->precision == MOSH2_F64) {
        const double *o = static_cast<const double *>(j->d_out);
        pack_rows_kernel<double><<<blocks, 256, 0, j->stream>>>(o + j->o_fullpose, o + j->o_trans, o + j->o_dmpls, o + j->o_errs, j->d_status, j->d_counters, d_rows, j->n_frames, PF, nd);
    } else {
        const float *o = static_cast<const float *>(j->d_out);
        pack_rows_kernel<float><<<blocks, 256, 0, j->stream>>>(o + j->o_fullpose, o + j->o_trans, o + j->o_dmpls, o + j->o_errs, j->d_status, j->d_counters, d_rows, j->n_frames, PF, nd);
    }
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(j->stream));
    return 0;
}

int mosh2_job_download(mosh2_job *j, const mosh2_result *r) {
    if (!j || !r) return fail(MOSH2_E_INVALID, "null argument");
    CU(cudaSetDevice(j->model->device));
    const size_t F = j->n_frames;
    CU(cudaMemcpyAsync(j->h_out, j->d_out, j->n_out * j->esz, cudaMemcpyDeviceToHost, j->stream));
    CU(cudaMemcpyAsync(j->h_status, j->d_status, F * sizeof(int), cudaMemcpyDeviceToHost, j->stream));
    CU(cudaMemcpyAsync(j->h_counters, j->d_counters, F * 4 * sizeof(int), cudaMemcpyDeviceToHost, j->stream));
    CU(cudaStreamSynchronize(j->stream));
    const size_t M = j->model->n_markers, PF = size_t(3) * j->model->n_joints, PR = j->model->p_red, nd = j->model->n_dmpl;
    auto conv = [&](double *dst, size_t off, size_t n) {
        if (!dst) return;
        if (j->precision == MOSH2_F64) memcpy(dst, static_cast<double *>(j->h_out) + off, n * sizeof(double));
        else {
            const float *s = static_cast<float *>(j->h_out) + off;
            for (size_t i = 0; i < n; ++i) dst[i] = double(s[i]);
        }
    };
    conv(r->fullpose, j->o_fullpose, F * PF);
    conv(r->pose, j->o_pose, F * PR);
    conv(r->trans, j->o_trans, F * 3);
    if (nd) conv(r->dmpls, j->o_dmpls, F * nd);
    conv(r->markers_sim, j->o_mk, F * M * 3);
    conv(r->errs, j->o_errs, F * mosh2::N_ERR);
    if (r->status) memcpy(r->status, j->h_status, F * sizeof(int));
    if (r->counters) memcpy(r->counters, j->h_counters, F * 4 * sizeof(int));
    return 0;
}

void mosh2_job_destroy(mosh2_job *j) {
    if (!j) return;
    cudaSetDevice(j->model->device);
    if (j->stream) cudaStreamSynchronize(j->stream);
    const int dv = j->model->device;
    for (void *p : {static_cast<void *>(j->d_chunk_tab), static_cast<void *>(j->d_chunk_ids), static_cast<void *>(j->d_warm_f), j->d_warm_x,
                    static_cast<void *>(j->d_delta), j->d_obs, j->d_out, static_cast<void *>(j->d_vis), static_cast<void *>(j->d_status),
                    static_cast<void *>(j->d_counters), static_cast<void *>(j->d_totals), static_cast<void *>(j->d_prof), j->d_gws})
        g_blocks.put(dv, p);
    g_blocks.put(dv, j->d_lin);
    g_blocks.put(dv, j->d_models);
    g_blocks.put(dv, j->d_model_of_chunk);
    g_blocks.put(dv, j->d_model_of_frame);
    g_blocks.put(dv, j->d_seq_nbr);
    g_blocks.put(dv, j->d_seq_ids);
    g_blocks.put(dv, j->d_seq_delta);
    for (void *p : {static_cast<void *>(j->d_fold_side), static_cast<void *>(j->d_fold_err), static_cast<void *>(j->d_fold_idx),
                    static_cast<void *>(j->d_fold_status)})
        g_blocks.put(dv, p);
    for (void *p : {j->h_obs, j->h_out, static_cast<void *>(j->h_vis), static_cast<void *>(j->h_status), static_cast<void *>(j->h_counters)})
        g_blocks.put(-1, p);
    for (auto &s : j->range_slots) {        // (the stream is idle: every slot's copy and kernel have finished)
        g_blocks.put(-1, s.h);
        g_blocks.put(dv, s.d);
        if (s.done) cudaEventDestroy(s.done);
    }
    if (j->ev0) cudaEventDestroy(j->ev0);
    if (j->ev1) cudaEventDestroy(j->ev1);
    if (j->ev_in) cudaEventDestroy(j->ev_in);
    if (j->stream) cudaStreamDestroy(j->stream);
    delete j;
}

int mosh2_solve(mosh2_model *m, const mosh2_options *opt, int32_t n_frames, const double *obs, const uint8_t *vis,
                const mosh2_schedule *sched, int32_t precision, const mosh2_result *res) {
    mosh2_job *j = nullptr;
    int rc = mosh2_job_create(m, opt, n_frames, sched, precision, &j);
    if (rc) return rc;
    rc = mosh2_job_upload(j, obs, vis);
    if (!rc) rc = mosh2_job_launch(j);
    if (!rc) rc = mosh2_job_download(j, res);
    mosh2_job_destroy(j);
    return rc;
}

// ---- Stage-I surface term: point-to-triangle-mesh distance with derivatives (mesh_distance.cuh) ----------------------------
int mosh2_mesh_distance(int32_t device, int32_t kind, double sigma, int32_t n_samples, const double *samples, int32_t n_verts,
                        const double *verts, int32_t n_tris, const int32_t *tris, const int32_t *nearest_tri,
                        const int32_t *nearest_part, const mosh2_mesh_distance_out *out, float *kernel_ms) {
    if (!samples || !verts || !tris || !out || n_samples < 1 || n_verts < 1 || n_tris < 1 || kind < 0 || kind > 2)
        return fail(MOSH2_E_INVALID, "bad argument");
    if ((nearest_tri == nullptr) != (nearest_part == nullptr)) return fail(MOSH2_E_INVALID, "nearest_tri and nearest_part go together");
    if (n_tris >= (1 << 28)) return fail(MOSH2_E_TOO_LARGE, "%d triangles (the search packs the index into 29 bits)", n_tris);
    for (int64_t i = 0; i < int64_t(3) * n_tris; ++i)
        if (tris[i] < 0 || tris[i] >= n_verts) return fail(MOSH2_E_INVALID, "triangle %lld refers to vertex %d of %d", (long long)(i / 3), tris[i], n_verts);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return fail(MOSH2_E_NO_DEVICE, "no CUDA device: libmosh2 has no CPU path"); }
    if (device < 0 || device >= ndev) return fail(MOSH2_E_INVALID, "device %d out of range (%d devices)", device, ndev);
    CU(cudaSetDevice(device));
    const size_t S = n_samples, V = n_verts, T = n_tris;
    struct Buf { int dev; void *p = nullptr; ~Buf() { g_blocks.put(dev, p); } };
    Buf d_s{device}, d_sf{device}, d_v{device}, d_f{device}, d_soup{device}, d_best{device}, d_tri{device}, d_part{device}, d_val{device}, d_ds{device}, d_dt{device};
    CU(g_blocks.get(device, S * 3 * sizeof(double), &d_s.p));
    CU(g_blocks.get(device, S * 3 * sizeof(float), &d_sf.p));
    CU(g_blocks.get(device, V * 3 * sizeof(double), &d_v.p));
    CU(g_blocks.get(device, T * 3 * sizeof(int), &d_f.p));
    CU(g_blocks.get(device, T * mosh2_md::kSoupFloats * sizeof(float), &d_soup.p));
    CU(g_blocks.get(device, S * sizeof(unsigned long long), &d_best.p));
    CU(g_blocks.get(device, S * sizeof(int), &d_tri.p));
    CU(g_blocks.get(device, S * sizeof(int), &d_part.p));
    CU(g_blocks.get(device, S * sizeof(double), &d_val.p));
    CU(g_blocks.get(device, S * 3 * sizeof(double), &d_ds.p));
    CU(g_blocks.get(device, S * 9 * sizeof(double), &d_dt.p));
    cudaStream_t st = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    CU(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    CU(cudaEventCreate(&e0));
    CU(cudaEventCreate(&e1));
    auto cleanup = [&]() { cudaEventDestroy(e0); cudaEventDestroy(e1); cudaStreamDestroy(st); };
    cudaError_t e = cudaSuccess;
    auto chk = [&](cudaError_t r) { if (e == cudaSuccess) e = r; };
    chk(cudaMemcpyAsync(d_s.p, samples, S * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
    chk(cudaMemcpyAsync(d_v.p, verts, V * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
    chk(cudaMemcpyAsync(d_f.p, tris, T * 3 * sizeof(int), cudaMemcpyHostToDevice, st));
    chk(cudaEventRecord(e0, st));
    if (nearest_tri) {
        chk(cudaMemcpyAsync(d_tri.p, nearest_tri, S * sizeof(int), cudaMemcpyHostToDevice, st));
        chk(cudaMemcpyAsync(d_part.p, nearest_part, S * sizeof(int), cudaMemcpyHostToDevice, st));
    } else {
        convert_kernel<double, float><<<int((S * 3 + 255) / 256), 256, 0, st>>>(static_cast<const double *>(d_s.p), static_cast<float *>(d_sf.p), S * 3);
        mosh2_md::soup_kernel<<<int((T + 255) / 256), 256, 0, st>>>(static_cast<const double *>(d_v.p), static_cast<const int *>(d_f.p), int(T), static_cast<float *>(d_soup.p));
        chk(cudaMemsetAsync(d_best.p, 0xff, S * sizeof(unsigned long long), st));
        // triangle ranges: enough blocks to fill the GPU (four blocks per SM), whole tiles per block
        int n_sm = 0;
        chk(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, device));
        const int sblocks = int((S + mosh2_md::kSamplesPerBlock - 1) / mosh2_md::kSamplesPerBlock);
        int splits = (4 * std::max(n_sm, 1) + sblocks - 1) / sblocks;
        const int tiles = int((T + mosh2_md::kTileTris - 1) / mosh2_md::kTileTris);
        if (splits > tiles) splits = tiles;
        if (splits < 1) splits = 1;
        const int per = ((tiles + splits - 1) / splits) * mosh2_md::kTileTris;
        splits = int((T + per - 1) / per);
        mosh2_md::nearest_kernel<<<dim3(sblocks, splits), mosh2_md::kSamplesPerBlock, 0, st>>>(
            static_cast<const float *>(d_sf.p), int(S), static_cast<const float *>(d_soup.p), int(T), per, static_cast<unsigned long long *>(d_best.p));
        mosh2_md::unpack_kernel<<<int((S + 255) / 256), 256, 0, st>>>(static_cast<const unsigned long long *>(d_best.p), int(S), static_cast<int *>(d_tri.p), static_cast<int *>(d_part.p));
    }
    mosh2_md::evaluate_kernel<<<int((S + 127) / 128), 128, 0, st>>>(kind, sigma, static_cast<const double *>(d_s.p), int(S), static_cast<const double *>(d_v.p),
                                                                   static_cast<const int *>(d_f.p), static_cast<const int *>(d_tri.p), static_cast<const int *>(d_part.p),
                                                                   static_cast<double *>(d_val.p), static_cast<double *>(d_ds.p), static_cast<double *>(d_dt.p));
    chk(cudaGetLastError());
    chk(cudaEventRecord(e1, st));
    if (out->value) chk(cudaMemcpyAsync(out->value, d_val.p, S * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (out->tri) chk(cudaMemcpyAsync(out->tri, d_tri.p, S * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (out->part) chk(cudaMemcpyAsync(out->part, d_part.p, S * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (out->d_sample) chk(cudaMemcpyAsync(out->d_sample, d_ds.p, S * 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (out->d_tri) chk(cudaMemcpyAsync(out->d_tri, d_dt.p, S * 9 * sizeof(double), cudaMemcpyDeviceToHost, st));
    chk(cudaStreamSynchronize(st));
    if (e == cudaSuccess && kernel_ms) chk(cudaEventElapsedTime(kernel_ms, e0, e1));
    cleanup();
    if (e != cudaSuccess) return fail(MOSH2_E_CUDA, "mosh2_mesh_distance: %s", cudaGetErrorString(e));
    return 0;
}

}  // extern "C"
