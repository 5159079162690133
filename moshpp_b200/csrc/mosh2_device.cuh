// mosh2_device.cuh -- the Stage-II "CTA program": one thread block solves one chunk of consecutive
// frames of one sequence, frame after frame, with the reference's per-frame schedule
// (src/moshpp/chmosh.py:584-724) and the chumpy dog-leg (SURVEY.md Appendix A.6) entirely on device.
//
// The program is written against a tiny CTA abstraction (tid, nthr, M2_SYNC, cta_reduce) so that the
// very same source also compiles as a single-"thread" host build (MOSH2_EMU, tests/emu/) which the
// CPU test-suite uses to check index math against the oracle.  The product library never contains
// that build; libmosh2.so has no CPU path.
//
// Maths (SURVEY.md Appendix A; DESIGN.md section 3 for the derivations):
//   forward   fullpose = [theta_body, hands_mean + theta_hand C]; R_j = exp([w_j]x);
//             v_posed = v0 + Sd delta + Pd vec(R_j - I); FK; p_i = Rg_j (v_posed - J_j) + tg_j;
//             v = sum_i w_i p_i + trans; marker = v_c0 + k1 f1 + k2 f2 + k3 f3.
//   Jacobian  d v / d w_{a,k} = u_{a,k} x sum_{j in subtree(a)} w_j (p_j - tg_a)            (rigid part)
//                              + Rskin Pd_j dvec(R_j)/dw_k                                    (pose blend)
//             with u_{a,k} = Rg_par(a) vee(dR_{a,k} R_a^T); hand columns chained through C^T.
//   normal eq A = J^T J and g = -J^T r are accumulated marker tile by marker tile (J^T J on the tensor cores: f32 as
//             split TF32 with mma.sync m16n8k8, f64 with DMMA m8n8k4); the prior, velocity, finger, face and DMPL / expression
//             terms have closed-form contributions (Q_k = .5 inv(cov_k), diagonals).
//   The workspace layout (struct Work) is computed on the host and arrives as a kernel parameter of shared-memory offsets.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__) && !defined(MOSH2_EMU)
#define M2_HD __host__ __device__ __forceinline__
#define M2_D __device__ __forceinline__
#define M2_NOINLINE __device__ __noinline__
#define M2_SYNC() __syncthreads()
#define M2_WSYNC() __syncwarp()
#define M2_GPU 1
#else
#define M2_HD inline
#define M2_D inline
#define M2_NOINLINE static inline
#define M2_SYNC() ((void)0)
#define M2_WSYNC() ((void)0)
#define M2_GPU 0
#endif

// Optional phase timers (development builds only: -DMOSH2_PROFILE): thread 0 accumulates clock64() deltas
// between barriers into Job::prof.  Compiled out of the product library.
#if defined(MOSH2_PROFILE) && M2_GPU
#define M2_T0() long long t_prev_ = clock64()
#define M2_TACC(slot) do { if (cta.tid == 0) { const long long t_now_ = clock64(); w.prof[(slot) + prof_base] += t_now_ - t_prev_; t_prev_ = t_now_; } } while (0)
#define M2_TRESET() do { t_prev_ = clock64(); } while (0)
#else
#define M2_T0() ((void)0)
#define M2_TACC(slot) ((void)0)
#define M2_TRESET() ((void)0)
#endif

namespace mosh2 {
// ---------------------------------------------------------------------------------------------
// workspace addressing
// ---------------------------------------------------------------------------------------------
// The workspace layout (struct Work below) is computed once on the host and travels as a kernel parameter: every
// array is a 32-bit offset into the block's dynamic shared memory.  An address is therefore "shared-memory base +
// a constant-bank word": it costs no long-lived register (the dominant source of spills when the layout was
// carved inside the kernel) and the compiler still knows the address space (LDS/STS).
#if M2_GPU
extern __shared__ __align__(16) unsigned char m2_dyn_smem[];
M2_D unsigned char *m2_smem() { return m2_dyn_smem; }
#else
inline unsigned char *&m2_smem_ref() { static thread_local unsigned char *base = nullptr; return base; }
inline unsigned char *m2_smem() { return m2_smem_ref(); }
#endif
constexpr unsigned kSmemHeader = 16;     // first bytes of the dynamic shared memory: base of the per-CTA global workspace

// One sample of the mocap input adapter (mosh2.cu gather_markers_kernel; tools/mocap_interface.py:186,223-225,254-279):
// `p` the sample's xyz in file units, or NULL when the file has no column for the marker.  A sample is missing when a
// coordinate is NaN or all three are exactly zero (:277); a missing sample comes out as zero.  Otherwise it is turned by
// `rot` (row-major Rz Ry Rx, mocap.rotate, may be NULL) and converted to metres.  Returns the visibility.
M2_HD bool gather_marker_sample(const double *p, double unit_per_metre, const double *rot, double out[3]) {
    double x = 0, y = 0, z = 0;
    bool ok = false;
    if (p) {
        x = p[0]; y = p[1]; z = p[2];
        ok = !(isnan(x) || isnan(y) || isnan(z)) && !(x == 0.0 && y == 0.0 && z == 0.0);
    }
    if (!ok) { x = y = z = 0; }
    else {
        if (rot) {      // the points turned before the unit conversion (mocap_interface.py:218-221)
            const double rx = rot[0] * x + rot[1] * y + rot[2] * z, ry = rot[3] * x + rot[4] * y + rot[5] * z, rz = rot[6] * x + rot[7] * y + rot[8] * z;
            x = rx; y = ry; z = rz;
        }
        x = x / unit_per_metre; y = y / unit_per_metre; z = z / unit_per_metre;
    }
    out[0] = x; out[1] = y; out[2] = z;
    return ok;
}

template <class T>
struct SPtr {                            // array in shared memory
    uint32_t ofs;
    M2_D operator T *() const { return reinterpret_cast<T *>(m2_smem() + ofs); }
};
template <class T, bool BIG>
struct BPtr {                            // array in shared memory, or (BIG: f64 / oversized models) in the per-CTA global workspace
    uint32_t ofs;
    M2_D operator T *() const {
        if (BIG) return reinterpret_cast<T *>(*reinterpret_cast<char *const *>(m2_smem()) + ofs);
        return reinterpret_cast<T *>(m2_smem() + ofs);
    }
};
}  // namespace mosh2

namespace mosh2 {

enum { ST_SOLVED = 1, ST_SKIPPED = 2, ST_HAS_VELO = 4, ST_HAS_EXTRAP = 8, ST_GN_FALLBACK = 16, ST_MAXITER = 32, ST_SHORT_WARMUP = 64 };
enum { ERR_DATA = 0, ERR_POSEB = 1, ERR_VELO = 2, ERR_POSEH = 3, ERR_DMPL = 4, ERR_EXTRAP = 5, ERR_POSEF = 6, ERR_EXPR = 7, N_ERR = 8 };

constexpr int kBS = 4;            // register tile of the J^T J accumulation and of the Cholesky update
constexpr int kBlendGroups = 4;   // upper bound of the joint groups of the pose-blend partial sums (run time: 1..3, one round of threads)
constexpr int kCholNB = 8;        // block column width of the Cholesky factorisation
constexpr int kMaxHandBlocks = 4;
constexpr int kChunkRec = 6;      // ints per chunk-table record
constexpr int kMaxJangles = 16;   // joint-angle prior entries (the horse model has 12)

struct Cta {
    int tid, nthr;
};

struct HandBlock {   // one dense block of the hand-PCA matrix: rows [r0,r1) of the reduced pose, columns [q0,q1)
    int r0, r1, q0, q1, ct_off, rw4;   // Ct[(q-q0)*rw4 + (r-r0)] at hct + ct_off, rw4 = round_up(r1-r0, 4)
};

template <class real>
struct Model {
    int nJ, M, body_dof, p_red, n_hand_red, n_hand_full, nd, kw;
    const int *parents, *w_joint;
    const int *fk_order;        // joints sorted by depth (parents before children); derived from `parents` by the host library
    int hb_n, hct_size;
    HandBlock hb[kMaxHandBlocks];
    const real *hct;            // compact transposed hand-PCA blocks
    const real *hands_mean, *v0, *sd, *w_val, *j0, *jd, *coefs;
    const real *pdc;            // pose-blend table [(nJ-1)][9 e][3 c][Sp], Sp = 3M rounded up to 4: no padding; eval() reads four slots per 16-byte load
    const real *pd4;            // the same table as [(nJ-1)][9 e][3M slots][x y z -]: build() reads one slot (all three coordinates) per 16-byte load
    int prior_k, prior_d, prior_d4;
    const int *prior_ids;       // [D] reduced-pose ids the prior sees, in the order of its dimensions (SMPL family: a contiguous run; the
                                // animal models pick a subset of the joints, prior/dog_body_prior.py:51-53)
    const real *prior_means, *prior_Q4, *prior_nlw;   // Q4: [K][D][D4]
    const real *prior_Qt;       // Q transposed per component, [K][D l][D4 i]: threads over rows i read consecutive words
    int n1, n2;
    const int *free1, *free2;
    int finger_lo, finger_hi;
    int n_expr, face_lo, face_hi;   // optimize_face: the last n_expr linear coefficients are expressions; jaw pose ids
    int n_jang;                     // animal_horse: joint-angle term exp(2 s x)^2 on these reduced-pose ids (prior/horse_body_prior.py:56-71)
    int jang_id[kMaxJangles];
    real jang_sign[kMaxJangles];
    int tile_markers;           // markers per Jacobian tile (20 or 10: a warp owns ten), chosen by the host from the shared-memory budget
    int dev_no_tc;              // development switch (host): 1 = J^T J stays on the CUDA cores
    const unsigned char *stage_blob;   // the small per-model tables laid out exactly like the staged region of the shared-memory
                                       // workspace (carve(): Work::stage_ofs / stage_bytes); one bulk asynchronous copy per chunk
};

struct Options {
    double wt_data, wt_poseB, wt_poseH, wt_velo, wt_dmpl, wt_annealing, wt_extrap;
    double num_train_markers, delta_0, e3_first, e3;
    int maxiter, optimize_fingers, optimize_dynamics;
    double wt_poseF, wt_expr;
    int optimize_face;
};

template <class real>
struct Job {
    int n_frames, n_chunks;
    const int *chunk_tab;   // [n_chunks][kChunkRec]: first emitted frame, end of the emitted range, first frame of the chunk's
                            // sequence, warm-up (solved frames), how many of them (the last ones) run the full per-frame schedule,
                            // full turns added to the root of the chunk's cold start (Solver::procrustes)
    const int *chunk_ids;   // launch of a subset of the chunks: blockIdx.x -> chunk, or null (all chunks)
    double merge_tol;       // resume mode: a re-solved frame within this of the row it replaces counts as merged (rad on root + body pose;
                            // x 10 on the other pose coefficients, x 0.1 m on the translation)
    real *warm_x;           // [n_chunks][NX] state after the chunk's last warm-up frame (boundary check against the emitted
    int *warm_f;            // [n_chunks]     result of that frame, which an earlier chunk produced), and that frame's index or -1
    const real *obs;        // F*M*3
    const uint8_t *vis;     // F*M
    real *fullpose, *pose, *trans, *dmpls, *markers_sim, *errs;
    int *status, *counters;
    int *totals;            // [8] iterations, evaluations, builds, minimisations over ALL processed frames (incl. warm-up), then over the emitted frames
    long long *prof;        // [32] phase clock sums (MOSH2_PROFILE builds only, else unused)
    char *gws;              // optional per-CTA global workspace (f64 / large models)
    size_t gws_stride;
    // Linearise mode (Stage I, mosh2_job_linearize): every frame is an independent problem evaluated at a GIVEN state; one
    // thread block per frame evaluates the residual there and, with lin_mode == 2, builds and exports the linearisation.
    int lin_mode;           // 0: the Stage-II frame loop; 1: residual only; 2: residual + normal equations + Jacobian rows
    int lin_step;           // free-variable list: 1 = free1, 2 = free2 (+ the finger term)
    const real *lin_x;      // [F][NX] states
    real *lin_A, *lin_g;    // [F][n][n], [F][n]: normal equations of the frame's own terms (data, pose prior, fingers)
    real *lin_J, *lin_r;    // [F][3M][n], [F][3M]: weighted data rows d r / d x_free and r = (sim - obs) wd (zero where invisible)
    real *lin_vp;           // [F][3M][3]: posed attachment vertices (slot = 3 marker + t)
    Options opt;
};

// ---------------------------------------------------------------------------------------------
// small math
// ---------------------------------------------------------------------------------------------
M2_HD float r_sqrt(float x) { return sqrtf(x); }
M2_HD double r_sqrt(double x) { return sqrt(x); }
// reciprocal square root: MUFU.RSQ plus one Newton step on the device (f32), exact division elsewhere
M2_HD float r_rsqrt(float x) {
#if M2_GPU
    const float y = rsqrtf(x);
    return y * (1.5f - 0.5f * x * y * y);
#else
    return 1.0f / sqrtf(x);
#endif
}
M2_HD double r_rsqrt(double x) { return 1.0 / sqrt(x); }
M2_HD float r_exp(float x) { return expf(x); }
M2_HD double r_exp(double x) { return exp(x); }
M2_HD float r_abs(float x) { return fabsf(x); }
M2_HD double r_abs(double x) { return fabs(x); }
M2_HD void r_sincos(float x, float *s, float *c) {
#if M2_GPU
    sincosf(x, s, c);
#else
    *s = sinf(x);
    *c = cosf(x);
#endif
}
M2_HD void r_sincos(double x, double *s, double *c) {
#if M2_GPU
    sincos(x, s, c);
#else
    *s = sin(x);
    *c = cos(x);
#endif
}
template <class real> M2_HD real series_thresh();
template <> M2_HD float series_thresh<float>() { return 0.25f; }
template <> M2_HD double series_thresh<double>() { return 1e-2; }
template <class real> M2_HD real pivot_eps();          // smallest accepted pivot of the unit-diagonal-scaled A
template <> M2_HD float pivot_eps<float>() { return 1e-6f; }
template <> M2_HD double pivot_eps<double>() { return 1e-13; }

// Acceptance slack of the dog-leg in units of the current SSE.  chumpy accepts a trial step iff the SSE decreases
// (rho > 0).  In float64 that test is exact enough (slack 0: reference semantics).  In float32 the SSE of a
// converged frame is only resolved to ~1e-6 relative, so the final tiny-improvement step that float64 accepts
// (and then stops on, e_3) would be rejected at random and trigger a cascade of trust-region shrinks; a step whose
// measured SSE change is within the slack is therefore treated like float64 would treat it: accepted, after
// which the e_3 rule stops the minimisation.  DESIGN.md section 5.
template <class real> M2_HD real accept_slack();
template <> M2_HD float accept_slack<float>() { return 1e-5f; }
template <> M2_HD double accept_slack<double>() { return 0.0; }

#if M2_GPU
// t == 0 ? a : (t == 1 ? b : c) as two select instructions
__device__ __forceinline__ float sel3(int t, float a, float b, float c) {
    float r;
    asm("{\n\t.reg .pred p, q;\n\tsetp.eq.s32 p, %1, 0;\n\tsetp.eq.s32 q, %1, 1;\n\tselp.f32 %0, %3, %4, q;\n\tselp.f32 %0, %2, %0, p;\n\t}"
        : "=&f"(r) : "r"(t), "f"(a), "f"(b), "f"(c));
    return r;
}
__device__ __forceinline__ double sel3(int t, double a, double b, double c) {
    double r;
    asm("{\n\t.reg .pred p, q;\n\tsetp.eq.s32 p, %1, 0;\n\tsetp.eq.s32 q, %1, 1;\n\tselp.f64 %0, %3, %4, q;\n\tselp.f64 %0, %2, %0, p;\n\t}"
        : "=&d"(r) : "r"(t), "d"(a), "d"(b), "d"(c));
    return r;
}
#endif

#if M2_GPU
// D = A B + D, one warp: A 8x4 (row), B 4x8 (col), D 8x8, float64 (lane: a = A[lane/4][lane%4], b = B[lane%4][lane/4],
// d0, d1 = D[lane/4][2 (lane%4) + 0, 1])
__device__ __forceinline__ void dmma_m8n8k4(double &d0, double &d1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
#endif

template <class real> struct alignas(16) Vec4 { real x, y, z, w; };
template <class real> M2_HD Vec4<real> ld4(const real *p) { return *reinterpret_cast<const Vec4<real> *>(p); }
template <class real>
M2_NOINLINE void mat3_mul(const real *A, const real *B, real *C) {   // C = A B (row-major 3x3); C must not alias A or B
#pragma unroll 1
    for (int i = 0; i < 3; ++i) {
        const real a0 = A[3 * i], a1 = A[3 * i + 1], a2 = A[3 * i + 2];
        C[3 * i] = a0 * B[0] + a1 * B[3] + a2 * B[6];
        C[3 * i + 1] = a0 * B[1] + a1 * B[4] + a2 * B[7];
        C[3 * i + 2] = a0 * B[2] + a1 * B[5] + a2 * B[8];
    }
}
template <class real>
M2_HD void mat3_mul_reg(const real *A, const real *B, real *C) {   // inline variant for register arrays
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
template <class real>
M2_HD void mat3_vec(const real *A, const real *v, real *o) {
    o[0] = A[0] * v[0] + A[1] * v[1] + A[2] * v[2];
    o[1] = A[3] * v[0] + A[4] * v[1] + A[5] * v[2];
    o[2] = A[6] * v[0] + A[7] * v[1] + A[8] * v[2];
}
template <class real>
M2_HD void cross3(const real *a, const real *b, real *o) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}
// block (bi, bj), bi <= bj, of the upper triangle of an nb x nb grid of blocks that are numbered row by row
M2_HD void upper_block(int idx, int nb, int &bi, int &bj) {
    int ti = 0, rem = idx;
    while (rem >= nb - ti) { rem -= nb - ti; ++ti; }
    bi = ti;
    bj = ti + rem;
}

// R = exp([w]x) and dR[k] = dR/dw_k (cv2.Rodrigues convention), cancellation-free near 0.
// `only_k` >= 0: this caller writes only dR[only_k] (and R when only_k == 0) -- three threads share a joint.
template <class real>
M2_NOINLINE void rodrigues(const real *w, real *R, real *dR, int only_k = -1) {
    const real x = w[0], y = w[1], z = w[2];
    const real t2 = x * x + y * y + z * z;
    real a, b, c1, c2;
    if (t2 < series_thresh<real>()) {
        a = real(1) + t2 * (real(-1. / 6) + t2 * (real(1. / 120) + t2 * (real(-1. / 5040) + t2 * real(1. / 362880))));
        b = real(.5) + t2 * (real(-1. / 24) + t2 * (real(1. / 720) + t2 * (real(-1. / 40320) + t2 * real(1. / 3628800))));
        c1 = real(-1. / 3) + t2 * (real(1. / 30) + t2 * (real(-1. / 840) + t2 * (real(1. / 45360) + t2 * real(-1. / 3991680))));
        c2 = real(-1. / 12) + t2 * (real(1. / 180) + t2 * (real(-1. / 6720) + t2 * (real(1. / 453600) + t2 * real(-1. / 47900160))));
    } else {
        const real t = r_sqrt(t2);
        real s, c;
        r_sincos(t, &s, &c);
        a = s / t;
        b = (real(1) - c) / t2;
        c1 = (t * c - s) / (t2 * t);
        c2 = (t * s - real(2) * (real(1) - c)) / (t2 * t2);
    }
    // K = [w]x, K2 = K K = w w^T - t2 I
    const real K[9] = {0, -z, y, z, 0, -x, -y, x, 0};
    const real K2[9] = {x * x - t2, x * y, x * z, x * y, y * y - t2, y * z, x * z, y * z, z * z - t2};
    if (only_k <= 0) {
#pragma unroll
        for (int i = 0; i < 9; ++i) R[i] = a * K[i] + b * K2[i] + ((i == 0 || i == 4 || i == 8) ? real(1) : real(0));
    }
    if (!dR) return;
    // dR/dw_k = c1 w_k K + a E_k + c2 w_k K2 + b (E_k K + K E_k),   E_k K + K E_k = e_k w^T + w e_k^T - 2 w_k I
#pragma unroll 1
    for (int k = (only_k < 0 ? 0 : only_k); k < (only_k < 0 ? 3 : only_k + 1); ++k) {
        const real wk = w[k];
        real *D = dR + 9 * k;
#pragma unroll
        for (int i = 0; i < 9; ++i) D[i] = c1 * wk * K[i] + c2 * wk * K2[i];
        if (k == 0) { D[5] -= a; D[7] += a; }
        if (k == 1) { D[2] += a; D[6] -= a; }
        if (k == 2) { D[1] -= a; D[3] += a; }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            D[3 * k + c] += b * w[c];
            D[3 * c + k] += b * w[c];
        }
        D[0] -= real(2) * b * wk;
        D[4] -= real(2) * b * wk;
        D[8] -= real(2) * b * wk;
    }
}

// ---------------------------------------------------------------------------------------------
// CTA-wide reduction of NV (<= 8) per-thread values; result broadcast to every thread.
// ---------------------------------------------------------------------------------------------
template <class real, int NV>
M2_D void cta_reduce(const Cta &c, real *vals, real *scratch /* >= 8*33 reals */) {
#if M2_GPU
    // warp sums by shuffles, one partial per warp through shared memory, then EVERY warp adds the partials with a second
    // shuffle tree (lane = warp of the partial): no serial loop over the warps and no broadcast round (the serial
    // version cost ~800 cycles a call, five calls per dog-leg iteration)
    const int lane = c.tid & 31, warp = c.tid >> 5, nwarp = (c.nthr + 31) >> 5;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        real v = vals[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) scratch[i * 33 + warp] = v;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        real v = lane < nwarp ? scratch[i * 33 + lane] : real(0);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        vals[i] = v;
    }
    __syncthreads();                 // (the partials may be overwritten by the next call)
#else
    (void)c; (void)vals; (void)scratch;
#endif
}

template <class real>
M2_D real warp_sum(real v) {
#if M2_GPU
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
#endif
    return v;
}

// ---------------------------------------------------------------------------------------------
// workspace
// ---------------------------------------------------------------------------------------------
template <class real, bool BIG = false>
struct Work {
    // state
    SPtr<real> x, xt, pose_prev, velo_tgt, dm_tgt;
    // forward scratch of the latest evaluation
    SPtr<real> fullpose, Rl, dRl, Jp, Rg, tg, vp, pj, Rsk, mk, rm, obs, py, pq, pxg;
    // Jacobian / normal equations (the build scratch Loc .. dtg is "big": laid over Lm, in the global workspace with BIG)
    BPtr<real, BIG> Loc, MtR, u, dtg;
    SPtr<real> Linv, Pn, g, Ag, dgn, d, tmp, ds;
    BPtr<real, BIG> Jt, Jf, A, Lm;
    SPtr<real> red, sc, hct;
    SPtr<int> colmap, colsrc, jlist, isc;
    SPtr<int> st_colmap, st_colsrc, st_jlist, st_meta;   // the two stage configurations (Step-1 / Step-2 variable lists), built once per chunk
    // small per-model tables staged in shared memory (a dependent global load costs several hundred cycles and the
    // kinematic-tree walk alone chains three of them per level)
    SPtr<int> c_parents, c_fk_order, c_wj, c_free1, c_free2, c_pids;
    SPtr<int> c_tin, c_tsz;   // pre-order index and subtree size of every joint: j in subtree(a) <=> tin[j]-tin[a] in [0, tsz[a])
    SPtr<real> c_wv, c_v0, c_coefs, c_j0, c_hmean, c_pmeans, c_pnlw;
    SPtr<real> c_jd;          // joint-position directions of the per-frame linear coefficients (DMPL, expressions); not staged
                              // with BIG, where the kernel reads Model::jd (Solver::jdir)
    SPtr<long long> prof;
    SPtr<uint8_t> vis;
    SPtr<uint32_t> c_chain;   // [joint][4 words]: the joint's ancestor chain, root first, one byte per joint id, 255-padded
    SPtr<uint8_t> c_amask;    // [slot][joint]: bit i set <=> the slot's i-th skinning joint lies in the subtree of the joint
    SPtr<unsigned long long> mbar;   // completion barrier of the table staging
    uint32_t stage_ofs, stage_bytes;   // the staged per-model tables: one contiguous, 16-byte aligned region (c_parents ... hct)
    int tc_ok;                // the model qualifies for the f32 tensor-core J^T J (f32, workspace in shared memory)
    int tc;                   // set by the launcher: tensor cores in use
};

// ---------------------------------------------------------------------------------------------
// tensor cores for the J^T J accumulation of the f32 kernel; bulk asynchronous copies
// ---------------------------------------------------------------------------------------------
// A warp computes one 16x16 block of the upper triangle of Jf^T Jf over the rows of a tile with mma.sync m16n8k8 on
// TF32 operands.  Every Jacobian value is split into a TF32 "hi" part and a TF32 "lo" remainder;
// hi hi^T goes to one register accumulator, lo hi^T + hi lo^T + lo lo^T to another, and their sum is added to A
// on the CUDA cores once per tile: close to fp32 accuracy (3xTF32), and the tensor core's truncating additions only
// ever span the rows of one tile.
constexpr int kMaxDepth = 16;         // deepest kinematic chain the tree walk unrolls (checked at model creation)
constexpr int kDR = 28;              // floats per joint in dRl: three 3x3 derivative matrices (27) padded to 16-byte vectors
constexpr int kM3 = 12;              // floats per padded 3x3 matrix (MtR per slot, Loc per marker vertex) and per joint in u (3 x 4)
#if M2_GPU
namespace tc {
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ uint32_t to_tf32(float v) { uint32_t r; asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v)); return r; }
// D += A B, one warp: A 16x8 (row), B 8x8 (col), D 16x8 f32 (g = lane / 4, t = lane % 4: a = A[g, g+8, g, g+8][t, t, t+4, t+4],
// b = B[t, t+4][g], d = D[g, g, g+8, g+8][2t, 2t+1, 2t, 2t+1])
__device__ __forceinline__ void mma_tf32_m16n8k8(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// One warp: block (rows i0.., columns j0..) of J^T J over `rows` rows of the row-major tile J (row length ld; columns
// >= cols read as zero).  hh[nj] / cr[nj]: the 16x8 accumulators of columns j0 + 8 nj.. (hi hi^T, and the cross terms).
__device__ __forceinline__ void jtj_block_tf32(const float *J, int ld, int rows, int cols, int i0, int j0,
                                               float (&hh)[2][4], float (&cr)[2][4]) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int ca0 = i0 + g, ca1 = i0 + 8 + g, cb0 = j0 + g, cb1 = j0 + 8 + g;
    for (int k0 = 0; k0 < rows; k0 += 8) {
        const int k1 = k0 + t, k2 = k0 + t + 4;
        const float *r1 = J + (k1 < rows ? k1 : 0) * ld, *r2 = J + (k2 < rows ? k2 : 0) * ld;
        const bool in1 = k1 < rows, in2 = k2 < rows;
        // A[i][k] = J[k][i], B[k][j] = J[k][j]
        const float av[4] = {(in1 && ca0 < cols) ? r1[ca0] : 0.f, (in1 && ca1 < cols) ? r1[ca1] : 0.f,
                             (in2 && ca0 < cols) ? r2[ca0] : 0.f, (in2 && ca1 < cols) ? r2[ca1] : 0.f};
        const float bv[2][2] = {{(in1 && cb0 < cols) ? r1[cb0] : 0.f, (in2 && cb0 < cols) ? r2[cb0] : 0.f},
                                {(in1 && cb1 < cols) ? r1[cb1] : 0.f, (in2 && cb1 < cols) ? r2[cb1] : 0.f}};
        uint32_t ahi[4], alo[4], bhi[2][2], blo[2][2];
#pragma unroll
        for (int q = 0; q < 4; ++q) { ahi[q] = to_tf32(av[q]); alo[q] = to_tf32(av[q] - __uint_as_float(ahi[q])); }
#pragma unroll
        for (int nj = 0; nj < 2; ++nj)
#pragma unroll
            for (int q = 0; q < 2; ++q) { bhi[nj][q] = to_tf32(bv[nj][q]); blo[nj][q] = to_tf32(bv[nj][q] - __uint_as_float(bhi[nj][q])); }
#pragma unroll
        for (int nj = 0; nj < 2; ++nj) {
            mma_tf32_m16n8k8(hh[nj], ahi, bhi[nj][0], bhi[nj][1]);
            mma_tf32_m16n8k8(cr[nj], alo, bhi[nj][0], bhi[nj][1]);
            mma_tf32_m16n8k8(cr[nj], ahi, blo[nj][0], blo[nj][1]);
            mma_tf32_m16n8k8(cr[nj], alo, blo[nj][0], blo[nj][1]);
        }
    }
}
__device__ __forceinline__ void mbar_init(uint32_t mbar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(mbar), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t mbar, uint32_t parity) {
    asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
                 "@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}\n" :: "r"(mbar), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t mbar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mbar), "r"(bytes) : "memory");
}
// bulk asynchronous copy global -> shared memory (the TMA engine on a contiguous run; 16-byte aligned, size a multiple of
// 16), completing on an mbarrier by byte count
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void *src, uint32_t bytes, uint32_t mbar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(dst_smem), "l"(src), "r"(bytes), "r"(mbar) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
}  // namespace tc
#endif

struct Dims {
    int nJ, M, S, PF, PR, nd, NX, NCt, n1, n2, ld, lda, ldp, npad, K, D, D4, kw, jt_size, tmk;
};

template <class real>
M2_HD Dims make_dims(const Model<real> &m) {
    Dims d;
    d.nJ = m.nJ; d.M = m.M; d.S = 3 * m.M; d.PF = 3 * m.nJ; d.PR = m.p_red; d.nd = m.nd;
    d.NX = 3 + m.p_red + m.nd; d.NCt = (m.n_hand_full + 3) & ~3;   /* columns of the full-pose hand tile Jt */ d.n1 = m.n1; d.n2 = m.n2;
    d.npad = (m.n2 + 3) & ~3;
    // Cholesky factor: rows are 16-byte aligned (vector read-modify-write of 4x4 tiles) and the row length is 4 mod 8
    // words, so that the panel's one-row-per-thread 16-byte accesses (eight consecutive rows per quarter warp) fall into
    // eight different groups of four banks (at 112 words every second row started in the same bank: 16-way conflicts)
    d.ld = ((m.n2 + 7) & ~7) + 4;   // (and >= the last 8-column block, which the panel reads whole)
    d.ldp = d.npad + 4;         // row length of the transposed panel (one extra row: the right-hand side)
    d.lda = d.npad | 1;         // A: odd leading dimension, so row-strided and transposed tile accesses spread over banks
    d.K = m.prior_k; d.D = m.prior_d; d.D4 = m.prior_d4; d.kw = m.kw;
    d.tmk = m.tile_markers > 0 ? m.tile_markers : 10;
    const int a = 3 * d.tmk * d.NCt, b = kBlendGroups * 9 * m.M + 16;   // Jt doubles as the pose-blend partial sums
    d.jt_size = a > b ? a : b;
    return d;
}

struct Arena {
    size_t off;
    template <class T> M2_HD uint32_t take(size_t n) {
        off = (off + 15) & ~size_t(15);
        const size_t o = off;
        off += n * sizeof(T);
        return uint32_t(o);
    }
};

// Lays the workspace out.  Arrays flagged "big" go to arena G when big_in_global is set (f64 runs, large
// models), everything else to arena S (shared memory).
template <class real, bool BIG>
M2_HD void carve(Work<real, BIG> &w, const Dims &d, const Model<real> &m, Arena &S, Arena &G) {
    // BIG is a compile-time switch so that, in the normal case, every workspace pointer provably points into
    // shared memory and the compiler emits LDS/STS instead of generic loads and stores
    const int hct_size = m.hct_size;
    Arena &B = BIG ? G : S;
    w.x.ofs = S.take<real>(d.NX); w.xt.ofs = S.take<real>(d.NX);
    w.pose_prev.ofs = S.take<real>(d.PR); w.velo_tgt.ofs = S.take<real>(d.PR); w.dm_tgt.ofs = S.take<real>(d.nd + 1);
    w.fullpose.ofs = S.take<real>(d.PF); w.Rl.ofs = S.take<real>(9 * d.nJ); w.dRl.ofs = S.take<real>(kDR * d.nJ);
    w.Jp.ofs = S.take<real>(3 * d.nJ); w.Rg.ofs = S.take<real>(9 * d.nJ); w.tg.ofs = S.take<real>(3 * d.nJ);
    w.vp.ofs = S.take<real>(3 * d.S); w.pj.ofs = S.take<real>(3 * d.S * d.kw); w.Rsk.ofs = S.take<real>(9 * d.S);
    w.mk.ofs = S.take<real>(3 * d.M); w.rm.ofs = S.take<real>(3 * d.M); w.obs.ofs = S.take<real>(3 * d.M);
    w.py.ofs = S.take<real>(d.K * d.D + 1); w.pq.ofs = S.take<real>(d.K + 1); w.pxg.ofs = S.take<real>(d.D + 1);
    // The Cholesky factor is alive only inside gauss_newton(); the Jacobian tiles and the other scratch of build()
    // (and the pose-blend partial sums of eval(), which live in Jt) are dead there, so they share its storage.
    // A and the Cholesky factor Lm are adjacent.  The factor is alive only inside gauss_newton(); the scratch of
    // build() (and the pose-blend partial sums of eval(), which live in Jt) is dead there and is laid over it.
    {
        w.A.ofs = B.take<real>(size_t(d.n2) * d.lda);
        w.tc_ok = (sizeof(real) == 4 && !BIG && !m.dev_no_tc) ? 1 : 0;
        w.tc = 0;
        const size_t mark_b = B.off;
        w.Lm.ofs = B.take<real>(size_t(d.n2 + 1) * d.ld);
        const size_t end_b = B.off;
        B.off = mark_b;
        w.Jt.ofs = B.take<real>(d.jt_size);
        w.Jf.ofs = B.take<real>(3 * d.tmk * d.npad);
        // (with BIG these go to the global workspace as well: in float64, 36 M words each for Loc and MtR and 3 nJ nd for dtg
        // -- 106 KB for SMPL-X with 80 expressions -- do not fit next to the rest of the shared part)
        w.Loc.ofs = B.take<real>(3 * kM3 * d.M); w.MtR.ofs = B.take<real>(kM3 * d.S);
        w.u.ofs = B.take<real>(kM3 * d.nJ); w.dtg.ofs = B.take<real>(3 * d.nJ * d.nd + 1);
        if (B.off < end_b) B.off = end_b;
    }
    w.Linv.ofs = S.take<real>(size_t((d.n2 + kCholNB - 1) / kCholNB) * kCholNB * kCholNB);
    w.Pn.ofs = S.take<real>(size_t(kCholNB) * d.ldp);
    w.g.ofs = S.take<real>(d.npad); w.Ag.ofs = S.take<real>(d.npad); w.dgn.ofs = S.take<real>(d.npad);
    w.d.ofs = S.take<real>(d.npad); w.tmp.ofs = S.take<real>(d.npad); w.ds.ofs = S.take<real>(d.npad);
    w.red.ofs = S.take<real>(8 * 33); w.sc.ofs = S.take<real>(16);
    w.colmap.ofs = S.take<int>(d.NX); w.colsrc.ofs = S.take<int>(d.n2); w.jlist.ofs = S.take<int>(d.nJ); w.isc.ofs = S.take<int>(8);
    w.st_colmap.ofs = S.take<int>(2 * d.NX); w.st_colsrc.ofs = S.take<int>(2 * d.n2); w.st_jlist.ofs = S.take<int>(2 * d.nJ); w.st_meta.ofs = S.take<int>(4);
    w.prof.ofs = S.take<long long>(32);
    w.mbar.ofs = S.take<unsigned long long>(1);
    w.vis.ofs = S.take<uint8_t>(d.M);
    // small per-model tables are always staged in shared memory (a dependent global load costs ~600 cycles and the
    // kinematic-tree walk chains three of them per level); the larger ones stay in global memory / L2.  The tables that
    // are plain copies of model arrays -- kinematic tree, skinning joints and weights, shaped template rows, marker
    // coefficients, joint positions and directions, prior means, hand-PCA blocks, free-variable lists -- form ONE
    // contiguous region: the host library keeps a byte-identical image of it (Model::stage_blob, stage_image below) and a chunk
    // fetches it with a single bulk asynchronous copy (cp.async.bulk completing on an mbarrier) instead of thirteen copy loops.
    // The joint directions c_jd come last and are left out with BIG (3 nJ nd words, as dtg): the image is laid out without
    // BIG, and a BIG block copies the prefix of it that ends with hct.
    S.off = (S.off + 15) & ~size_t(15);
    w.stage_ofs = uint32_t(S.off);
    w.c_parents.ofs = S.take<int>(d.nJ); w.c_fk_order.ofs = S.take<int>(d.nJ);
    w.c_wj.ofs = S.take<int>(d.S * d.kw); w.c_free1.ofs = S.take<int>(d.n1); w.c_free2.ofs = S.take<int>(d.n2);
    w.c_pids.ofs = S.take<int>(d.D + 1);
    w.c_wv.ofs = S.take<real>(d.S * d.kw); w.c_v0.ofs = S.take<real>(3 * d.S); w.c_coefs.ofs = S.take<real>(3 * d.M);
    w.c_j0.ofs = S.take<real>(3 * d.nJ); w.c_hmean.ofs = S.take<real>(m.n_hand_full + 1);
    w.c_pmeans.ofs = S.take<real>(d.K * d.D + 1); w.c_pnlw.ofs = S.take<real>(d.K + 1);
    w.hct.ofs = S.take<real>(hct_size + 4);
    if (!BIG) w.c_jd.ofs = S.take<real>(size_t(3) * d.nJ * d.nd + 1);
    S.off = (S.off + 15) & ~size_t(15);
    w.stage_bytes = uint32_t(S.off) - w.stage_ofs;
    // tables the chunk derives itself
    w.c_tin.ofs = S.take<int>(d.nJ); w.c_tsz.ofs = S.take<int>(d.nJ); w.c_amask.ofs = S.take<uint8_t>(size_t(d.S) * d.nJ);
    w.c_chain.ofs = S.take<uint32_t>(size_t(d.nJ) * (kMaxDepth / 4));
}

// The host-side image of the staged region: every table converted to the compute precision at the offset carve() gave it
// (relative to Work::stage_ofs).  `put(byte offset, table id, element count)` is supplied by the caller and copies table
// `id` (0-5: int tables, 6-14: real tables, in the order below) from wherever it keeps it.
template <class real, bool BIG, class Put>
inline void stage_image(const Work<real, BIG> &w, const Dims &d, int hct_size, int n_hand_full, Put put) {
    const uint32_t b = w.stage_ofs;
    put(w.c_parents.ofs - b, 0, size_t(d.nJ)); put(w.c_fk_order.ofs - b, 1, size_t(d.nJ));
    put(w.c_wj.ofs - b, 2, size_t(d.S) * d.kw); put(w.c_free1.ofs - b, 3, size_t(d.n1)); put(w.c_free2.ofs - b, 4, size_t(d.n2));
    put(w.c_pids.ofs - b, 5, size_t(d.D));
    put(w.c_wv.ofs - b, 6, size_t(d.S) * d.kw); put(w.c_v0.ofs - b, 7, size_t(3) * d.S); put(w.c_coefs.ofs - b, 8, size_t(3) * d.M);
    put(w.c_j0.ofs - b, 9, size_t(3) * d.nJ); put(w.c_hmean.ofs - b, 10, size_t(n_hand_full));
    put(w.c_pmeans.ofs - b, 11, size_t(d.K) * d.D); put(w.c_pnlw.ofs - b, 12, size_t(d.K));
    put(w.c_jd.ofs - b, 13, size_t(3) * d.nJ * d.nd); put(w.hct.ofs - b, 14, size_t(hct_size));
}

// configuration of one minimisation (one ch.minimize call of the reference)
template <class real>
struct StepCfg {
    const int *free;
    int n;
    real wp;          // prior weight (0: no prior term)
    real e3;
    bool velo, poseH, dm_terms, extrap;
    bool face;        // poseF (jaw) and expr terms (chmosh.py:685-687)
};

// ---------------------------------------------------------------------------------------------
// the solver
// ---------------------------------------------------------------------------------------------
template <class real, bool BIG = false>
struct Solver {
    const Model<real> &m;
    const Job<real> &job;
    const Work<real, BIG> &w;
    const Cta cta;
    const Dims &d;
    // per-frame scalars (identical in every thread)
    real wd, wp_frame, wH, wv, wdm, wex, wF, wxp;
    int nvis, njl;            // njl: joints whose full-pose columns the current step needs
    bool has_velo, has_extrap, hand_free;
    // counters of the current frame
    int n_iter, n_eval, n_build, n_min, frame_flags;
    int prof_base = 0;        // development builds: offset of the phase-timer slots
    bool fwd_at_x = false;    // the forward scratch of the latest evaluation belongs to the current state w.x ...
    bool fwd_has_prior = false;   // ... including the prior products
    bool resuming = false;    // boundary repair: the chunk continues from emitted rows (run_chunk)
    int root_turns = 0;       // full turns added to the angle of the cold start's root (run_chunk, procrustes)
    real resume_diff = 0;     // ... and how far the frame just solved is from the row it replaces
    int lin_f = -1;           // linearise mode: the frame this block works on (else -1)

    M2_D Solver(const Model<real> &m_, const Job<real> &j_, const Work<real, BIG> &w_, const Dims &d_, Cta c_)
        : m(m_), job(j_), w(w_), cta(c_), d(d_) {}

#define CTA_FOR(i, n) _Pragma("unroll 1") for (int i = cta.tid; i < (n); i += cta.nthr)

    // joint-position directions of the linear coefficients [nJ][3][nd]: staged in shared memory, or with BIG the model's own
    // table (carve() leaves them out of the staged region there)
    M2_D const real *jdir() const { return BIG ? m.jd : static_cast<const real *>(w.c_jd); }

    // ---- CTA-wide maximum of one per-thread value, broadcast (rare path: boundary repair)
    M2_D void cta_max(real *v) {
#if M2_GPU
        real x = v[0];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { const real y = __shfl_xor_sync(0xffffffffu, x, o); x = y > x ? y : x; }
        const int lane = cta.tid & 31, warp = cta.tid >> 5, nwarp = (cta.nthr + 31) >> 5;
        if (lane == 0) w.red[warp] = x;
        __syncthreads();
        if (cta.tid == 0) { real mx = w.red[0]; for (int q = 1; q < nwarp; ++q) mx = w.red[q] > mx ? w.red[q] : mx; w.red[32] = mx; }
        __syncthreads();
        v[0] = w.red[32];
        __syncthreads();
#else
        (void)v;
#endif
    }

    // ---- FK, executed by `nl` lanes (one warp on the GPU) starting at lane id `l`.  Every lane multiplies down the
    //      ancestor chain of its own joint (root first), which it reads as four words: no level-by-level hand-over
    //      through shared memory -- under the load of the pose-blend stream of the other warps a dependent shared-
    //      memory hop costs hundreds of cycles, and the level-wise walk chained three of them per level.  Same
    //      products in the same order as the level-wise recursion.
    M2_D void fk(int l, int nl) {
        for (int j = l; j < d.nJ; j += nl) {
            uint32_t cw[kMaxDepth / 4];
#pragma unroll
            for (int q = 0; q < kMaxDepth / 4; ++q) cw[q] = w.c_chain[j * (kMaxDepth / 4) + q];
            int prev = int(cw[0] & 255u);
            real R[9], t[3];
#pragma unroll
            for (int i = 0; i < 9; ++i) R[i] = w.Rl[9 * prev + i];
#pragma unroll
            for (int i = 0; i < 3; ++i) t[i] = w.Jp[3 * prev + i];
#pragma unroll
            for (int k = 1; k < kMaxDepth; ++k) {
                const int c = int((cw[k >> 2] >> (8 * (k & 3))) & 255u);
                if (c != 255) {
                    const real *Rc = w.Rl + 9 * c;
                    const real dj[3] = {w.Jp[3 * c] - w.Jp[3 * prev], w.Jp[3 * c + 1] - w.Jp[3 * prev + 1], w.Jp[3 * c + 2] - w.Jp[3 * prev + 2]};
                    real rc[9], o[9];
#pragma unroll
                    for (int i = 0; i < 9; ++i) rc[i] = Rc[i];
#pragma unroll
                    for (int i = 0; i < 3; ++i) t[i] += R[3 * i] * dj[0] + R[3 * i + 1] * dj[1] + R[3 * i + 2] * dj[2];
                    mat3_mul_reg(R, rc, o);
#pragma unroll
                    for (int i = 0; i < 9; ++i) R[i] = o[i];
                    prev = c;
                }
            }
#pragma unroll
            for (int i = 0; i < 9; ++i) w.Rg[9 * j + i] = R[i];
#pragma unroll
            for (int i = 0; i < 3; ++i) w.tg[3 * j + i] = t[i];
        }
    }

    // ---- pose-blend partial sums: item (joint group, slot) -> x,y,z of the slot; part[g][3 s + c] (aliases Jt).
    //      Lanes run over consecutive slots, so every warp load is one contiguous run of 16-byte vectors.
    M2_D int blend_groups(int nl) const {      // as many joint groups as fit one round of the nl blending threads
        const int per_group = 3 * ((d.S + 3) >> 2);
        int g = nl / per_group;
        return g < 1 ? 1 : (g > kBlendGroups ? kBlendGroups : g);
    }
    // item = (joint group, coordinate c, four consecutive slots): nine 16-byte loads per joint, no padding bytes; two
    // joints are in flight per thread
    M2_D void blend_partials(int l, int nl) {
        const int G = blend_groups(nl);
        const int per = (d.nJ - 1 + G - 1) / G;
        const int Sq = (d.S + 3) >> 2;
        const size_t cs = size_t(Sq) * 4;               // stride between the 27 (e, c) rows of a joint
        for (int it = l; it < 3 * Sq * G; it += nl) {
            const int g = it / (3 * Sq), rem = it - g * 3 * Sq, c = rem / Sq, sq = rem - c * Sq;
            int j0 = 1 + g * per, j1 = j0 + per;
            if (j1 > d.nJ) j1 = d.nJ;
            real acc[4] = {0, 0, 0, 0};
            for (int j = j0; j < j1; j += 2) {
                const bool two = j + 1 < j1;
                const real *P = m.pdc + (size_t(j - 1) * 27 + c) * cs + 4 * sq, *Q = P + (two ? 27 * cs : 0);
                Vec4<real> pa[9], pb[9];
#pragma unroll
                for (int e = 0; e < 9; ++e) pa[e] = ld4(P + 3 * e * cs);
#pragma unroll
                for (int e = 0; e < 9; ++e) pb[e] = ld4(Q + 3 * e * cs);
                const real *R = w.Rl + 9 * j, *R2 = R + (two ? 9 : 0);
                const real tw = two ? real(1) : real(0);
#pragma unroll
                for (int e = 0; e < 9; ++e) {
                    const real id = (e == 0 || e == 4 || e == 8) ? real(1) : real(0);
                    const real fa = R[e] - id, fb = (R2[e] - id) * tw;
                    acc[0] += pa[e].x * fa + pb[e].x * fb;
                    acc[1] += pa[e].y * fa + pb[e].y * fb;
                    acc[2] += pa[e].z * fa + pb[e].z * fb;
                    acc[3] += pa[e].w * fa + pb[e].w * fb;
                }
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int sl = 4 * sq + q;
                if (sl < d.S) w.Jt[(g * d.S + sl) * 3 + c] = acc[q];
            }
        }
    }

    // ---- forward evaluation at state xs; leaves SSE terms in w.sc[0..6], argmin component in w.isc[0]
    //      `reuse`: the forward scratch of the previous evaluation already belongs to this state (the last trial step was
    //      accepted, so x = that trial point): only the terms that depend on the frame's observations, weights and targets
    //      are computed again -- same numbers as a full evaluation, since the forward depends on the state alone.
    M2_D void eval(const real *xs, const StepCfg<real> &c, bool reuse = false) {
        ++n_eval;
        M2_T0();
        const real *th = xs + 3;
        const real *dl = xs + 3 + d.PR;
        if (!reuse) {
        CTA_FOR(i, d.PF) {
            real v;
            if (i < m.body_dof) {
                v = th[i];
            } else {
                const int q = i - m.body_dof;
                v = w.c_hmean[q];
                for (int b = 0; b < m.hb_n; ++b) {
                    const HandBlock hb = m.hb[b];
                    if (q >= hb.q0 && q < hb.q1) {
                        const real *ct = w.hct + hb.ct_off + (q - hb.q0) * hb.rw4;
                        for (int r = hb.r0; r < hb.r1; ++r) v += th[m.body_dof + r] * ct[r - hb.r0];
                    }
                }
            }
            w.fullpose[i] = v;
        }
        CTA_FOR(i, 3 * d.nJ) {
            real v = w.c_j0[i];
            for (int q = 0; q < d.nd; ++q) v += jdir()[i * d.nd + q] * dl[q];
            w.Jp[i] = v;
        }
        CTA_FOR(i, d.D) w.pxg[i] = th[w.c_pids[i]];          // the pose coefficients the prior sees, in its own order
        M2_SYNC();
        M2_TACC(0);
#if M2_GPU
        CTA_FOR(jk, 3 * d.nJ) { const int j = jk / 3; rodrigues(w.fullpose + 3 * j, w.Rl + 9 * j, w.dRl + kDR * j, jk - 3 * j); }
#else
        CTA_FOR(j, d.nJ) rodrigues(w.fullpose + 3 * j, w.Rl + 9 * j, w.dRl + kDR * j);
#endif
        M2_SYNC();
        M2_TACC(1);
#if M2_GPU
        const int nblend = cta.nthr > 64 ? cta.nthr - 32 : cta.nthr;
        if (cta.nthr > 64) {                      // warp 0 walks the kinematic tree while the others blend
            if (cta.tid < 32) {
                fk(cta.tid, 32);
#if defined(MOSH2_PROFILE)
                if (cta.tid == 0) w.prof[18 + prof_base] += clock64() - t_prev_;      // the kinematic-tree walk alone
#endif
            } else blend_partials(cta.tid - 32, nblend);
        } else {
            fk(cta.tid, cta.nthr); __syncthreads(); blend_partials(cta.tid, nblend);
        }
#else
        const int nblend = 1;
        fk(0, 1);
        blend_partials(0, 1);
#endif
        const int nbg = blend_groups(nblend);
        M2_SYNC();
        M2_TACC(2);
        // max-mixture prior: y_k = Q_k (x - mu_k).  GPU: an item is four rows of one component times a quarter of the
        // columns -- sixteen independent 16-byte loads down the transposed copy of Q, all in flight at once (the
        // product is bound by load latency, not by bytes); four adjacent lanes then add their quarters by shuffles.
        if (c.wp > real(0)) {
            const int D = d.D, D4 = d.D4;
            const real *xb = w.pxg;
#if M2_GPU
            const int nq = D4 >> 2, lchunk = (D + 3) >> 2;          // row quads per component, columns per quarter
            const int nitem = d.K * nq * 4, nround = (nitem + cta.nthr - 1) / cta.nthr;
#pragma unroll 1
            for (int rd = 0; rd < nround; ++rd) {
                const int it = rd * cta.nthr + cta.tid, lr = it & 3, kq = it >> 2;
                const bool on = it < nitem;
                const int k = on ? kq / nq : 0, quad = on ? kq - k * nq : 0;
                const int l0 = lr * lchunk, l1 = (l0 + lchunk < D) ? l0 + lchunk : D;
                const real *Q = m.prior_Qt + (size_t(k) * D + l0) * D4 + 4 * quad, *mu = w.c_pmeans + k * D;
                real s0 = 0, s1 = 0, s2 = 0, s3 = 0;
                for (int lb = l0; on && lb < l1; lb += 16) {        // blocks of sixteen columns: a fixed trip count, so the
                    Vec4<real> q4[16];                              // sixteen loads issue back to back (predicated tail)
#pragma unroll
                    for (int u = 0; u < 16; ++u) {
                        if (lb + u < l1) q4[u] = ld4(Q + size_t(lb + u - l0) * D4);
                        else q4[u].x = q4[u].y = q4[u].z = q4[u].w = 0;
                    }
#pragma unroll
                    for (int u = 0; u < 16; ++u) {
                        const int l = (lb + u < l1) ? lb + u : l0;
                        const real dx = xb[l] - mu[l];
                        s0 += q4[u].x * dx; s1 += q4[u].y * dx; s2 += q4[u].z * dx; s3 += q4[u].w * dx;
                    }
                }
#pragma unroll
                for (int off = 1; off <= 2; off <<= 1) {
                    s0 += __shfl_xor_sync(0xffffffffu, s0, off); s1 += __shfl_xor_sync(0xffffffffu, s1, off);
                    s2 += __shfl_xor_sync(0xffffffffu, s2, off); s3 += __shfl_xor_sync(0xffffffffu, s3, off);
                }
                if (on && lr == 0) {
                    const int i0 = 4 * quad;
                    real *o = w.py + k * D + i0;
                    if (i0 < D) o[0] = s0;
                    if (i0 + 1 < D) o[1] = s1;
                    if (i0 + 2 < D) o[2] = s2;
                    if (i0 + 3 < D) o[3] = s3;
                }
            }
#else
            for (int idx = 0; idx < d.K * D; ++idx) {
                const int k = idx / D, i = idx - k * D;
                const real *Q = m.prior_Qt + size_t(k) * D * D4 + i, *mu = w.c_pmeans + k * D;
                real s = 0;
                for (int l = 0; l < D; ++l) s += Q[size_t(l) * D4] * (xb[l] - mu[l]);
                w.py[idx] = s;
            }
#endif
        }
#if defined(MOSH2_PROFILE) && M2_GPU
        __syncthreads();
        M2_TACC(19);                                   // development: the prior products alone
#endif
        // skinning of the 3M slots
        CTA_FOR(s, d.S) {
            real vpo[3];
#pragma unroll
            for (int q = 0; q < 3; ++q) vpo[q] = w.c_v0[3 * s + q];
            // linear directions (DMPL, expressions): blocks of eight coefficients with a fixed trip count, so that the
            // 24 (L2) loads of a block issue back to back
            for (int e0 = 0; e0 < d.nd; e0 += 8) {
                real sv[24];
#pragma unroll
                for (int u = 0; u < 24; ++u) {
                    const int q = u >> 3, e = e0 + (u & 7);
                    sv[u] = e < d.nd ? m.sd[(3 * s + q) * d.nd + e] : real(0);
                }
#pragma unroll
                for (int u = 0; u < 24; ++u) {
                    const int e = e0 + (u & 7);
                    vpo[u >> 3] += sv[u] * (e < d.nd ? dl[e] : real(0));
                }
            }
            for (int q = 0; q < 3; ++q)
                for (int g = 0; g < nbg; ++g) vpo[q] += w.Jt[(g * d.S + s) * 3 + q];
            real v[3] = {0, 0, 0};
            real Rs[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
            for (int i = 0; i < d.kw; ++i) {
                const int j = w.c_wj[s * d.kw + i];
                real *pp = w.pj + 3 * (s * d.kw + i);
                if (j < 0) { pp[0] = pp[1] = pp[2] = 0; continue; }
                const real wt = w.c_wv[s * d.kw + i];
                real dv[3] = {vpo[0] - w.Jp[3 * j], vpo[1] - w.Jp[3 * j + 1], vpo[2] - w.Jp[3 * j + 2]};
                real o[3];
                mat3_vec(w.Rg + 9 * j, dv, o);
                for (int q = 0; q < 3; ++q) {
                    pp[q] = o[q] + w.tg[3 * j + q];
                    v[q] += wt * pp[q];
                }
                for (int q = 0; q < 9; ++q) Rs[q] += wt * w.Rg[9 * j + q];
            }
            for (int q = 0; q < 3; ++q) w.vp[3 * s + q] = v[q] + xs[q];
            for (int q = 0; q < 9; ++q) w.Rsk[9 * s + q] = Rs[q];
        }
        M2_SYNC();
        M2_TACC(3);
        }   // !reuse
        // simulated markers and data residual (transformed_lm.py:130-159); the prior products share the phase
        if (reuse) {
            CTA_FOR(mi, d.M) {
                const bool vis = w.vis[mi] != 0;
                for (int q = 0; q < 3; ++q) w.rm[3 * mi + q] = vis ? (w.mk[3 * mi + q] - w.obs[3 * mi + q]) * wd : real(0);
            }
        } else
        CTA_FOR(mi, d.M) {
            const real *v0 = w.vp + 9 * mi, *v1 = v0 + 3, *v2 = v0 + 6;
            real e1[3] = {v1[0] - v0[0], v1[1] - v0[1], v1[2] - v0[2]};
            real e2[3] = {v2[0] - v0[0], v2[1] - v0[1], v2[2] - v0[2]};
            const real n1 = r_sqrt(e1[0] * e1[0] + e1[1] * e1[1] + e1[2] * e1[2]);
            real f1[3] = {e1[0] / n1, e1[1] / n1, e1[2] / n1};
            real nn[3];
            cross3(e1, e2, nn);
            const real n2 = r_sqrt(nn[0] * nn[0] + nn[1] * nn[1] + nn[2] * nn[2]);
            real f2[3] = {nn[0] / n2, nn[1] / n2, nn[2] / n2};
            real f3[3];
            cross3(f1, f2, f3);
            const real k1 = w.c_coefs[3 * mi], k2 = w.c_coefs[3 * mi + 1], k3 = w.c_coefs[3 * mi + 2];
            const bool vis = w.vis[mi] != 0;
            for (int q = 0; q < 3; ++q) {
                const real mk = v0[q] + k1 * f1[q] + k2 * f2[q] + k3 * f3[q];
                w.mk[3 * mi + q] = mk;
                w.rm[3 * mi + q] = vis ? (mk - w.obs[3 * mi + q]) * wd : real(0);
            }
        }
        M2_SYNC();
        M2_TACC(4);
        if (c.wp > real(0)) {                  // q_k = (x - mu_k)^T y_k - log w_k, one warp per component
#if M2_GPU
            const int lane = cta.tid & 31, warp = cta.tid >> 5, nwarp = cta.nthr >> 5;
            for (int k = warp; k < d.K; k += nwarp) {
                const real *mu = w.c_pmeans + k * d.D;
                real sacc = 0;
                for (int i = lane; i < d.D; i += 32) sacc += (w.pxg[i] - mu[i]) * w.py[k * d.D + i];
                sacc = warp_sum(sacc);
                if (lane == 0) w.pq[k] = sacc + w.c_pnlw[k];
            }
#else
            for (int k = 0; k < d.K; ++k) {
                const real *mu = w.c_pmeans + k * d.D;
                real sacc = w.c_pnlw[k];
                for (int i = 0; i < d.D; ++i) sacc += (w.pxg[i] - mu[i]) * w.py[k * d.D + i];
                w.pq[k] = sacc;
            }
#endif
        }
        real part[N_ERR] = {0, 0, 0, 0, 0, 0, 0, 0};
        const int nd_dm = d.nd - m.n_expr;             // DMPL coefficients come first, expressions after them
        CTA_FOR(i, 3 * d.M) part[ERR_DATA] += w.rm[i] * w.rm[i];
        if (c.velo) CTA_FOR(i, d.PR) { const real e = (th[i] - w.velo_tgt[i]) * wv; part[ERR_VELO] += e * e; }
        if (c.poseH) CTA_FOR(i, m.finger_hi - m.finger_lo) { const real e = th[m.finger_lo + i] * wH; part[ERR_POSEH] += e * e; }
        // joint-angle term of the horse model: r_i = 2 wp exp(2 s_i x_i) (chmosh.py:615-617: power(exp(.), 2) * wt_pose * 2);
        // animal models have no finger term, its column carries this one
        if (c.wp > real(0)) CTA_FOR(i, m.n_jang) { const real e = real(2) * c.wp * r_exp(real(2) * m.jang_sign[i] * th[m.jang_id[i]]); part[ERR_POSEH] += e * e; }
        if (c.face) {
            CTA_FOR(i, m.face_hi - m.face_lo) { const real e = th[m.face_lo + i] * wF; part[ERR_POSEF] += e * e; }
            CTA_FOR(i, m.n_expr) { const real e = dl[nd_dm + i] * wxp; part[ERR_EXPR] += e * e; }
        }
        if (c.dm_terms) CTA_FOR(i, nd_dm) {
            const real e = dl[i] * wdm;
            part[ERR_DMPL] += e * e;
            if (c.extrap) { const real e2 = (dl[i] - w.dm_tgt[i]) * wex; part[ERR_EXTRAP] += e2 * e2; }
        }
        cta_reduce<real, N_ERR>(cta, part, w.red);
        if (cta.tid == 0) {
            int ks = 0;
            real sp = 0;
            if (c.wp > real(0)) {
                for (int k = 1; k < d.K; ++k) if (w.pq[k] < w.pq[ks]) ks = k;
                sp = c.wp * c.wp * w.pq[ks];
            }
            w.isc[0] = ks;
            part[ERR_POSEB] = sp;
            real tot = 0;
            for (int i = 0; i < N_ERR; ++i) { w.sc[1 + i] = part[i]; tot += part[i]; }
            w.sc[0] = tot;
        }
        M2_SYNC();
        M2_TACC(5);
    }

    // ---- local 3x9 Jacobian of a marker wrt its three (skinned) vertices, at the latest eval()
    M2_D void marker_local_jacobian(int mi) {
        const real *v0 = w.vp + 9 * mi, *v1 = v0 + 3, *v2 = v0 + 6;
        real e1[3] = {v1[0] - v0[0], v1[1] - v0[1], v1[2] - v0[2]};
        real e2[3] = {v2[0] - v0[0], v2[1] - v0[1], v2[2] - v0[2]};
        const real n1 = r_sqrt(e1[0] * e1[0] + e1[1] * e1[1] + e1[2] * e1[2]);
        real f1[3] = {e1[0] / n1, e1[1] / n1, e1[2] / n1};
        real nn[3];
        cross3(e1, e2, nn);
        const real n2 = r_sqrt(nn[0] * nn[0] + nn[1] * nn[1] + nn[2] * nn[2]);
        real f2[3] = {nn[0] / n2, nn[1] / n2, nn[2] / n2};
        const real k1 = w.c_coefs[3 * mi], k2 = w.c_coefs[3 * mi + 1], k3 = w.c_coefs[3 * mi + 2];
        // d marker / d(e1, e2):  N(u) = (I - uh uh^T)/|u|
        real N1[9], Nn[9];
        for (int r = 0; r < 3; ++r)
            for (int q = 0; q < 3; ++q) {
                N1[3 * r + q] = ((r == q ? real(1) : real(0)) - f1[r] * f1[q]) / n1;
                Nn[3 * r + q] = ((r == q ? real(1) : real(0)) - f2[r] * f2[q]) / n2;
            }
        const real Se1[9] = {0, -e1[2], e1[1], e1[2], 0, -e1[0], -e1[1], e1[0], 0};
        const real Se2[9] = {0, -e2[2], e2[1], e2[2], 0, -e2[0], -e2[1], e2[0], 0};
        const real Sf1[9] = {0, -f1[2], f1[1], f1[2], 0, -f1[0], -f1[1], f1[0], 0};
        const real Sf2[9] = {0, -f2[2], f2[1], f2[2], 0, -f2[0], -f2[1], f2[0], 0};
        real df2e1[9], df2e2[9], t1[9], t2[9], df3e1[9], df3e2[9];
        mat3_mul_reg(Nn, Se2, df2e1);                       // d f2/d e1 = N(n) (-[e2]x)
        for (int q = 0; q < 9; ++q) df2e1[q] = -df2e1[q];
        mat3_mul_reg(Nn, Se1, df2e2);                       // d f2/d e2 = N(n) [e1]x
        mat3_mul_reg(Sf2, N1, t1);                          // d f3/d e1 = -[f2]x N1 + [f1]x df2e1
        mat3_mul_reg(Sf1, df2e1, t2);
        for (int q = 0; q < 9; ++q) df3e1[q] = t2[q] - t1[q];
        mat3_mul_reg(Sf1, df2e2, df3e2);
        real *L = w.Loc + 3 * kM3 * mi;                    // three padded 3x3 blocks: d marker / d vertex t
        for (int q = 0; q < 9; ++q) {
            const real de1 = k1 * N1[q] + k2 * df2e1[q] + k3 * df3e1[q];
            const real de2 = k2 * df2e2[q] + k3 * df3e2[q];
            const real id = (q == 0 || q == 4 || q == 8) ? real(1) : real(0);
            L[q] = id - de1 - de2;
            L[kM3 + q] = de1;
            L[2 * kM3 + q] = de2;
        }
    }

    // ---- the padded 3x3 matrices of slot sl in registers: MtR (pose-blend part of T1) and Loc (rigid part)
    M2_D void slot_mats(int sl, real (&Mt)[9], real (&Lc)[9]) {
        const real *Mp = w.MtR + kM3 * sl, *Lp = w.Loc + kM3 * sl;
        const Vec4<real> m0 = ld4(Mp), m1 = ld4(Mp + 4), m2 = ld4(Mp + 8), l0 = ld4(Lp), l1 = ld4(Lp + 4), l2 = ld4(Lp + 8);
        Mt[0] = m0.x; Mt[1] = m0.y; Mt[2] = m0.z; Mt[3] = m0.w; Mt[4] = m1.x; Mt[5] = m1.y; Mt[6] = m1.z; Mt[7] = m1.w; Mt[8] = m2.x;
        Lc[0] = l0.x; Lc[1] = l0.y; Lc[2] = l0.z; Lc[3] = l0.w; Lc[4] = l1.x; Lc[5] = l1.y; Lc[6] = l1.z; Lc[7] = l1.w; Lc[8] = l2.x;
    }

    // ---- T1: the part of slot sl (marker sl / 3, vertex sl % 3) in the 3x3 Jacobian block of joint a, blk[3 r + k] (row r,
    //      rotation axis k).  Mt, Lc: slot_mats(sl); Pslot: the slot's pose-blend vectors, m.pd4 + 4 sl.
    M2_D void slot_pose_block(int sl, int a, const real (&Mt)[9], const real (&Lc)[9], const real *Pslot, real (&blk)[9]) {
        const int mask = w.c_amask[sl * d.nJ + a];          // the slot's skinning joints in the subtree of a
#pragma unroll
        for (int q = 0; q < 9; ++q) blk[q] = 0;
        if (a >= 1) {
            // pose-blend part: E[c][k] = sum_e Pd[c][e] dR_k[e], then blk = (Loc_t Rsk_s) E
            // (requesting the NEXT joint's vectors here, right after E has consumed the current ones, was
            // measured slower: the loop is bound by instruction issue -- about 500 warp instructions per
            // joint, a quarter of them FMAs -- not by the latency of these loads)
            const size_t es = size_t(d.S) * 4;
            const real *P = Pslot + size_t(a - 1) * 9 * es;
            Vec4<real> pv[9];
#pragma unroll
            for (int e = 0; e < 9; ++e) pv[e] = ld4(P + e * es);
            const real *dR = w.dRl + kDR * a;
            real dr[kDR];
#pragma unroll
            for (int v = 0; v < kDR / 4; ++v) {
                const Vec4<real> q4 = ld4(dR + 4 * v);
                dr[4 * v] = q4.x; dr[4 * v + 1] = q4.y; dr[4 * v + 2] = q4.z; dr[4 * v + 3] = q4.w;
            }
            real E[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
            for (int e = 0; e < 9; ++e) {
                const real q0 = dr[e], q1 = dr[9 + e], q2 = dr[18 + e];
                E[0] += pv[e].x * q0; E[1] += pv[e].x * q1; E[2] += pv[e].x * q2;
                E[3] += pv[e].y * q0; E[4] += pv[e].y * q1; E[5] += pv[e].y * q2;
                E[6] += pv[e].z * q0; E[7] += pv[e].z * q1; E[8] += pv[e].z * q2;
            }
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int k = 0; k < 3; ++k)
                    blk[3 * r + k] = Mt[3 * r] * E[k] + Mt[3 * r + 1] * E[3 + k] + Mt[3 * r + 2] * E[6 + k];
        }
        // rigid part: the slot's skinning joints below a turn about a:  d v / d omega_{a,k} = u_{a,k} x q
        if (mask) {
            real q[3] = {0, 0, 0};
            if (d.kw == 4) {
                // four skinning joints per slot (every released model): weights and joint-relative positions
                // of the slot as four 16-byte vectors, the subtree mask applied to the weights -- no branches
                const Vec4<real> wv = ld4(w.c_wv + 4 * sl);
                const real *pp = w.pj + 12 * sl;
                const Vec4<real> a0 = ld4(pp), a1 = ld4(pp + 4), a2 = ld4(pp + 8);
                const real g0 = w.tg[3 * a], g1 = w.tg[3 * a + 1], g2 = w.tg[3 * a + 2];
                const real w0 = (mask & 1) ? wv.x : real(0), w1 = (mask & 2) ? wv.y : real(0);
                const real w2 = (mask & 4) ? wv.z : real(0), w3 = (mask & 8) ? wv.w : real(0);
                q[0] = w0 * (a0.x - g0); q[1] = w0 * (a0.y - g1); q[2] = w0 * (a0.z - g2);
                q[0] += w1 * (a0.w - g0); q[1] += w1 * (a1.x - g1); q[2] += w1 * (a1.y - g2);
                q[0] += w2 * (a1.z - g0); q[1] += w2 * (a1.w - g1); q[2] += w2 * (a2.x - g2);
                q[0] += w3 * (a2.y - g0); q[1] += w3 * (a2.z - g1); q[2] += w3 * (a2.w - g2);
            } else
                for (int i = 0; i < d.kw; ++i)
                    if ((mask >> i) & 1) {
                        const real wt = w.c_wv[sl * d.kw + i];
                        const real *pp = w.pj + 3 * (sl * d.kw + i);
                        for (int r = 0; r < 3; ++r) q[r] += wt * (pp[r] - w.tg[3 * a + r]);
                    }
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const Vec4<real> uk = ld4(w.u + kM3 * a + 4 * k);
                const real uv[3] = {uk.x, uk.y, uk.z};
                real cr[3];
                cross3(uv, q, cr);
#pragma unroll
                for (int r = 0; r < 3; ++r) blk[3 * r + k] += Lc[3 * r] * cr[0] + Lc[3 * r + 1] * cr[1] + Lc[3 * r + 2] * cr[2];
            }
        }
    }

    // ---- the three residual rows of marker `ml` of the tile (already weighted) in free-variable column `col`
    M2_D void jf_store3(int ml, int col, real v0, real v1, real v2) {
        real *J = w.Jf + 3 * ml * d.npad + col;
        J[0] = v0; J[d.npad] = v1; J[2 * d.npad] = v2;
    }

    // ---- column k (rows b0, b1, b2) of the finished 3x3 T1 block of marker `ml` of the tile and joint a: body joints go
    //      straight to their free column of the tile, weighted by sc (wd, or 0 for an invisible marker); hand joints go to
    //      the full-pose tile for the PCA chain (T2b)
    M2_D void pose_col_store(int ml, int a, int k, real sc, real b0, real b1, real b2) {
        if (3 * a < m.body_dof) {
            const int col = w.colmap[3 + 3 * a + k];
            if (col >= 0) jf_store3(ml, col, b0 * sc, b1 * sc, b2 * sc);
        } else {
            real *Jr = w.Jt + 3 * ml * d.NCt + (3 * a - m.body_dof) + k;
            Jr[0] = b0; Jr[d.NCt] = b1; Jr[2 * d.NCt] = b2;
        }
    }

    // ---- u_{a,k} = Rg_par(a) vee(dR_{a,k} R_a^T), the rotation axes of the rigid part of T1
    M2_D void joint_axes() {
        CTA_FOR(idx, 3 * d.nJ) {
            const int a = idx / 3, k = idx - 3 * a;
            const real *D = w.dRl + kDR * a + 9 * k, *R = w.Rl + 9 * a;
            real om[3];     // vee(dR R^T)
            om[0] = D[6] * R[3] + D[7] * R[4] + D[8] * R[5];
            om[1] = D[0] * R[6] + D[1] * R[7] + D[2] * R[8];
            om[2] = D[3] * R[0] + D[4] * R[1] + D[5] * R[2];
            const int par = w.c_parents[a];
            real *uo = w.u + kM3 * a + 4 * k;
            if (par < 0) { for (int q = 0; q < 3; ++q) uo[q] = om[q]; }
            else mat3_vec(w.Rg + 9 * par, om, uo);
        }
    }

    // ---- d tg_j / d delta_i = d tg_par + Rg_par (Jd_j - Jd_par): every (joint, coefficient) item sums down the joint's own
    //      ancestor chain (root first, the order of the level-wise recursion), so there is no barrier per tree level
    M2_D void dtg_chains() {
        if (!d.nd) return;
        CTA_FOR(q, d.nJ * d.nd) {
            const int j = q / d.nd, i = q - j * d.nd;
            uint32_t cw[kMaxDepth / 4];
#pragma unroll
            for (int u = 0; u < kMaxDepth / 4; ++u) cw[u] = w.c_chain[j * (kMaxDepth / 4) + u];
            int prev = int(cw[0] & 255u);
            real acc[3];
            for (int r = 0; r < 3; ++r) acc[r] = jdir()[(3 * prev + r) * d.nd + i];
            for (int k = 1; k < kMaxDepth; ++k) {
                const int cj = int((cw[k >> 2] >> (8 * (k & 3))) & 255u);
                if (cj == 255) break;
                real dj[3], t[3];
                for (int r = 0; r < 3; ++r) dj[r] = jdir()[(3 * cj + r) * d.nd + i] - jdir()[(3 * prev + r) * d.nd + i];
                mat3_vec(w.Rg + 9 * prev, dj, t);
                for (int r = 0; r < 3; ++r) acc[r] = acc[r] + t[r];
                prev = cj;
            }
            real *o = w.dtg + 3 * (j * d.nd + i);
            for (int r = 0; r < 3; ++r) o[r] = acc[r];
        }
    }

    // ---- T1: full-pose 3x3 Jacobian blocks (marker, joint) of the tile's tm markers from t0 on, for the joints this step
    //      needs.  A block is the sum over the marker's three slots; on the GPU three adjacent lanes take one slot each (their
    //      pose-blend vectors are adjacent in memory) and are summed with two shuffles.
    M2_D void tile_pose_columns(int t0, int tm) {
#if M2_GPU
        // A warp owns up to ten markers of the tile (lane = marker vertex: 30 lanes) and walks a strided share
        // of the joints, so everything that belongs to the slot stays in registers.  The three partial 3x3
        // blocks of a marker are summed by rotation -- lane t ends up with column t -- and every lane stores
        // its own column.
        const int lane = cta.tid & 31, warp = cta.tid >> 5, nwarp = cta.nthr >> 5;
        const int t = lane % 3, grp = lane / 3;
        const int nmg = (tm + 9) / 10, nch = nwarp / nmg;         // marker groups, joint shares
        const int mg = warp % nmg, ch = warp / nmg;
        const int ml = mg * 10 + grp;
        const bool valid = lane < 30 && ml < tm;
        if (ch < nch) {
            const int mi = t0 + (valid ? ml : 0), sl = 3 * mi + t;
            const real sc = (valid && w.vis[mi]) ? wd : real(0);
            real Mt[9], Lc[9];
            slot_mats(sl, Mt, Lc);
            const real *Pslot = m.pd4 + size_t(sl) * 4;
            const int src1 = lane - t + (t + 2) % 3, src2 = lane - t + (t + 1) % 3;   // lanes whose t is t-1, t-2 (mod 3)
#pragma unroll 1
            for (int ji = ch; ji < njl; ji += nch) {
                const int a = w.jlist[ji];
                real blk[9];
                slot_pose_block(sl, a, Mt, Lc, Pslot, blk);
                // lane t collects column t of the marker's block: own part + the parts of the two other vertices
                real col3[3];
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const real b0 = blk[3 * r], b1 = blk[3 * r + 1], b2 = blk[3 * r + 2];
                    // (two selects each; written as nested conditionals the compiler turned them into three divergent
                    // branches per row -- every warp holds all three values of t)
                    const real own = sel3(t, b0, b1, b2);
                    const real to1 = sel3(t, b1, b2, b0);
                    const real to2 = sel3(t, b2, b0, b1);
                    col3[r] = own + __shfl_sync(0xffffffffu, to1, src1) + __shfl_sync(0xffffffffu, to2, src2);
                }
                if (valid) pose_col_store(ml, a, t, sc, col3[0], col3[1], col3[2]);
            }
        }
#else
        for (int gi = 0; gi < tm * njl; ++gi) {
            const int ml = gi % tm, a = w.jlist[gi / tm], mi = t0 + ml;
            real blk[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
            for (int t = 0; t < 3; ++t) {
                const int sl = 3 * mi + t;
                real Mt[9], Lc[9], part[9];
                slot_mats(sl, Mt, Lc);
                slot_pose_block(sl, a, Mt, Lc, m.pd4 + size_t(sl) * 4, part);
                for (int q = 0; q < 9; ++q) blk[q] += part[q];
            }
            const real sc = w.vis[mi] ? wd : real(0);
            for (int k = 0; k < 3; ++k) pose_col_store(ml, a, k, sc, blk[k], blk[3 + k], blk[6 + k]);
        }
#endif
    }

    // ---- linear-block (DMPL / expression) columns of the tile, from the vertex directions `sd` and the joint-position
    //      derivatives of dtg_chains()
    M2_D void tile_linear_columns(int t0, int tm) {
        CTA_FOR(it, tm * d.nd) {
            const int ml = it / d.nd, i = it - ml * d.nd, mi = t0 + ml;
            real val[3] = {0, 0, 0};
            real sdv[9];                              // the nine (L2) loads of the item, issued together
#pragma unroll
            for (int u = 0; u < 9; ++u) sdv[u] = m.sd[(9 * mi + u) * d.nd + i];
            for (int t = 0; t < 3; ++t) {
                const int s = 3 * mi + t;
                real dv[3] = {0, 0, 0};
                for (int kk = 0; kk < d.kw; ++kk) {
                    const int j = w.c_wj[s * d.kw + kk];
                    if (j < 0) continue;
                    const real wt = w.c_wv[s * d.kw + kk];
                    real df[3], o[3];
                    for (int r = 0; r < 3; ++r) df[r] = sdv[3 * t + r] - jdir()[(3 * j + r) * d.nd + i];
                    mat3_vec(w.Rg + 9 * j, df, o);
                    for (int r = 0; r < 3; ++r) dv[r] += wt * (o[r] + w.dtg[3 * (j * d.nd + i) + r]);
                }
                const real *L = w.Loc + kM3 * s;
                for (int r = 0; r < 3; ++r) val[r] += L[3 * r] * dv[0] + L[3 * r + 1] * dv[1] + L[3 * r + 2] * dv[2];
            }
            const int col = w.colmap[3 + d.PR + i];
            const real sc = w.vis[mi] ? wd : real(0);
            if (col >= 0) jf_store3(ml, col, val[0] * sc, val[1] * sc, val[2] * sc);
        }
    }

    // ---- translation columns of the tile (identity) and the zero padding of its rows beyond the n free columns
    M2_D void tile_translation_columns(int t0, int tm, int n) {
        CTA_FOR(idx, tm * 3) {
            const int ml = idx / 3, q = idx - 3 * ml, col = w.colmap[q];
            const real v = w.vis[t0 + ml] ? wd : real(0);
            if (col >= 0) jf_store3(ml, col, q == 0 ? v : real(0), q == 1 ? v : real(0), q == 2 ? v : real(0));
        }
        const int npadc = d.npad - n;
        CTA_FOR(idx, 3 * tm * npadc) w.Jf[(idx / npadc) * d.npad + n + idx % npadc] = 0;
    }

    // ---- T2b: hand columns = Jt[:, hand block] * C^T as a register-tiled product (one marker's 3 rows x 4 outputs)
    M2_D void tile_hand_columns(int t0, int tm) {
        if (!hand_free) return;
        int ngt = 0;                                  // output groups of 4 over all blocks
        for (int b = 0; b < m.hb_n; ++b) ngt += m.hb[b].rw4 / 4;
        CTA_FOR(it, tm * ngt) {
            const int ml = it / ngt;
            int rg = it - ml * ngt, b = 0;
            while (rg >= m.hb[b].rw4 / 4) { rg -= m.hb[b].rw4 / 4; ++b; }
            const HandBlock hb = m.hb[b];
            const int nq = hb.q1 - hb.q0;
            const real *J0 = w.Jt + 3 * ml * d.NCt + hb.q0, *J1 = J0 + d.NCt, *J2 = J1 + d.NCt;
            const real *ct = w.hct + hb.ct_off + 4 * rg;
            real acc[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
            // (global-workspace layout: the full-pose tile lives in L2 -- five columns in flight; same order of the sums)
            constexpr int U = BIG ? 5 : 1;
            for (int q = 0; q < nq; q += U) {
                real j0[U], j1[U], j2[U];
                Vec4<real> cv[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int qq = q + u < nq ? q + u : nq - 1;
                    j0[u] = J0[qq]; j1[u] = J1[qq]; j2[u] = J2[qq];
                    cv[u] = ld4(ct + qq * hb.rw4);
                }
#pragma unroll
                for (int u = 0; u < U; ++u)
                    if (q + u < nq) {
                        acc[0] += j0[u] * cv[u].x; acc[1] += j0[u] * cv[u].y; acc[2] += j0[u] * cv[u].z; acc[3] += j0[u] * cv[u].w;
                        acc[4] += j1[u] * cv[u].x; acc[5] += j1[u] * cv[u].y; acc[6] += j1[u] * cv[u].z; acc[7] += j1[u] * cv[u].w;
                        acc[8] += j2[u] * cv[u].x; acc[9] += j2[u] * cv[u].y; acc[10] += j2[u] * cv[u].z; acc[11] += j2[u] * cv[u].w;
                    }
            }
            const real sc = w.vis[t0 + ml] ? wd : real(0);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = hb.r0 + 4 * rg + e;
                if (r < hb.r1) {
                    const int col = w.colmap[3 + m.body_dof + r];
                    if (col >= 0) jf_store3(ml, col, acc[e] * sc, acc[4 + e] * sc, acc[8 + e] * sc);
                }
            }
        }
    }

#if M2_GPU
    // ---- A += the 16x16 block at (i0, j0) of the upper triangle that the calling warp holds in the layout of the mma
    //      accumulators: c[mi][ni][e] is entry (i0 + 8 mi + g, j0 + 8 ni + 2 tq + e), g = lane / 4, tq = lane % 4.  The old
    //      values are fetched together (in the global-workspace layout A lives in L2, and sixteen read-modify-writes one
    //      after the other cost a launch's worth of latency per tile: that, not the product, was the phase); the mirror
    //      entry receives the same sum -- it has received the same terms.
    M2_D void add_upper_block16(int i0, int j0, int n, const real (&c)[2][2][2]) {
        const int lane = cta.tid & 31, g = lane >> 2, tq = lane & 3, ld = d.lda;
        real old[2][2][2];
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int ni = 0; ni < 2; ++ni)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int i = i0 + 8 * mi + g, j = j0 + 8 * ni + 2 * tq + e;
                    old[mi][ni][e] = (j < n && i <= j) ? w.A[i * ld + j] : real(0);
                }
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int ni = 0; ni < 2; ++ni)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int i = i0 + 8 * mi + g, j = j0 + 8 * ni + 2 * tq + e;
                    if (j < n && i <= j) {
                        const real v = old[mi][ni][e] + c[mi][ni][e];
                        w.A[i * ld + j] = v;
                        if (i < j) w.A[j * ld + i] = v;
                    }
                }
    }
#endif

    // ---- T3: A += Jf^T Jf, g -= Jf^T r over the tile's rows; in linearise mode the finished rows go out first, as they are
    M2_D void tile_normal_equations(int t0, int tm, int n) {
        const int trows = 3 * tm, ld = d.lda;
        if (lin_f >= 0 && job.lin_J) {
            real *Jo = job.lin_J + (size_t(lin_f) * 3 * d.M + 3 * t0) * n;
            CTA_FOR(idx, trows * n) { const int row = idx / n, cc = idx - row * n; Jo[idx] = w.Jf[row * d.npad + cc]; }
        }
#if M2_GPU
        if constexpr (sizeof(real) == 8) {
            // float64: J^T J on the tensor cores as well -- mma.sync m8n8k4 (DMMA), a warp per 16x16 block of the upper
            // triangle, K = the tile's rows in steps of four.  The FP64 pipe of the CUDA cores issues one warp
            // instruction per ~25 cycles and SM sub-partition here: the register-tile product below took half of the
            // float64 kernel's time (measured; 8x8 register tiles, i.e. half the operand bytes, took twice as long).
            const int lane = cta.tid & 31, warp = cta.tid >> 5, nwarp = cta.nthr >> 5;
            const int g = lane >> 2, tq = lane & 3;
            const int nb16 = (n + 15) >> 4, ntile = nb16 * (nb16 + 1) / 2;
            for (int tile = warp; tile < ntile; tile += nwarp) {
                int ti, tj;
                upper_block(tile, nb16, ti, tj);
                const int i0 = 16 * ti, j0 = 16 * tj;
                double c[2][2][2] = {{{0, 0}, {0, 0}}, {{0, 0}, {0, 0}}};
                // operand columns of this lane (beyond the padded row length: nothing to read)
                const int ca0 = i0 + g, ca1 = i0 + 8 + g, cb0 = j0 + g, cb1 = j0 + 8 + g;
                for (int k0 = 0; k0 < trows; k0 += 4) {
                    const int k = k0 + tq;
                    const bool kin = k < trows;
                    const real *Jr = w.Jf + (kin ? k : 0) * d.npad;
                    const double a0 = (kin && ca0 < d.npad) ? double(Jr[ca0]) : 0.0, a1 = (kin && ca1 < d.npad) ? double(Jr[ca1]) : 0.0;
                    const double b0 = (kin && cb0 < d.npad) ? double(Jr[cb0]) : 0.0, b1 = (kin && cb1 < d.npad) ? double(Jr[cb1]) : 0.0;
                    dmma_m8n8k4(c[0][0][0], c[0][0][1], a0, b0);
                    dmma_m8n8k4(c[0][1][0], c[0][1][1], a0, b1);
                    dmma_m8n8k4(c[1][0][0], c[1][0][1], a1, b0);
                    dmma_m8n8k4(c[1][1][0], c[1][1][1], a1, b1);
                }
                add_upper_block16(i0, j0, n, c);
            }
        } else if (w.tc) {
            // float32: split TF32 on the tensor cores (tc::jtj_block_tf32), a warp per 16x16 block of the upper
            // triangle; A += (hi hi^T + cross terms)
            const int warp = cta.tid >> 5, nwarp = cta.nthr >> 5;
            const int nb16 = (n + 15) >> 4, ntile = nb16 * (nb16 + 1) / 2;
            for (int tile = warp; tile < ntile; tile += nwarp) {
                int ti, tj;
                upper_block(tile, nb16, ti, tj);
                const int i0 = 16 * ti, j0 = 16 * tj;
                float hh[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}}, cr[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
                tc::jtj_block_tf32(w.Jf, d.npad, trows, d.npad, i0, j0, hh, cr);
                real c[2][2][2];
#pragma unroll
                for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                    for (int ni = 0; ni < 2; ++ni)
#pragma unroll
                        for (int e = 0; e < 2; ++e) c[mi][ni][e] = hh[ni][2 * mi + e] + cr[ni][2 * mi + e];
                add_upper_block16(i0, j0, n, c);
            }
        } else
#endif
        {
            const int nb = (n + kBS - 1) / kBS, nblk = nb * (nb + 1) / 2;
            CTA_FOR(b, nblk) {
                int bi, bj;
                upper_block(b, nb, bi, bj);
                real acc[kBS * kBS];
#pragma unroll
                for (int q = 0; q < kBS * kBS; ++q) acc[q] = 0;
                // four rows in flight: in the float64 / oversized layout the tile lives in the global workspace (L2), and a
                // loop that waits for every row's two loads before its sixteen FMAs ran at a fourteenth of the FP64 rate
                // (half of the float64 kernel's time).  Same products in the same order.
                for (int row = 0; row < trows; row += 4) {
                    Vec4<real> av[4], bv[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const real *Jr = w.Jf + (row + u < trows ? row + u : trows - 1) * d.npad;
                        av[u] = ld4(Jr + bi * kBS);
                        bv[u] = ld4(Jr + bj * kBS);
                    }
#pragma unroll
                    for (int u = 0; u < 4; ++u)
                        if (row + u < trows) {
                            const real ai[4] = {av[u].x, av[u].y, av[u].z, av[u].w}, bjv[4] = {bv[u].x, bv[u].y, bv[u].z, bv[u].w};
#pragma unroll
                            for (int p = 0; p < kBS; ++p)
#pragma unroll
                                for (int q = 0; q < kBS; ++q) acc[p * kBS + q] += ai[p] * bjv[q];
                        }
                }
#pragma unroll
                for (int p = 0; p < kBS; ++p)
#pragma unroll
                    for (int q = 0; q < kBS; ++q) {
                        const int i = bi * kBS + p, j = bj * kBS + q;
                        if (j < n && i <= j) {
                            w.A[i * ld + j] += acc[p * kBS + q];
                            if (i < j) w.A[j * ld + i] += acc[p * kBS + q];
                        }
                    }
            }
        }
        // J^T r, a thread per column: on the tensor-core paths the first (ntile mod nwarp) warps took one 16x16 block more,
        // so the columns start at the warp after them (the same sums in the same order, on other threads)
        int jr_tid = cta.tid;
#if M2_GPU
        if (sizeof(real) == 8 || w.tc) {
            const int nb16 = (n + 15) >> 4, nwarp = cta.nthr >> 5;
            jr_tid = (cta.tid + cta.nthr - 32 * ((nb16 * (nb16 + 1) / 2) % nwarp)) % cta.nthr;
        }
#endif
#pragma unroll 1
        for (int cc = jr_tid; cc < n; cc += cta.nthr) {  // (six rows in flight, for the same reason; same order of the sum)
            real s = 0;
            for (int row = 0; row < trows; row += 6) {
                real jv[6];
#pragma unroll
                for (int u = 0; u < 6; ++u) jv[u] = w.Jf[(row + u < trows ? row + u : trows - 1) * d.npad + cc];
#pragma unroll
                for (int u = 0; u < 6; ++u) if (row + u < trows) s += jv[u] * w.rm[3 * t0 + row + u];
            }
            w.g[cc] -= s;
        }
    }

    // ---- closed-form terms at state xs: the prior block, the diagonals of the velocity, finger, face and linear-block
    //      terms, the joint angles of the horse model
    M2_D void closed_form_terms(const real *xs, const StepCfg<real> &c) {
        const real *th = xs + 3;
        const real *dl = xs + 3 + d.PR;
        const int n = c.n, ld = d.lda;
        if (c.wp > real(0)) {
            const int D = d.D, ks = w.isc[0];
            const real w2 = c.wp * c.wp;
            const real *Q = m.prior_Q4 + size_t(ks) * D * d.D4;
            // item = (row i, four columns): one 16-byte (L2) load, three items in flight per thread, the column map looked up
            // once per row and once per column of the vector
            const int nq = d.D4 >> 2;
#pragma unroll 1
            for (int base = cta.tid; base < D * nq; base += 3 * cta.nthr) {
                Vec4<real> qv[3];
                int ci[3], l0[3];
#pragma unroll
                for (int u = 0; u < 3; ++u) {
                    const int idx = base + u * cta.nthr;
                    ci[u] = -1;
                    l0[u] = 0;
                    qv[u].x = qv[u].y = qv[u].z = qv[u].w = real(0);
                    if (idx < D * nq) {
                        const int i = idx / nq;
                        l0[u] = 4 * (idx - i * nq);
                        ci[u] = w.colmap[3 + w.c_pids[i]];
                        if (ci[u] >= 0) qv[u] = ld4(Q + i * d.D4 + l0[u]);
                    }
                }
#pragma unroll
                for (int u = 0; u < 3; ++u)
                    if (ci[u] >= 0) {
                        const real q4[4] = {qv[u].x, qv[u].y, qv[u].z, qv[u].w};
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int l = l0[u] + e;
                            if (l < D) {
                                const int cl = w.colmap[3 + w.c_pids[l]];
                                if (cl >= 0) w.A[ci[u] * ld + cl] += w2 * q4[e];
                            }
                        }
                    }
            }
            CTA_FOR(i, D) {
                const int ci = w.colmap[3 + w.c_pids[i]];
                if (ci >= 0) w.g[ci] -= w2 * w.py[ks * D + i];
            }
            M2_SYNC();
        }
        CTA_FOR(cc, n) {
            const int fv = c.free[cc];
            real da = 0, dg = 0;
            if (fv >= 3 && fv < 3 + d.PR) {
                const int i = fv - 3;
                if (c.velo) { da += wv * wv; dg += wv * wv * (th[i] - w.velo_tgt[i]); }
                if (c.poseH && i >= m.finger_lo && i < m.finger_hi) { da += wH * wH; dg += wH * wH * th[i]; }
                if (c.face && i >= m.face_lo && i < m.face_hi) { da += wF * wF; dg += wF * wF * th[i]; }
            } else if (fv >= 3 + d.PR) {
                const int i = fv - 3 - d.PR;
                if (i < d.nd - m.n_expr) {
                    if (c.dm_terms) {
                        da += wdm * wdm;
                        dg += wdm * wdm * dl[i];
                        if (c.extrap) { da += wex * wex; dg += wex * wex * (dl[i] - w.dm_tgt[i]); }
                    }
                } else if (c.face) { da += wxp * wxp; dg += wxp * wxp * dl[i]; }
            }
            w.A[cc * ld + cc] += da;
            w.g[cc] -= dg;
        }
        if (c.wp > real(0) && m.n_jang) {
            M2_SYNC();
            CTA_FOR(i, m.n_jang) {                 // J_ii = d r_i / d x_i = 4 wp s exp(2 s x);  A += J^2,  g -= J r
                const int ci = w.colmap[3 + m.jang_id[i]];
                if (ci >= 0) {
                    const real sg = m.jang_sign[i], ex = r_exp(real(2) * sg * th[m.jang_id[i]]);
                    const real Jd = real(4) * c.wp * sg * ex, rr = real(2) * c.wp * ex;
                    w.A[ci * ld + ci] += Jd * Jd;
                    w.g[ci] -= Jd * rr;
                }
            }
        }
    }

    // ---- normal equations at the state of the latest eval():  A = J^T J (full symmetric), g = -J^T r, built marker tile by
    //      marker tile (DESIGN.md, "Per linearisation")
    M2_D void build(const real *xs, const StepCfg<real> &c) {
        ++n_build;
        M2_T0();
        const int n = c.n;
        joint_axes();
        CTA_FOR(mi, d.M) marker_local_jacobian(mi);
        CTA_FOR(i, n * d.lda) w.A[i] = 0;
        CTA_FOR(i, n) w.g[i] = 0;
        dtg_chains();
        M2_SYNC();
        CTA_FOR(s, d.S) mat3_mul(w.Loc + kM3 * s, w.Rsk + 9 * s, w.MtR + kM3 * s);
        M2_SYNC();
        M2_TACC(6);
        for (int t0 = 0; t0 < d.M; t0 += d.tmk) {
            const int tm = (d.M - t0 < d.tmk) ? d.M - t0 : d.tmk;
            tile_pose_columns(t0, tm);
            tile_linear_columns(t0, tm);
            tile_translation_columns(t0, tm, n);
            M2_SYNC();
            M2_TACC(7);
            tile_hand_columns(t0, tm);
            M2_SYNC();
            M2_TACC(8);
            tile_normal_equations(t0, tm, n);
            M2_SYNC();
            M2_TACC(9);
        }
        closed_form_terms(xs, c);
        M2_SYNC();
        M2_TACC(10);
    }

    // out = A v for the full symmetric A: one warp per row, lanes along the row
    M2_D void symv(const real *v, real *out, int n) {
#if M2_GPU
        // three adjacent lanes per row, each a third of the columns (A has an odd leading dimension: the rows of a warp
        // start in different banks), two shuffles to add the thirds.  (One warp per row with a five-step shuffle tree, four
        // rows in flight, needed three passes over the warps and ~1.5k cycles.)
        {
            const int lane = cta.tid & 31, warp = cta.tid >> 5, nwarp = cta.nthr >> 5;
            const int part = lane % 3, rl = lane / 3;                      // 10 rows per warp (lanes 30, 31 idle)
            const int third = (n + 2) / 3, j0 = part * third, j1 = (j0 + third < n) ? j0 + third : n;
            const int src0 = lane - part;
            for (int i0 = warp * 10; i0 < n; i0 += nwarp * 10) {
                const int i = i0 + rl;
                const bool on = lane < 30 && i < n;
                const real *Ar = w.A + (on ? i : 0) * d.lda;
                real s0 = 0, s1 = 0;
                int j = j0;
                for (; j + 1 < j1; j += 2) { s0 += Ar[j] * v[j]; s1 += Ar[j + 1] * v[j + 1]; }
                if (j < j1) s0 += Ar[j] * v[j];
                real sacc = on ? s0 + s1 : real(0);
                const real a1 = __shfl_sync(0xffffffffu, sacc, (src0 + 1) & 31), a2 = __shfl_sync(0xffffffffu, sacc, (src0 + 2) & 31);
                if (on && part == 0) out[i] = (sacc + a1) + a2;
            }
        }
        __syncthreads();
#else
        for (int i = 0; i < n; ++i) {
            real s = 0;
            for (int j = 0; j < n; ++j) s += w.A[i * d.lda + j] * v[j];
            out[i] = s;
        }
#endif
    }

    // ---- factor and invert the 8x8 diagonal block at k0 (GPU: the calling warp, all 32 lanes; host: one thread).
    //      Returns false if a pivot is not above pivot_eps (GPU: in every lane of the warp; host: also clears w.isc[3]).
    M2_D bool chol_diag(int k0, int n) {
        const int ld = d.ld;
        constexpr int NB = kCholNB;
        const int kb = (n - k0 < NB) ? n - k0 : NB;
        real *Li = w.Linv + (k0 / NB) * NB * NB;
#if M2_GPU
        {

            // warp 0: every lane factors the whole 8x8 block in registers (all loops unrolled: no shuffles, no local
            // memory) and lane c forward-substitutes column c of the inverse.  One warp executes this alone, so what counts
            // is the dependent chain and the instruction count: rows come in as 16-byte vectors, the elimination is written
            // right-looking (every entry receives its updates in the order of the left-looking sums -- the same numbers --
            // but each as soon as its inputs exist), and one lane stores the factor back as vectors.  (Scalar loads and
            // per-element predicated stores were 60 % of the instructions: 2k cycles per block.)
            const int lane = cta.tid;
            real *base = w.Lm + (k0 * ld + k0);
            real Lb[NB][NB], invd[NB], x[NB];
#pragma unroll
            for (int r = 0; r < NB; ++r) {
                Vec4<real> v0, v1;
                v0.x = v0.y = v0.z = v0.w = real(0);
                v1 = v0;
                if (r < kb) {
                    v0 = ld4(base + r * ld);
                    if (r >= 4) v1 = ld4(base + r * ld + 4);
                } else {                                   // identity padding of a short last block
                    if (r == 0) v0.x = real(1);
                    if (r == 1) v0.y = real(1);
                    if (r == 2) v0.z = real(1);
                    if (r == 3) v0.w = real(1);
                    if (r == 4) v1.x = real(1);
                    if (r == 5) v1.y = real(1);
                    if (r == 6) v1.z = real(1);
                    if (r == 7) v1.w = real(1);
                }
                Lb[r][0] = v0.x; Lb[r][1] = v0.y; Lb[r][2] = v0.z; Lb[r][3] = v0.w;
                Lb[r][4] = v1.x; Lb[r][5] = v1.y; Lb[r][6] = v1.z; Lb[r][7] = v1.w;
            }
            bool ok = true;
#pragma unroll
            for (int cc = 0; cc < NB; ++cc) {
                const real piv = Lb[cc][cc];
                if (!(piv > pivot_eps<real>())) ok = false;    // (the factor is discarded then: no substitute pivot on the chain)
                const real iv = r_rsqrt(piv);
                Lb[cc][cc] = piv * iv;
                invd[cc] = iv;
#pragma unroll
                for (int r = cc + 1; r < NB; ++r) Lb[r][cc] *= iv;
#pragma unroll
                for (int r = cc + 1; r < NB; ++r)
#pragma unroll
                    for (int q = cc + 1; q <= r; ++q) Lb[r][q] -= Lb[r][cc] * Lb[q][cc];
            }
            const int c = lane & (NB - 1);
#pragma unroll
            for (int r = 0; r < NB; ++r) x[r] = (r == c) ? real(1) : real(0);
#pragma unroll
            for (int pp = 0; pp < NB; ++pp) {              // x = column c of the inverse
                x[pp] *= invd[pp];
#pragma unroll
                for (int r = pp + 1; r < NB; ++r) x[r] -= Lb[r][pp] * x[pp];
            }
            if (lane < NB) {
#pragma unroll
                for (int r = 0; r < NB; ++r) Li[r * NB + lane] = x[r];   // rows/columns >= kb hold identity padding
            }
            __syncwarp();                               // every lane has read the block before one lane rewrites it
            if (lane == 0) {
#pragma unroll
                for (int r = 0; r < NB; ++r)
                    if (r < kb) {                           // (the block's upper triangle is never read: zeros)
                        Vec4<real> v0, v1;
                        v0.x = Lb[r][0]; v0.y = r >= 1 ? Lb[r][1] : real(0); v0.z = r >= 2 ? Lb[r][2] : real(0); v0.w = r >= 3 ? Lb[r][3] : real(0);
                        *reinterpret_cast<Vec4<real> *>(base + r * ld) = v0;
                        if (r >= 4) {
                            v1.x = Lb[r][4]; v1.y = r >= 5 ? Lb[r][5] : real(0); v1.z = r >= 6 ? Lb[r][6] : real(0); v1.w = r >= 7 ? Lb[r][7] : real(0);
                            *reinterpret_cast<Vec4<real> *>(base + r * ld + 4) = v1;
                        }
                    }
            }
            return ok;
                }
#else
        {

            real Lk[NB * NB], id[NB];
            bool ok = true;
            for (int r = 0; r < kb; ++r)
                for (int cc = 0; cc <= r; ++cc) {
                    real sacc = w.Lm[(k0 + r) * ld + k0 + cc];
                    for (int p = 0; p < cc; ++p) sacc -= Lk[r * NB + p] * Lk[cc * NB + p];
                    if (cc == r) {
                        if (!(sacc > pivot_eps<real>())) { ok = false; sacc = real(1); }
                        const real sq = r_sqrt(sacc);
                        Lk[r * NB + r] = sq;
                        id[r] = real(1) / sq;
                    } else Lk[r * NB + cc] = sacc * id[cc];
                }
            for (int cc = 0; cc < kb; ++cc)
                for (int r = 0; r < kb; ++r) {
                    real v = 0;
                    if (r == cc) v = id[r];
                    else if (r > cc) {
                        real sacc = 0;
                        for (int p = cc; p < r; ++p) sacc -= Lk[r * NB + p] * Li[p * NB + cc];
                        v = sacc * id[r];
                    }
                    Li[r * NB + cc] = v;
                }
            for (int r = 0; r < kb; ++r)
                for (int cc = 0; cc <= r; ++cc) w.Lm[(k0 + r) * ld + k0 + cc] = Lk[r * NB + cc];
            for (int r = 0; r < NB; ++r)
                for (int cc = 0; cc < NB; ++cc)
                    if (r >= kb || cc >= kb) Li[r * NB + cc] = (r == cc) ? real(1) : real(0);
            if (!ok) w.isc[3] = 0;
            return ok;
                }
#endif
    }

    // ---- one 4x4 tile of the trailing update after the panel of block k0:  Lm[i][j] -= sum_c Pn[c][i] Pn[c][j]
    M2_D void chol_tile(int it, int r0, int n) {
        const int ld = d.ld;
        constexpr int NB = kCholNB;
        int ti = 0, rem = it;
        while (rem > ti) { rem -= ti + 1; ++ti; }
        const int tj = rem;
        real acc[kBS * kBS];
#pragma unroll
        for (int q = 0; q < kBS * kBS; ++q) acc[q] = 0;
#pragma unroll
        for (int cc = 0; cc < NB; ++cc) {
            const Vec4<real> av = ld4(w.Pn + cc * d.ldp + r0 + ti * kBS), bv = ld4(w.Pn + cc * d.ldp + r0 + tj * kBS);
            const real ai[4] = {av.x, av.y, av.z, av.w}, bj[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
            for (int p = 0; p < kBS; ++p)
#pragma unroll
                for (int q = 0; q < kBS; ++q) acc[p * kBS + q] += ai[p] * bj[q];
        }
#pragma unroll
        for (int p = 0; p < kBS; ++p) {
            const int i = r0 + ti * kBS + p;
            if (i <= n && r0 + tj * kBS < n) {
                real *dst = w.Lm + i * ld + r0 + tj * kBS;
                Vec4<real> v = ld4(dst);
                v.x -= acc[p * kBS]; v.y -= acc[p * kBS + 1]; v.z -= acc[p * kBS + 2]; v.w -= acc[p * kBS + 3];
                *reinterpret_cast<Vec4<real> *>(dst) = v;
            }
        }
    }

    // ---- one row of the panel below the diagonal block at k0 (kb columns):  x = a Linv^T  (x_c = sum_{p<=c} a_p Linv[c][p]),
    //      written in place and, transposed, into Pn[c][row] (rows beyond n: zeros), which the trailing update reads
    M2_D void panel_row(int i, int k0, int kb, const real *Li, int n) {
        const int ld = d.ld;
        constexpr int NB = kCholNB;
        real xr[NB];
#pragma unroll
        for (int cc = 0; cc < NB; ++cc) xr[cc] = 0;
        if (i <= n) {
            real *row = w.Lm + i * ld + k0;
            real av[NB];
            {   // (k0 is a multiple of 8 and ld of 4: two aligned 16-byte loads; columns >= kb are masked below)
                const Vec4<real> a0 = ld4(row), a1 = ld4(row + 4);
                av[0] = a0.x; av[1] = a0.y; av[2] = a0.z; av[3] = a0.w; av[4] = a1.x; av[5] = a1.y; av[6] = a1.z; av[7] = a1.w;
            }
#pragma unroll
            for (int cc = 0; cc < NB; ++cc) if (cc >= kb) av[cc] = real(0);
#pragma unroll
            for (int cc = 0; cc < NB; ++cc) {
                const Vec4<real> l0 = ld4(Li + cc * NB);
                real sacc = av[0] * l0.x;
                if (cc >= 1) sacc += av[1] * l0.y;
                if (cc >= 2) sacc += av[2] * l0.z;
                if (cc >= 3) sacc += av[3] * l0.w;
                if (cc >= 4) {
                    const Vec4<real> l1 = ld4(Li + cc * NB + 4);
                    sacc += av[4] * l1.x;
                    if (cc >= 5) sacc += av[5] * l1.y;
                    if (cc >= 6) sacc += av[6] * l1.z;
                    if (cc >= 7) sacc += av[7] * l1.w;
                }
                xr[cc] = cc < kb ? sacc : real(0);
            }
            if (kb == NB) {
                Vec4<real> o0, o1;
                o0.x = xr[0]; o0.y = xr[1]; o0.z = xr[2]; o0.w = xr[3]; o1.x = xr[4]; o1.y = xr[5]; o1.z = xr[6]; o1.w = xr[7];
                *reinterpret_cast<Vec4<real> *>(row) = o0;
                *reinterpret_cast<Vec4<real> *>(row + 4) = o1;
            } else {
#pragma unroll
                for (int cc = 0; cc < NB; ++cc) if (cc < kb) row[cc] = xr[cc];
            }
        }
#pragma unroll
        for (int cc = 0; cc < NB; ++cc) w.Pn[cc * d.ldp + i] = xr[cc];
    }

    // Gauss-Newton step dgn = A^-1 g by a Jacobi-scaled, blocked right-looking Cholesky in w.Lm (lower
    // triangle incl. diagonal).  One lane factors each 8x8 diagonal block and also inverts it; the panel and
    // both triangular solves then use the explicit block inverses (plain dot products, no divides and no
    // dependent chains).  Returns false if A is not numerically positive definite.
    M2_D bool gauss_newton(int n) {
        const int ld = d.ld;
        constexpr int NB = kCholNB;
        M2_T0();
        CTA_FOR(i, n) {
            const real a = w.A[i * d.lda + i];
            w.ds[i] = (a > real(0)) ? real(1) / r_sqrt(a) : real(0);
        }
        M2_SYNC();
#if M2_GPU
        {
            const int lane = cta.tid & 31, warp = cta.tid >> 5, nwarp = cta.nthr >> 5;
            for (int i = warp; i < n; i += nwarp)
                for (int j = lane; j <= i; j += 32) w.Lm[i * ld + j] = w.A[i * d.lda + j] * w.ds[i] * w.ds[j];
        }
#else
        for (int i = 0; i < n; ++i)
            for (int j = 0; j <= i; ++j) w.Lm[i * ld + j] = w.A[i * d.lda + j] * w.ds[i] * w.ds[j];
#endif
        // the scaled right-hand side rides along as row n: after the factorisation it holds z = L^-1 (ds*g)
        CTA_FOR(j, n) w.Lm[n * ld + j] = w.g[j] * w.ds[j];
        M2_SYNC();
        M2_TACC(11);
#if M2_GPU
        // Pipelined variant: warp 0 runs the serial chain of a block -- the eight panel rows that make up the next diagonal
        // block, the update of that block, its factorisation and inversion -- while the other warps solve the rest of the
        // panel and apply the trailing update; they only wait (named barrier 1) for warp 0's eight panel rows.  One full
        // barrier per block, and a single call site of the diagonal-block factorisation (the pseudo-block k0 = -NB
        // factors the first one).  (The launcher never starts fewer than 128 threads.)  The block's full barrier also carries
        // warp 0's verdict on the block it factored: a flag in shared memory would be cleared by warp 0 in its next
        // chol_diag before a slow warp had read it (warp 0 passes no blocking barrier in between), and that warp would
        // return one block early while the others wait for it on barrier 1.
        {
            const int nthr = cta.nthr;
#pragma unroll 1
            for (int k0 = -NB; k0 < n; k0 += NB) {
                bool ok = true;
                const int kb = k0 < 0 ? 0 : ((n - k0 < NB) ? n - k0 : NB);
                const int r0 = k0 < 0 ? 0 : k0 + kb;
                const real *Li = w.Linv + (k0 < 0 ? 0 : k0 / NB) * NB * NB;
                const bool trail = k0 >= 0 && r0 < n;
                if (cta.tid < 32) {
                    if (k0 >= 0) {
                        const int i = r0 + cta.tid;
                        M2_TACC(14);
                        if (cta.tid < NB && i < d.ldp) panel_row(i, k0, kb, Li, n);
                        if (trail) {
                            __threadfence_block();
                            __syncwarp();
                            asm volatile("bar.arrive 1, %0;" :: "r"(nthr) : "memory");
                            // the next diagonal block (and the right-hand-side row where it falls into these eight rows):
                            // lane -> row p, columns q0, q0 + 1 of the 8x8 square (its upper triangle is never read)
                            {
                                const int pr = cta.tid >> 2, q0 = (cta.tid & 3) * 2;
                                const int ii = r0 + pr, jj = r0 + q0;
                                if (ii <= n && jj < n) {
                                    real acc0 = 0, acc1 = 0;
#pragma unroll
                                    for (int cc = 0; cc < NB; ++cc) {
                                        const real pi = w.Pn[cc * d.ldp + ii];
                                        acc0 += pi * w.Pn[cc * d.ldp + jj];
                                        acc1 += pi * w.Pn[cc * d.ldp + jj + 1];
                                    }
                                    w.Lm[ii * ld + jj] -= acc0;
                                    w.Lm[ii * ld + jj + 1] -= acc1;
                                }
                            }
                            __syncwarp();
                        }
                    }
                    M2_TACC(12);
                    if (r0 < n) ok = chol_diag(r0, n);
                    M2_TACC(13);
                } else {
                    if (k0 >= 0) {
                        const int t = cta.tid - 32, nt_ = nthr - 32;
                        for (int i = r0 + NB + t; i < d.ldp; i += nt_) panel_row(i, k0, kb, Li, n);
                        if (trail) {
                            asm volatile("bar.sync 1, %0;" :: "r"(nthr) : "memory");
                            const int R = n + 1 - r0, ntl = (R + kBS - 1) / kBS, ntri = ntl * (ntl + 1) / 2;
                            for (int it = 3 + t; it < ntri; it += nt_) chol_tile(it, r0, n);
                        }
                    }
                }
                if (__syncthreads_or(!ok)) return false;
            }
            M2_TACC(14);
        }
#else
        // host build: the same blocked right-looking factorisation, one block after the other
        w.isc[3] = 1;
        chol_diag(0, n);
        if (w.isc[3] == 0) return false;
        for (int k0 = 0; k0 < n; k0 += NB) {
            const int kb = (n - k0 < NB) ? n - k0 : NB;
            const real *Li = w.Linv + (k0 / NB) * NB * NB;
            for (int i = k0 + kb; i < d.ldp; ++i) panel_row(i, k0, kb, Li, n);
            const int r0 = k0 + kb, R = r0 < n ? n + 1 - r0 : 0;   // rows r0..n (row n = right-hand side), columns r0..n-1
            if (R > 0) {
                const int nt = (R + kBS - 1) / kBS, ntri = nt * (nt + 1) / 2;
                for (int it = 0; it < ntri; ++it) chol_tile(it, r0, n);
                chol_diag(r0, n);
                if (w.isc[3] == 0) return false;
            }
        }
#endif
        // backward solve L^T y = z by the first warp (the forward solve happened inside the factorisation), column
        // oriented: once the block y_k = Linv_k^T z_k is known, every lane subtracts its contribution from the entries
        // z_i, i < k0, it owns -- that reads rows of L (consecutive words) and needs no reduction across lanes, where
        // the row-oriented form read columns (16-way bank conflicts at ld = 112) and eight warp reductions per block.
#if M2_GPU
        // Four warps (named barrier 2): every warp forms y_k = Linv_k^T z_k itself, the 128 threads share the rows i < k0 of
        // the update z_i -= L[k, i] y_k -- one round per block instead of four by a single warp (560 -> cycles per block
        // are the dependent shared-memory round trips, not the arithmetic).
        if (cta.tid < 128) {
            const int tid = cta.tid;
            for (int i = tid; i < n; i += 128) w.tmp[i] = w.Lm[n * ld + i];     // z = L^-1 (ds*g), see above
            asm volatile("bar.sync 2, 128;" ::: "memory");
#pragma unroll 1
            for (int k0 = ((n - 1) / NB) * NB; k0 >= 0; k0 -= NB) {
                const int kb = (n - k0 < NB) ? n - k0 : NB;
                const real *Li = w.Linv + (k0 / NB) * NB * NB;
                real zv[NB], y[NB], Lr[NB][NB];
                {
                    const Vec4<real> z0 = ld4(w.tmp + k0), z1 = ld4(w.tmp + k0 + 4);
                    zv[0] = z0.x; zv[1] = z0.y; zv[2] = z0.z; zv[3] = z0.w; zv[4] = z1.x; zv[5] = z1.y; zv[6] = z1.z; zv[7] = z1.w;
                }
#pragma unroll
                for (int cc = 1; cc < NB; ++cc) if (cc >= kb) zv[cc] = real(0);
#pragma unroll
                for (int pp = 0; pp < NB; ++pp) {
                    const Vec4<real> l0 = ld4(Li + pp * NB);
                    Lr[pp][0] = l0.x; Lr[pp][1] = l0.y; Lr[pp][2] = l0.z; Lr[pp][3] = l0.w;
                    if (pp >= 4) {
                        const Vec4<real> l1 = ld4(Li + pp * NB + 4);
                        Lr[pp][4] = l1.x; Lr[pp][5] = l1.y; Lr[pp][6] = l1.z; Lr[pp][7] = l1.w;
                    }
                }
#pragma unroll
                for (int cc = 0; cc < NB; ++cc) {          // y = Linv^T z (every thread, redundantly)
                    real sacc = 0;
#pragma unroll
                    for (int pp = cc; pp < NB; ++pp) sacc += Lr[pp][cc] * zv[pp];
                    y[cc] = sacc;
                }
                for (int i = tid; i < k0; i += 128) {
                    real zi = w.tmp[i];
#pragma unroll
                    for (int cc = 0; cc < NB; ++cc) if (cc < kb) zi -= w.Lm[(k0 + cc) * ld + i] * y[cc];
                    w.tmp[i] = zi;
                }
                asm volatile("bar.sync 2, 128;" ::: "memory");   // (every thread has read z_k before thread 0 replaces it by y_k)
                if (tid == 0) {
                    if (kb == NB) {
                        Vec4<real> o0, o1;
                        o0.x = y[0]; o0.y = y[1]; o0.z = y[2]; o0.w = y[3]; o1.x = y[4]; o1.y = y[5]; o1.z = y[6]; o1.w = y[7];
                        *reinterpret_cast<Vec4<real> *>(w.tmp + k0) = o0;
                        *reinterpret_cast<Vec4<real> *>(w.tmp + k0 + 4) = o1;
                    } else {
#pragma unroll
                        for (int cc = 0; cc < NB; ++cc) if (cc < kb) w.tmp[k0 + cc] = y[cc];
                    }
                }
            }
            asm volatile("bar.sync 2, 128;" ::: "memory");
            for (int i = tid; i < n; i += 128) w.dgn[i] = w.tmp[i] * w.ds[i];
        }
#else
        const int wl = cta.nthr < 32 ? cta.nthr : 32;
        if (cta.tid < wl) {
            const int lane = cta.tid;
            for (int i = lane; i < n; i += wl) w.tmp[i] = w.Lm[n * ld + i];     // z = L^-1 (ds*g), see above
            M2_WSYNC();
            for (int k0 = ((n - 1) / NB) * NB; k0 >= 0; k0 -= NB) {
                const int kb = (n - k0 < NB) ? n - k0 : NB;
                const real *Li = w.Linv + (k0 / NB) * NB * NB;
                real zv[NB], y[NB];
#pragma unroll
                for (int cc = 0; cc < NB; ++cc) zv[cc] = cc < kb ? w.tmp[k0 + cc] : real(0);
#pragma unroll
                for (int cc = 0; cc < NB; ++cc) {          // y = Linv^T z (every lane, redundantly)
                    real sacc = 0;
#pragma unroll
                    for (int pp = cc; pp < NB; ++pp) sacc += Li[pp * NB + cc] * zv[pp];
                    y[cc] = sacc;
                }
                for (int i = lane; i < k0; i += wl) {
                    real zi = w.tmp[i];
#pragma unroll
                    for (int cc = 0; cc < NB; ++cc) if (cc < kb) zi -= w.Lm[(k0 + cc) * ld + i] * y[cc];
                    w.tmp[i] = zi;
                }
                M2_WSYNC();                                // (all lanes have read z_k before lane 0 overwrites it)
                if (lane == 0) {
#pragma unroll
                    for (int cc = 0; cc < NB; ++cc) if (cc < kb) w.tmp[k0 + cc] = y[cc];
                }
                M2_WSYNC();
            }
            for (int i = lane; i < n; i += wl) w.dgn[i] = w.tmp[i] * w.ds[i];
        }
#endif
        M2_SYNC();
        M2_TACC(15);
        return true;
    }

    // ---- column maps and needed joints of one free-variable list (Step 1: which = 0, Step 2: which = 1), built once per
    //      chunk (prologue) into the stage cache
    M2_D void stage_tables(int which) {
        const int *free = which ? static_cast<const int *>(w.c_free2) : static_cast<const int *>(w.c_free1);
        const int n = which ? m.n2 : m.n1;
        CTA_FOR(i, d.NX) w.colmap[i] = -1;
        CTA_FOR(i, d.nJ) w.jlist[i] = 0;
        M2_SYNC();
        CTA_FOR(i, n) {
            const int fv = free[i];
            w.colmap[fv] = i;
            int src;
            if (fv < 3) src = -1 - fv;
            else if (fv < 3 + m.body_dof) { src = fv - 3; w.jlist[(fv - 3) / 3] = 1; }
            else if (fv < 3 + d.PR) src = -4;
            else src = d.PF + (fv - 3 - d.PR);
            w.colsrc[i] = src;
        }
        M2_SYNC();
        if (cta.tid == 0) {
            // joints needed by this step: body joints with a free column, hand joints of blocks with a free row
            int hf = 0;
            for (int b = 0; b < m.hb_n; ++b) {
                bool any = false;
                for (int r = m.hb[b].r0; r < m.hb[b].r1; ++r) any = any || w.colmap[3 + m.body_dof + r] >= 0;
                if (any) {
                    hf = 1;
                    for (int q = m.hb[b].q0; q < m.hb[b].q1; ++q) w.jlist[(m.body_dof + q) / 3] = 1;
                }
            }
            int cnt = 0;
            for (int j = 0; j < d.nJ; ++j) if (w.jlist[j]) w.jlist[cnt++] = j;
            w.st_meta[2 * which] = cnt;
            w.st_meta[2 * which + 1] = hf;
        }
        M2_SYNC();
        CTA_FOR(i, d.NX) w.st_colmap[which * d.NX + i] = w.colmap[i];
        CTA_FOR(i, n) w.st_colsrc[which * d.n2 + i] = w.colsrc[i];
        CTA_FOR(i, d.nJ) w.st_jlist[which * d.nJ + i] = w.jlist[i];
        M2_SYNC();
    }

    // ---- per-stage set-up of one ch.minimize call: the column maps and the joints whose columns are needed come from the
    //      stage cache (the thread-0 loops that build them cost 7k cycles per call, twice per frame)
    M2_D void stage_setup(const StepCfg<real> &c) {
        ++n_min;
        const int which = c.free == static_cast<const int *>(w.c_free2) ? 1 : 0;
        CTA_FOR(i, d.NX) w.colmap[i] = w.st_colmap[which * d.NX + i];
        CTA_FOR(i, c.n) w.colsrc[i] = w.st_colsrc[which * d.n2 + i];
        CTA_FOR(i, d.nJ) w.jlist[i] = w.st_jlist[which * d.nJ + i];
        njl = w.st_meta[2 * which];
        hand_free = w.st_meta[2 * which + 1] != 0;
        M2_SYNC();
    }

    // ---- one frame: [Procrustes] + the ch.minimize calls of the reference + the output evaluation, written as
    //      one loop around a single eval() / build() / gauss_newton() call site each (the 32 KB instruction cache
    //      makes code size a first-order cost; see DESIGN.md section 3).  The dog-leg control flow is chumpy's
    //      (SURVEY.md Appendix A.6): outer iterations, inner retries until a step improves, e_3 / e_2 / maxiter.
    //      `light` (warm-up frames of a chunk only, never an emitted frame): the frame is tracked with a single
    //      linearisation of the Step-2 problem (one accepted dog-leg step) instead of the two minimisations -- enough to
    //      carry the state along the sequential trajectory until the last, fully solved warm-up frames (DESIGN.md 4).
    M2_D void solve_frame(int f, bool emit, bool first, bool fingers, bool dyn, bool face, bool light) {
        const Options &o = job.opt;
        const real e1 = real(1e-15), e2 = real(1e-15);
        enum { OP_PROCRUSTES, OP_BEGIN, OP_TRIAL, OP_OUTPUT };
        int op = first ? OP_PROCRUSTES : OP_BEGIN;
        int stage = first ? 0 : (light ? 4 : 3);   // 0..2 first-frame annealing (chmosh.py:637-653), 3 Step 1 (665-671), 4 Step 2 (676-705)
        if (lin_f >= 0) stage = job.lin_step == 2 ? 4 : 3;      // linearise mode: the stage names the free-variable list
        const int maxit = light ? 1 : o.maxiter;
        StepCfg<real> c;
        c.free = w.c_free1; c.n = m.n1; c.velo = has_velo; c.poseH = false; c.dm_terms = false; c.extrap = false; c.face = false;
        c.wp = 0; c.e3 = real(o.e3_first);
        bool need_setup = !first;
        // dog-leg state of the running minimisation
        real sse0 = 0, delta = 0, alpha = 0, nsd = 0, ngn2 = 0, gn_sd = 0, nstep = 0, npn = 0, gd = 0, dAd = 0;
        bool done = false, in_iter = false, have_gn = false, gn_ok = true;
        int iter = 0;
        M2_T0();
        while (true) {
            if (need_setup) {
                M2_TACC(25);
                // configuration of this stage
                c.free = w.c_free1; c.n = m.n1; c.poseH = false; c.dm_terms = false; c.extrap = false; c.face = false;
                if (stage < 3) {
                    c.wp = wp_frame * (stage == 0 ? real(10) : (stage == 1 ? real(5) : real(1)));
                    c.e3 = real(o.e3_first);
                } else {
                    c.wp = wp_frame;
                    c.e3 = real(o.e3);
                    if (stage == 4) { c.free = w.c_free2; c.n = m.n2; c.poseH = fingers; c.dm_terms = dyn; c.extrap = has_extrap; c.face = face; }
                }
                stage_setup(c);
                need_setup = false;
                M2_TACC(20);
            }
            const int n = c.n;
            // ---------------- the one evaluation site
            {
                // A stage that starts where the last accepted trial step ended (Step 2 after Step 1, Step 1 of the next
                // frame, the output evaluation) finds the forward pass of that state still in shared memory.
                const bool reuse = op != OP_TRIAL && fwd_at_x && (fwd_has_prior || !(c.wp > real(0)));
                M2_TACC(25);
                eval(op == OP_TRIAL ? w.xt : w.x, c, reuse);
                M2_TRESET();
                if (!reuse) fwd_has_prior = c.wp > real(0);
                fwd_at_x = op != OP_TRIAL;                     // (a trial point becomes the state only if it is accepted)
            }
            if (lin_f >= 0) {                                  // linearise mode: what the evaluation left goes out
                CTA_FOR(i, 3 * d.M) { job.markers_sim[size_t(f) * 3 * d.M + i] = w.mk[i]; if (job.lin_r) job.lin_r[size_t(f) * 3 * d.M + i] = w.rm[i]; }
                CTA_FOR(i, N_ERR) job.errs[size_t(f) * N_ERR + i] = w.sc[1 + i];
                if (job.lin_vp) CTA_FOR(i, 3 * d.S) job.lin_vp[size_t(f) * 3 * d.S + i] = w.vp[i];
                if (job.lin_mode < 2) break;
            }
            if (op == OP_PROCRUSTES) {                         // chmosh.py:634
                procrustes();
                fwd_at_x = false;
                op = OP_BEGIN;
                need_setup = true;
                continue;
            }
            if (op == OP_OUTPUT) break;
            bool do_build = false, improved = false;
            if (op == OP_BEGIN) {
                sse0 = w.sc[0];
                delta = real(o.delta_0);
                done = false; in_iter = false; iter = 0;
                do_build = true;
            } else {
                const real sse1 = w.sc[0];
                real rho = sse0 - sse1;
                improved = rho > real(0) || rho >= -accept_slack<real>() * sse0;
                if (rho > real(0)) rho = rho / (real(2) * gd - dAd);
                if (improved) {
                    CTA_FOR(i, d.NX) w.x[i] = w.xt[i];
                    fwd_at_x = true;
                    M2_SYNC();
                    if (c.e3 > real(0) && (sse0 - sse1) / sse0 < c.e3) done = true;
                    else { do_build = true; sse0 = sse1; }
                }
                if (rho > real(0.9)) { const real cand = real(2.5) * nstep; if (cand > delta) delta = cand; }
                else if (rho < real(0.05)) delta *= real(0.25);
                if (delta <= e2 * npn) done = true;
                if (done || improved) {
                    in_iter = false;
                    if (!done && iter >= maxit) { done = true; if (!light) frame_flags |= ST_MAXITER; }
                }
            }
            // ---------------- the one linearisation site
            M2_TACC(21);
            if (do_build && !done) build(w.x, c);
            M2_TRESET();
            if (lin_f >= 0) {                                  // linearise mode: the normal equations go out, nothing is solved
                CTA_FOR(idx, n * n) { const int i = idx / n, j = idx - i * n; job.lin_A[size_t(f) * n * n + idx] = w.A[i * d.lda + j]; }
                CTA_FOR(i, n) job.lin_g[size_t(f) * n + i] = w.g[i];
                break;
            }
            if (op == OP_BEGIN) {
                // chumpy stops on ||g||_inf < e_1 = 1e-15, i.e. only for a numerically zero gradient
                real sq[1] = {0};
                CTA_FOR(i, n) sq[0] += w.g[i] * w.g[i];
                cta_reduce<real, 1>(cta, sq, w.red);
                if (r_sqrt(sq[0]) < e1) done = true;
            }
            if (!done) {
                if (!in_iter) {                                // start of an outer iteration
                    ++iter;
                    ++n_iter;
                    symv(w.g, w.Ag, n);
                    real r2[2] = {0, 0};
                    CTA_FOR(i, n) { r2[0] += w.g[i] * w.g[i]; r2[1] += w.g[i] * w.Ag[i]; }
                    cta_reduce<real, 2>(cta, r2, w.red);
                    alpha = r2[0] / r2[1];
                    nsd = alpha * r_sqrt(r2[0]);
                    have_gn = false; gn_ok = true;
                    in_iter = true;
                }
                // ---- update_step
                int kind;           // 0 stunted Cauchy, 1 Gauss-Newton, 2 blend
                real beta = 0, scale_sd = 0;
                if (nsd >= delta) { kind = 0; scale_sd = delta / nsd * alpha; }
                else {
                    if (!have_gn) {
                        M2_TACC(22);
                        gn_ok = gauss_newton(n);               // the one factorisation site
                        M2_TRESET();
                        have_gn = true;
                        if (gn_ok) {
                            real q[2] = {0, 0};
                            CTA_FOR(i, n) { q[0] += w.dgn[i] * w.dgn[i]; q[1] += w.dgn[i] * w.g[i]; }
                            cta_reduce<real, 2>(cta, q, w.red);
                            ngn2 = q[0];
                            gn_sd = alpha * q[1];
                        } else frame_flags |= ST_GN_FALLBACK;
                    }
                    if (!gn_ok) { kind = 0; scale_sd = alpha; }         // Cauchy step (documented deviation)
                    else if (r_sqrt(ngn2) <= delta) kind = 1;
                    else {
                        kind = 2;
                        const real dsq = delta * delta, sd2 = nsd * nsd;
                        const real diff2 = ngn2 - real(2) * gn_sd + sd2;          // |dgn - dsd|^2
                        const real pnow = diff2 * dsq + gn_sd * gn_sd - ngn2 * sd2;
                        beta = (dsq - sd2) / ((gn_sd - sd2) + r_sqrt(pnow));
                    }
                }
                CTA_FOR(i, n) {
                    real v;
                    if (kind == 0) v = scale_sd * w.g[i];
                    else if (kind == 1) v = w.dgn[i];
                    else v = alpha * w.g[i] + beta * (w.dgn[i] - alpha * w.g[i]);
                    w.d[i] = v;
                }
                M2_SYNC();
                symv(w.d, w.tmp, n);
                real q[4] = {0, 0, 0, 0};
                CTA_FOR(i, n) {
                    q[0] += w.d[i] * w.d[i];
                    q[1] += w.g[i] * w.d[i];
                    q[2] += w.d[i] * w.tmp[i];
                    const real pv = w.x[c.free[i]];
                    q[3] += pv * pv;
                }
                cta_reduce<real, 4>(cta, q, w.red);
                nstep = r_sqrt(q[0]); gd = q[1]; dAd = q[2]; npn = r_sqrt(q[3]);
                if (nstep <= e2 * npn) done = true;
                else {
                    CTA_FOR(i, d.NX) w.xt[i] = w.x[i];
                    M2_SYNC();
                    CTA_FOR(i, n) w.xt[c.free[i]] += w.d[i];
                    M2_SYNC();
                    op = OP_TRIAL;
                    M2_TACC(23);
                    continue;
                }
            }
            // the minimisation of this stage has terminated
            if (stage < 4) { ++stage; op = OP_BEGIN; need_setup = true; continue; }
            if (!emit) break;
            op = OP_OUTPUT;                                    // per-term SSE and markers at the solution
        }
        if (cta.tid == 0 && job.totals) {
#if M2_GPU
            atomicAdd(job.totals + 0, n_iter); atomicAdd(job.totals + 1, n_eval);
            atomicAdd(job.totals + 2, n_build); atomicAdd(job.totals + 3, n_min);
            if (emit) {
                atomicAdd(job.totals + 4, n_iter); atomicAdd(job.totals + 5, n_eval);
                atomicAdd(job.totals + 6, n_build); atomicAdd(job.totals + 7, n_min);
            }
#else
            job.totals[0] += n_iter; job.totals[1] += n_eval; job.totals[2] += n_build; job.totals[3] += n_min;
            if (emit) { job.totals[4] += n_iter; job.totals[5] += n_eval; job.totals[6] += n_build; job.totals[7] += n_min; }
#endif
        }
        if (emit && resuming) {
            // how far is the re-solved frame from the row it replaces?  (run_chunk stops the repair once the two
            // trajectories have merged: the remaining rows of the chunk are then still valid)
            real dm[1] = {0};
            if (job.status[f] & ST_SOLVED) {
                // root + body pose at full weight, the remaining pose coefficients (finger PCA, jaw) at a tenth: the ratio of
                // their per-frame tolerances (BASELINE.md section 4) and of the boundary tolerances (chmosh.BOUNDARY_TOL)
                const int nbody = m.body_dof < 66 ? m.body_dof : 66;
                CTA_FOR(i, d.PR) {
                    real e = r_abs(w.x[3 + i] - job.pose[size_t(f) * d.PR + i]);
                    if (i >= nbody) e *= real(0.1);
                    if (e > dm[0]) dm[0] = e;
                }
                CTA_FOR(i, 3) { const real e = real(10) * r_abs(w.x[i] - job.trans[size_t(f) * 3 + i]); if (e > dm[0]) dm[0] = e; }
            } else dm[0] = real(1);
            // (max via the sum reduction of a one-hot power is overkill: reduce the maximum over threads with shuffles)
            cta_max(dm);
            resume_diff = dm[0];
        }
        if (emit) {
            CTA_FOR(i, d.PF) job.fullpose[size_t(f) * d.PF + i] = w.fullpose[i];
            CTA_FOR(i, d.PR) job.pose[size_t(f) * d.PR + i] = w.x[3 + i];
            CTA_FOR(i, 3) job.trans[size_t(f) * 3 + i] = w.x[i];
            if (job.dmpls) CTA_FOR(i, d.nd) job.dmpls[size_t(f) * d.nd + i] = w.x[3 + d.PR + i];
            CTA_FOR(i, 3 * d.M) job.markers_sim[size_t(f) * 3 * d.M + i] = w.mk[i];
            CTA_FOR(i, N_ERR) job.errs[size_t(f) * N_ERR + i] = w.sc[1 + i];
            if (cta.tid == 0) {
                job.status[f] = ST_SOLVED | frame_flags | (has_velo ? ST_HAS_VELO : 0) | (has_extrap ? ST_HAS_EXTRAP : 0);
                job.counters[4 * f + 0] = n_iter;
                job.counters[4 * f + 1] = n_eval;
                job.counters[4 * f + 2] = n_build;
                job.counters[4 * f + 3] = n_min;
            }
            M2_SYNC();
        }
        M2_TACC(24);
    }

    // ---- Procrustes initialisation of root orientation and translation (rigid_transformations.py:39-83)
    M2_D void procrustes() {
        if (cta.tid == 0) {
            double ca[3] = {0, 0, 0}, cb[3] = {0, 0, 0};
            int cnt = 0;
            for (int mi = 0; mi < d.M; ++mi)
                if (w.vis[mi]) {
                    for (int q = 0; q < 3; ++q) { ca[q] += double(w.mk[3 * mi + q]); cb[q] += double(w.obs[3 * mi + q]); }
                    ++cnt;
                }
            for (int q = 0; q < 3; ++q) { ca[q] /= cnt; cb[q] /= cnt; }
            double S[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};          // S[r][c] = sum a_r b_c
            for (int mi = 0; mi < d.M; ++mi)
                if (w.vis[mi])
                    for (int r = 0; r < 3; ++r)
                        for (int q = 0; q < 3; ++q)
                            S[3 * r + q] += (double(w.mk[3 * mi + r]) - ca[r]) * (double(w.obs[3 * mi + q]) - cb[q]);
            // Horn's quaternion matrix; its top eigenvector is the optimal proper rotation a -> b,
            // i.e. the SVD solution with the det fix of rigid_transformations.py:57-63.
            double N[16] = {
                S[0] + S[4] + S[8], S[5] - S[7], S[6] - S[2], S[1] - S[3],
                S[5] - S[7], S[0] - S[4] - S[8], S[1] + S[3], S[6] + S[2],
                S[6] - S[2], S[1] + S[3], -S[0] + S[4] - S[8], S[5] + S[7],
                S[1] - S[3], S[6] + S[2], S[5] + S[7], -S[0] - S[4] + S[8]};
            double V[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
            for (int sweep = 0; sweep < 30; ++sweep) {
                double off = 0;
                for (int p = 0; p < 4; ++p)
                    for (int q = p + 1; q < 4; ++q) off += N[4 * p + q] * N[4 * p + q];
                if (off < 1e-30) break;
                for (int p = 0; p < 4; ++p)
                    for (int q = p + 1; q < 4; ++q) {
                        const double apq = N[4 * p + q];
                        if (fabs(apq) < 1e-300) continue;
                        const double th = (N[4 * q + q] - N[4 * p + p]) / (2 * apq);
                        const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1));
                        const double cs = 1 / sqrt(t * t + 1), sn = t * cs;
                        for (int k = 0; k < 4; ++k) {
                            const double akp = N[4 * k + p], akq = N[4 * k + q];
                            N[4 * k + p] = cs * akp - sn * akq;
                            N[4 * k + q] = sn * akp + cs * akq;
                        }
                        for (int k = 0; k < 4; ++k) {
                            const double apk = N[4 * p + k], aqk = N[4 * q + k];
                            N[4 * p + k] = cs * apk - sn * aqk;
                            N[4 * q + k] = sn * apk + cs * aqk;
                        }
                        for (int k = 0; k < 4; ++k) {
                            const double vkp = V[4 * k + p], vkq = V[4 * k + q];
                            V[4 * k + p] = cs * vkp - sn * vkq;
                            V[4 * k + q] = sn * vkp + cs * vkq;
                        }
                    }
            }
            int best = 0;
            for (int k = 1; k < 4; ++k) if (N[5 * k] > N[5 * best]) best = k;
            double qw = V[best], qx = V[4 + best], qy = V[8 + best], qz = V[12 + best];
            if (qw < 0) { qw = -qw; qx = -qx; qy = -qy; qz = -qz; }
            const double vn = sqrt(qx * qx + qy * qy + qz * qz);
            // (the angle lies in [0, pi], as the reference's cv2.Rodrigues returns it; a chunk whose cold start lies behind a pi
            // crossing of the sequence's root is told how many full turns the sequential trajectory has added by then)
            const double ang = 2 * atan2(vn, qw) + 6.283185307179586 * root_turns;
            double rv[3] = {0, 0, 0};
            if (vn > 1e-300) { rv[0] = qx / vn * ang; rv[1] = qy / vn * ang; rv[2] = qz / vn * ang; }
            const double R[9] = {1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qz * qw), 2 * (qx * qz + qy * qw),
                                 2 * (qx * qy + qz * qw), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qx * qw),
                                 2 * (qx * qz - qy * qw), 2 * (qy * qz + qx * qw), 1 - 2 * (qx * qx + qy * qy)};
            for (int r = 0; r < 3; ++r) {
                w.x[3 + r] = real(rv[r]);
                w.x[r] = real(cb[r] - (R[3 * r] * ca[0] + R[3 * r + 1] * ca[1] + R[3 * r + 2] * ca[2]));
            }
        }
        M2_SYNC();
    }

    // ---- the chunk loop
    // ---- per-block set-up: zero state, the per-model tables, the kinematic tree numbering and subtree masks
    M2_D void prologue() {
        CTA_FOR(i, d.NX) w.x[i] = 0;
        // the per-model tables: one bulk asynchronous copy of the host-built image (see carve()), waited for below
#if M2_GPU
        {
            const uint32_t bar = tc::smem_u32(static_cast<unsigned long long *>(w.mbar));
            if (cta.tid == 0) tc::mbar_init(bar, 1);
            __syncthreads();
            if (cta.tid == 0) {
                // (the region was last touched through the generic proxy, by the previous chunk of this block at most:
                // order those accesses before the asynchronous writes)
                tc::fence_async_smem();
                tc::mbar_expect_tx(bar, w.stage_bytes);
                tc::bulk_g2s(tc::smem_u32(m2_smem() + w.stage_ofs), m.stage_blob, w.stage_bytes, bar);
            }
            tc::mbar_wait(bar, 0);
            __syncthreads();
            if (cta.tid == 0) asm volatile("mbarrier.inval.shared::cta.b64 [%0];" :: "r"(bar) : "memory");
        }
#else
        for (uint32_t i = 0; i < w.stage_bytes; ++i) (m2_smem() + w.stage_ofs)[i] = m.stage_blob[i];
#endif
        CTA_FOR(i, 32) w.prof[i] = 0;
        M2_SYNC();
        if (cta.tid == 0) {                                    // pre-order numbering of the kinematic tree
            int *cur = w.jlist;
            for (int i = 0; i < d.nJ; ++i) w.c_tsz[i] = 1;
            for (int i = d.nJ - 1; i >= 0; --i) {              // fk_order lists parents before children
                const int j = w.c_fk_order[i], a = w.c_parents[j];
                if (a >= 0) w.c_tsz[a] += w.c_tsz[j];
            }
            int next_root = 0;
            for (int i = 0; i < d.nJ; ++i) {
                const int j = w.c_fk_order[i], a = w.c_parents[j];
                if (a < 0) { w.c_tin[j] = next_root; next_root += w.c_tsz[j]; }
                else { w.c_tin[j] = cur[a]; cur[a] += w.c_tsz[j]; }
                cur[j] = w.c_tin[j] + 1;
            }
        }
        M2_SYNC();
        CTA_FOR(j, d.nJ) {                                     // ancestor chain of every joint, root first
            int chain[kMaxDepth], depth = 0;
            for (int a = j; a >= 0 && depth < kMaxDepth; a = w.c_parents[a]) chain[depth++] = a;
            uint32_t cw[kMaxDepth / 4];
            for (int q = 0; q < kMaxDepth / 4; ++q) cw[q] = 0xffffffffu;
            for (int k = 0; k < depth; ++k) {
                const int c = chain[depth - 1 - k];
                cw[k >> 2] = (cw[k >> 2] & ~(255u << (8 * (k & 3)))) | (uint32_t(c) << (8 * (k & 3)));
            }
            for (int q = 0; q < kMaxDepth / 4; ++q) w.c_chain[j * (kMaxDepth / 4) + q] = cw[q];
        }
        CTA_FOR(idx, d.S * d.nJ) {                             // which of a slot's skinning joints hang below joint a
            const int sl = idx / d.nJ, a = idx - sl * d.nJ;
            const int ta = w.c_tin[a], na = w.c_tsz[a];
            int mask = 0;
            for (int i = 0; i < d.kw; ++i) {
                const int j = w.c_wj[sl * d.kw + i];
                if (j >= 0 && unsigned(w.c_tin[j] - ta) < unsigned(na)) mask |= 1 << i;
            }
            w.c_amask[idx] = uint8_t(mask);
        }
        M2_SYNC();
        stage_tables(0);
        stage_tables(1);
    }

    M2_D void run_chunk(int chunk) {
        const Options &o = job.opt;
        // Linearise mode (Stage I, Job::lin_mode): the block's "chunk" is the single frame `chunk`, taken at the state the
        // caller gives and left after its first evaluation / linearisation.  The frame's own terms are the Stage-II ones
        // without the temporal coupling -- data, pose prior (+ joint angles), with lin_step == 2 the finger term and, with
        // optimize_face, the jaw (poseF) and expression terms -- under the weights of the options as they are (no per-frame
        // visibility scaling: chmosh.py:327,350; the expression weight is never visibility-scaled).  It runs through the
        // same frame loop and the same solve_frame call as a chunk (one call site each: instruction cache, DESIGN.md 3).
        const bool lin = job.lin_mode != 0;
        // chunk table (host-built, mosh2_host::chunk_table): the chunk emits frames [f_emit, f_end) of the sequence that
        // starts at frame s0 of the job's frame axis (a job may hold several sequences of one subject back to back)
        const int *rec = job.chunk_tab + kChunkRec * chunk;
        const int f_emit = lin ? chunk : rec[0], f_end = lin ? chunk + 1 : rec[1], s0 = lin ? chunk : rec[2];
        const int warmup = lin ? 0 : rec[3], warm_full = lin ? 0 : rec[4];
        root_turns = lin ? 0 : rec[5];
        int f_begin = f_emit, f_full = f_emit;
        bool short_warmup = false;
        if (cta.tid == 0 && job.warm_f) job.warm_f[chunk] = -1;
        if (f_emit > s0 && warmup > 0) {   // (warmup < 0: resume, see below)
            // The warm-up is counted in SOLVED frames (frames with at least one visible marker; the others are skipped,
            // chmosh.py:586-588): walk back from the first emitted frame until `warmup` of them are found, so that a
            // marker drop-out in front of a chunk does not shorten the history the chunk converges on.  The last
            // `warm_full` solved warm-up frames run the full schedule.  A chunk that reaches the first frame of its
            // sequence is the reference's own recursion from its own start: exact, never "short".
            uint8_t *flag = reinterpret_cast<uint8_t *>(static_cast<real *>(w.red));      // >= 8*33*4 bytes of scratch
            const int per = cta.nthr < 512 ? cta.nthr : 512;
            const int max_back = 8 * warmup + 64;             // give up behind very long gaps
            if (cta.tid == 0) { w.isc[4] = 0; w.isc[5] = f_emit; w.isc[6] = f_emit; w.isc[7] = 0; }
            M2_SYNC();
            for (int base = f_emit - 1; base >= s0; base -= per) {
                if (cta.tid < per) {
                    const int f = base - cta.tid;
                    uint8_t any = 0;
                    if (f >= s0) for (int i = 0; i < d.M; ++i) any |= job.vis[size_t(f) * d.M + i];
                    flag[cta.tid] = any;
                }
                M2_SYNC();
                if (cta.tid == 0) {
                    int cnt = w.isc[4], fb = w.isc[5], ff = w.isc[6], stop = 0;
                    for (int t = 0; t < per && !stop; ++t) {
                        const int f = base - t;
                        if (f < s0 || cnt >= warmup) { stop = 1; break; }
                        if (f_emit - f > max_back) { stop = 2; break; }
                        if (flag[t]) { ++cnt; fb = f; if (cnt <= warm_full) ff = f; }
                    }
                    if (cnt >= warmup) stop = 1;
                    w.isc[4] = cnt; w.isc[5] = fb; w.isc[6] = ff; w.isc[7] = stop;
                }
                M2_SYNC();
                if (w.isc[7]) break;
            }
            f_begin = w.isc[5]; f_full = w.isc[6];
            // fewer solved warm-up frames than asked for, without having reached the start of the sequence
            short_warmup = w.isc[4] < warmup && w.isc[7] == 2;
            // The walk-back ran into the first frame of the sequence: the chunk starts where the reference starts.  It solves
            // the frames in front of it with the full schedule -- it is then the reference's own recursion from its own
            // start, bit for bit the rows the chunks in front of it emit, instead of a shortened warm-up whose first frames
            // are a light-frame approximation.  (At most warmup - 1 fully solved frames; with mosh2_schedule::first_extra
            // at the cost of a warm-up only the second chunk of a short-chunk schedule gets here.)
            if (w.isc[4] < warmup && w.isc[7] != 2) f_full = f_begin;
            M2_SYNC();
        }
        prologue();
        M2_T0();
        bool first = true, have_prev = false, have_dm_prev = false;
        fwd_at_x = false;
        if (warmup < 0 && f_emit > s0) {
            // Resume (boundary repair, mosh2_job_relaunch_chunks with chunk_warmup < 0): no warm-up of its own -- the chunk
            // continues the recursion from the rows the previous launch EMITTED for the last two solved frames in front of
            // it (the end of the previous chunk's trajectory, stored in the compute precision), i.e. exactly as that
            // chunk would have gone on.
            if (cta.tid == 0) {
                int f1 = -1, f2 = -1;
                for (int f = f_emit - 1; f >= s0 && f2 < 0; --f)
                    if (job.status[f] & ST_SOLVED) { if (f1 < 0) f1 = f; else f2 = f; }
                w.isc[4] = f1; w.isc[5] = f2;
            }
            M2_SYNC();
            const int f1 = w.isc[4], f2 = w.isc[5];
            if (f1 >= 0) {
                CTA_FOR(i, 3) w.x[i] = job.trans[size_t(f1) * 3 + i];
                CTA_FOR(i, d.PR) w.x[3 + i] = job.pose[size_t(f1) * d.PR + i];
                if (job.dmpls) CTA_FOR(i, d.nd) w.x[3 + d.PR + i] = job.dmpls[size_t(f1) * d.nd + i];
                if (f2 >= 0) CTA_FOR(i, d.PR) w.pose_prev[i] = job.pose[size_t(f2) * d.PR + i];
                first = false;
                have_prev = f2 >= 0;
                resuming = true;
                M2_SYNC();
                // the boundary check of a resumed chunk: the state it started from against the row of that frame as it
                // is when the check runs (it differs if the previous chunk was itself repaired afterwards)
                if (job.warm_x) {
                    CTA_FOR(i, d.NX) job.warm_x[size_t(chunk) * d.NX + i] = w.x[i];
                    if (cta.tid == 0) job.warm_f[chunk] = f1;
                }
            }
            M2_SYNC();
        }
        int calm = 0;                              // consecutive re-solved frames that coincide with the rows they replace
        wv = real(o.wt_velo); wdm = real(o.wt_dmpl); wex = real(o.wt_extrap);
        wxp = real(o.wt_expr);
        const bool fingers = o.optimize_fingers != 0, dyn = o.optimize_dynamics != 0 && d.nd - m.n_expr > 0;
        const bool face = o.optimize_face != 0 && m.face_hi > m.face_lo;
        const bool has_prior = d.K > 0;
        njl = 0;
        hand_free = false;
#pragma unroll 1
        for (int f = f_begin; f < f_end; ++f) {
            n_iter = n_eval = n_build = n_min = 0;
            frame_flags = 0;
            CTA_FOR(i, d.M) w.vis[i] = job.vis[size_t(f) * d.M + i];
            CTA_FOR(i, 3 * d.M) w.obs[i] = job.obs[size_t(f) * 3 * d.M + i];
            M2_SYNC();
            {
                real cnt[1] = {0};
                CTA_FOR(i, d.M) cnt[0] += w.vis[i] ? real(1) : real(0);
                cta_reduce<real, 1>(cta, cnt, w.red);
                nvis = int(cnt[0] + real(0.5));
            }
            if (nvis == 0) {                                   // chmosh.py:586-588
                if (f >= f_emit && cta.tid == 0) job.status[f] = ST_SKIPPED;
                continue;
            }
            real anneal = 1;                                   // (none in linearise mode: wp_frame, wH and wF stay the options')
            if (nvis < d.M && !lin) anneal += real(d.M - nvis) / real(d.M) * real(o.wt_annealing);
            wd = real(o.wt_data) * (real(o.num_train_markers) / real(nvis));
            wp_frame = has_prior ? real(o.wt_poseB) * anneal : real(0);
            wH = real(o.wt_poseH) * anneal;
            wF = real(o.wt_poseF) * anneal;
            has_velo = have_prev;                              // chmosh.py:624-626
            if (has_velo) {
                CTA_FOR(i, d.PR) w.velo_tgt[i] = real(2) * w.x[3 + i] - w.pose_prev[i];
                M2_SYNC();
            }
            if (!first) {
                CTA_FOR(i, d.PR) w.pose_prev[i] = w.x[3 + i];                               // chmosh.py:656-659
                have_prev = true;
                if (dyn) { CTA_FOR(i, d.nd - m.n_expr) w.dm_tgt[i] = w.x[3 + d.PR + i]; have_dm_prev = true; }
                M2_SYNC();
            }
            has_extrap = dyn && have_dm_prev;
            if (short_warmup && f >= f_emit) frame_flags |= ST_SHORT_WARMUP;
            if (lin) {
                lin_f = f;
                CTA_FOR(i, d.NX) w.x[i] = job.lin_x[size_t(f) * d.NX + i];
                wd = real(o.wt_data);
                wp_frame = has_prior ? real(o.wt_poseB) : real(0);
                wH = real(o.wt_poseH);
                has_velo = false; has_extrap = false;
                first = false;
                M2_SYNC();
            }
            solve_frame(f, !lin && f >= f_emit, first, fingers, dyn, face, /*light=*/!first && f < f_full);
            if (lin && cta.tid == 0) job.status[f] = ST_SOLVED;
            if (resuming) {
                // merged with the old trajectory (two frames in a row within round-off of the rows they replace: the state
                // the recursion carries, pose_t and pose_{t-1}, is the old one): the rest of the chunk stands as it is
                calm = resume_diff <= real(job.merge_tol) ? calm + 1 : 0;
                if (calm >= 2) break;
            }
            if (f < f_emit && job.warm_x) {      // (overwritten until the last warm-up frame: its state is what counts)
                CTA_FOR(i, d.NX) job.warm_x[size_t(chunk) * d.NX + i] = w.x[i];
                if (cta.tid == 0) job.warm_f[chunk] = f;
            }
            first = false;
        }
        M2_TACC(17);
#if defined(MOSH2_PROFILE) && M2_GPU
        if (cta.tid == 0 && job.prof) for (int i = 0; i < 32; ++i) atomicAdd(reinterpret_cast<unsigned long long *>(job.prof + i), (unsigned long long)w.prof[i]);
#endif
    }
#undef CTA_FOR
};

}  // namespace mosh2
