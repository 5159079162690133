// Development test (GPU): the Stage-II kernel's device Gauss-Newton solve -- Solver::gauss_newton (Jacobi scaling, the
// pipelined blocked Cholesky with the right-hand side as row n, the four-warp backward solve) and Solver::symv -- on one
// given system, driven by a test kernel through the kernel's own device functions.
//   built by moshpp_b200.build.build_gn_test() as a shared library, called through ctypes by tests/test_gpu_gauss_newton.py
//
// The workspace is the product's layout for the model dimensions passed in (gauss_newton_case.h).  Before A and g are
// written, the whole dynamic shared memory and the global workspace are filled with NaN bytes, so that a read of anything
// the solve did not write first -- identity padding, masked columns, the tail of tmp -- turns the result non-finite.
// This kernel is not mosh2_stageii_kernel: the same source, compiled in a different kernel, gets a different register
// allocation.  It pins the algorithm, the masks and the synchronisation of the GPU branch, not the product's binary.
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>

#include "../../moshpp_b200/csrc/mosh2_device.cuh"
#include "gauss_newton_case.h"

namespace {

// the launch bound of mosh2_stageii_kernel (mosh2.cu threads_for)
template <class real> constexpr int kThreads = sizeof(real) == 4 ? 384 : 256;

template <class real, bool BIG>
__global__ void __launch_bounds__(kThreads<real>, 1)
gn_kernel(const __grid_constant__ mosh2::Model<real> m, const __grid_constant__ mosh2::Work<real, BIG> w,
          const __grid_constant__ mosh2::Dims d, char *gws, unsigned smem, int n, const real *A, const real *g,
          real *dgn, real *Ag, int *ok) {
    unsigned char *sm = mosh2::m2_smem();
    for (unsigned i = threadIdx.x; i < smem; i += blockDim.x) sm[i] = gn_case::kNaN;
    __syncthreads();
    if (BIG) {      // as mosh2_stageii_kernel: the global workspace's base parked in the shared-memory header
        if (threadIdx.x == 0) *reinterpret_cast<char **>(sm) = gws;
        __syncthreads();
    }
    real *wA = w.A, *wg = w.g;
    for (int e = threadIdx.x; e < n * n; e += blockDim.x) wA[(e / n) * d.lda + e % n] = A[e];
    for (int i = threadIdx.x; i < n; i += blockDim.x) wg[i] = g[i];
    __syncthreads();
    const mosh2::Job<real> job{};
    mosh2::Solver<real, BIG> s(m, job, w, d, mosh2::Cta{int(threadIdx.x), int(blockDim.x)});
    const bool solved = s.gauss_newton(n);
    s.symv(w.g, w.Ag, n);
    for (int i = threadIdx.x; i < n; i += blockDim.x) { dgn[i] = w.dgn[i]; Ag[i] = w.Ag[i]; }
    if (threadIdx.x == 0) *ok = solved ? 1 : 0;
}

#define CK(x) do { const cudaError_t e_ = (x); if (e_ != cudaSuccess) { std::fprintf(stderr, "gauss_newton_test: %s at line %d\n", cudaGetErrorString(e_), __LINE__); rc = -2; goto done; } } while (0)

template <class real, bool BIG>
int run(int threads, const mosh2_model_desc *desc, int n, const double *A, const double *g, double *dgn_out, double *Ag_out,
        int *ok_out) {
    mosh2::Model<real> m = mosh2_host::model_dims<real>(*desc);
    mosh2::Dims d;
    mosh2::Work<real, BIG> w;
    size_t smem = 0, gws_bytes = 0;
    if (n < 1 || n > m.n2 || threads < 128 || threads > kThreads<real> || threads % 32) return -1;
    if (!gn_case::layout<real, BIG>(m, d, w, smem, gws_bytes)) return -1;
    const size_t nn = size_t(n) * n;
    std::vector<real> h_in(nn + n), h_out(2 * size_t(n));
    for (size_t i = 0; i < nn; ++i) h_in[i] = real(A[i]);
    for (int i = 0; i < n; ++i) h_in[nn + i] = real(g[i]);
    real *d_in = nullptr, *d_out = nullptr;
    char *d_gws = nullptr;
    int *d_ok = nullptr, ok = -1, rc = 0;
    CK(cudaMalloc(&d_in, h_in.size() * sizeof(real)));
    CK(cudaMalloc(&d_out, h_out.size() * sizeof(real)));
    CK(cudaMalloc(&d_ok, sizeof(int)));
    if (BIG) {
        CK(cudaMalloc(&d_gws, gws_bytes));
        CK(cudaMemset(d_gws, gn_case::kNaN, gws_bytes));
    }
    CK(cudaMemcpy(d_in, h_in.data(), h_in.size() * sizeof(real), cudaMemcpyHostToDevice));
    CK(cudaMemset(d_out, gn_case::kNaN, h_out.size() * sizeof(real)));
    CK(cudaFuncSetAttribute(gn_kernel<real, BIG>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    gn_kernel<real, BIG><<<1, threads, smem>>>(m, w, d, d_gws, unsigned(smem), n, d_in, d_in + nn, d_out, d_out + n, d_ok);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(h_out.data(), d_out, h_out.size() * sizeof(real), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(&ok, d_ok, sizeof(int), cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; ++i) { dgn_out[i] = double(h_out[i]); Ag_out[i] = double(h_out[n + i]); }
    *ok_out = ok;
done:
    cudaFree(d_in); cudaFree(d_out); cudaFree(d_ok); cudaFree(d_gws);
    return rc;
}

}  // namespace

// Solves A dgn = g (A: n x n row-major, the lower triangle is what the factorisation reads) and forms Ag = A g in the
// workspace of a model with the dimensions of `desc` (n <= desc->n_free2), in float32 or float64 (rounded on the way in,
// widened on the way out), with the workspace in shared memory (big = 0) or in a global workspace (big = 1), on
// `threads` threads (a multiple of 32 from 128 up to the kernel's launch bound).  *ok: gauss_newton's return value.
// Returns 0, -1 for arguments or a layout the library would not launch, -2 on a CUDA error.
extern "C" int gn_run(int precision, int big, int threads, const mosh2_model_desc *desc, int n, const double *A, const double *g,
                      double *dgn_out, double *Ag_out, int *ok_out) {
    if (precision == MOSH2_F64)
        return big ? run<double, true>(threads, desc, n, A, g, dgn_out, Ag_out, ok_out)
                   : run<double, false>(threads, desc, n, A, g, dgn_out, Ag_out, ok_out);
    return big ? run<float, true>(threads, desc, n, A, g, dgn_out, Ag_out, ok_out)
               : run<float, false>(threads, desc, n, A, g, dgn_out, Ag_out, ok_out);
}
