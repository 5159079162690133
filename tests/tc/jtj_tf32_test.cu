// Development test (GPU): A = J^T J on the tensor cores with the 3xTF32 split the Stage-II kernel uses
// (mosh2::tc::jtj_block_tf32: mma.sync m16n8k8, hi hi^T and the cross terms in separate register accumulators, their
// sum added to A once per tile), against a float64 product, for the operand shapes of all model families.
//   built by moshpp_b200.build.build_tc_test(), run by tests/test_gpu_parity.py::test_tf32_jtj_building_block
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cmath>
#include <vector>
#include <cuda_runtime.h>

#include "../../moshpp_b200/csrc/mosh2_device.cuh"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e_), __LINE__); exit(2); } } while (0)

// One block: the rows of J in tiles of KT rows; a tile is copied into shared memory with the kernel's row length
// (columns rounded up to 4, zero padded), then every warp adds its 16x16 blocks of the upper triangle to D.
__global__ void __launch_bounds__(384, 1) jtj_kernel(const float *J, int rows, int n, float *D, int KT) {
    extern __shared__ __align__(16) float tile[];
    const int npad = (n + 3) & ~3, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    const int g = lane >> 2, tq = lane & 3, nb16 = (n + 15) >> 4, ntile = nb16 * (nb16 + 1) / 2;
    for (int r0 = 0; r0 < rows; r0 += KT) {
        const int tr = rows - r0 < KT ? rows - r0 : KT;
        for (int e = threadIdx.x; e < tr * npad; e += blockDim.x) {
            const int k = e / npad, i = e - k * npad;
            tile[e] = i < n ? J[(r0 + k) * n + i] : 0.f;
        }
        __syncthreads();
        for (int t = warp; t < ntile; t += nwarp) {
            int ti, tj;
            mosh2::upper_block(t, nb16, ti, tj);
            const int i0 = 16 * ti, j0 = 16 * tj;
            float hh[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}}, cr[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
            mosh2::tc::jtj_block_tf32(tile, npad, tr, npad, i0, j0, hh, cr);
            for (int mi = 0; mi < 2; ++mi)
                for (int ni = 0; ni < 2; ++ni)
                    for (int e = 0; e < 2; ++e) {
                        const int i = i0 + 8 * mi + g, j = j0 + 8 * ni + 2 * tq + e;
                        if (j < n && i <= j) {
                            const float v = D[i * n + j] + (hh[ni][2 * mi + e] + cr[ni][2 * mi + e]);
                            D[i * n + j] = v;
                            D[j * n + i] = v;
                        }
                    }
        }
        __syncthreads();
    }
}

static int run(int rows, int n, int KT) {
    std::vector<float> J(rows * n);
    srand(1);
    for (auto &v : J) v = (rand() / float(RAND_MAX) - 0.5f) * ((rand() % 7 == 0) ? 40.f : 1.f);
    std::vector<double> ref(n * n, 0.0);
    for (int r = 0; r < rows; ++r)
        for (int i = 0; i < n; ++i)
            for (int j = 0; j < n; ++j) ref[i * n + j] += double(J[r * n + i]) * double(J[r * n + j]);
    float *dJ, *dD;
    CK(cudaMalloc(&dJ, J.size() * 4)); CK(cudaMalloc(&dD, n * n * 4));
    CK(cudaMemcpy(dJ, J.data(), J.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaMemset(dD, 0, n * n * 4));
    const size_t smem = size_t(KT) * ((n + 3) & ~3) * 4;
    CK(cudaFuncSetAttribute(jtj_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    jtj_kernel<<<1, 384, smem>>>(dJ, rows, n, dD, KT);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    std::vector<float> D(n * n);
    CK(cudaMemcpy(D.data(), dD, n * n * 4, cudaMemcpyDeviceToHost));
    double scale = 0, e = 0;
    for (int i = 0; i < n; ++i) scale = fmax(scale, ref[i * n + i]);
    for (int i = 0; i < n * n; ++i) e = fmax(e, fabs(D[i] - ref[i]));
    printf("rows %3d n %3d KT %2d  3xTF32: max |D - ref| / max diag = %.3e\n", rows, n, KT, e / scale);
    cudaFree(dJ); cudaFree(dD);
    return !(e / scale < 1.5e-6);
}

int main() {
    int bad = 0;
    bad |= run(159, 111, 30);     // SMPL-H body + fingers, 10-marker tiles
    bad |= run(159, 111, 60);     // ... 20-marker tiles
    bad |= run(80, 30, 30);
    bad |= run(80, 6, 60);
    bad |= run(40, 30, 60);
    bad |= run(212, 111, 60);
    bad |= run(212, 130, 60);
    printf(bad ? "FAILED\n" : "OK\n");
    return bad;
}
