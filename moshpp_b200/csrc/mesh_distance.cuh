// mesh_distance.cuh -- point-to-triangle-mesh distance with derivatives on the GPU: the surface term of MoSh++ Stage I
// (SURVEY.md 8(f-2)), the one native component of the reference:
//   scan2mesh/mesh_distance/sample2meshdist.h:67-207   distance of a sample to the plane / an edge / a vertex of its nearest
//                                                      triangle under f = identity | square | Geman-McClure(square), with
//                                                      the derivatives wrt the sample and the triangle's vertices;
//   scan2mesh/mesh_distance/sample2meshdist.pyx:55-103 the loop over samples (OpenMP prange);
//   scan2mesh/mesh_distance_main.py:346-376            the nearest (triangle, part) query (CGAL AABB tree of psbody.mesh).
//
// Three kernels:
//   soup     gathers the triangles into a contiguous float32 "soup" (12 floats per triangle, 16-byte aligned) once per mesh;
//   nearest  brute-force closest-point search.  grid = (blocks of 128 samples) x (triangle ranges): every block streams its
//            triangle range through a two-stage shared-memory ring filled by bulk asynchronous copies (cp.async.bulk -- the
//            TMA engine -- completing on an mbarrier); lane = sample, every lane tests the same triangle (shared-memory
//            broadcast); the per-sample winner over all blocks is a 64-bit atomicMin on (distance^2 bits, triangle, part);
//   evaluate the reference's closed forms for the winning (triangle, part) in float64, one thread per sample.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace mosh2_md {

constexpr int kSoupFloats = 12;          // a(3) b(3) c(3) + 3 pad: 48 bytes, so any tile is 16-byte aligned and sized
constexpr int kTileTris = 384;           // triangles per stage: 18 KB (two stages stay inside the static 48 KB)
constexpr int kSamplesPerBlock = 128;

__global__ void soup_kernel(const double *__restrict__ verts, const int *__restrict__ faces, int T, float *__restrict__ soup) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    for (int k = 0; k < 3; ++k) {
        const int v = faces[3 * t + k];
        for (int c = 0; c < 3; ++c) soup[size_t(t) * kSoupFloats + 3 * k + c] = float(verts[3 * size_t(v) + c]);
    }
    for (int c = 9; c < kSoupFloats; ++c) soup[size_t(t) * kSoupFloats + c] = 0.f;
}

__device__ __forceinline__ uint32_t smem_addr(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
                 "@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}\n" :: "r"(bar), "r"(parity) : "memory");
}
// bulk asynchronous copy global -> shared (TMA engine, no tensor map needed for a contiguous run)
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// A triangle whose sides are parallel to within 1e-5 rad (|ab x ac|^2 <= 1e-10 |ab|^2 |ac|^2, far above the float32
// rounding of the cross product) has no plane to speak of: the Voronoi tests below can fall through to the interior
// with va + vb + vc at round-off level, and the plane distance of such a triangle is 0 / 0.
__device__ __forceinline__ bool degenerate(const float ab[3], const float ac[3]) {
    const float n0 = ab[1] * ac[2] - ab[2] * ac[1], n1 = ab[2] * ac[0] - ab[0] * ac[2], n2 = ab[0] * ac[1] - ab[1] * ac[0];
    const float l2 = (ab[0] * ab[0] + ab[1] * ab[1] + ab[2] * ab[2]) * (ac[0] * ac[0] + ac[1] * ac[1] + ac[2] * ac[2]);
    return !(n0 * n0 + n1 * n1 + n2 * n2 > 1e-10f * l2);
}

// squared distance from p to the closest of the three edges of a degenerate triangle, as edge (1..3) or, where the
// closest point is an end of the edge, vertex (4..6) part
__device__ __noinline__ float closest_on_edges(const float p[3], const float *__restrict__ tri, int *part) {
    float best = 3.0e38f;
    int bp = 4;
    for (int e = 0; e < 3; ++e) {
        const float *u = tri + 3 * e, *v = tri + 3 * ((e + 1) % 3);
        const float uv[3] = {v[0] - u[0], v[1] - u[1], v[2] - u[2]}, up[3] = {p[0] - u[0], p[1] - u[1], p[2] - u[2]};
        const float l2 = uv[0] * uv[0] + uv[1] * uv[1] + uv[2] * uv[2], t = up[0] * uv[0] + up[1] * uv[1] + up[2] * uv[2];
        float s;
        int pt;
        if (t <= 0.f || !(l2 > 0.f)) { s = 0.f; pt = 4 + e; }
        else if (t >= l2) { s = 1.f; pt = 4 + (e + 1) % 3; }
        else { s = t / l2; pt = 1 + e; }
        float d = 0.f;
        for (int k = 0; k < 3; ++k) { const float qk = up[k] - s * uv[k]; d += qk * qk; }
        if (d < best) { best = d; bp = pt; }
    }
    *part = bp;
    return best;
}

// squared distance from p to triangle (a, b, c) and the part the closest point lies on: 0 interior, 1..3 the edges
// ab / bc / ca, 4..6 the vertices a / b / c (Voronoi regions of the triangle)
__device__ __forceinline__ float closest_part(const float p[3], const float *__restrict__ tri, int *part) {
    const float ab[3] = {tri[3] - tri[0], tri[4] - tri[1], tri[5] - tri[2]};
    const float ac[3] = {tri[6] - tri[0], tri[7] - tri[1], tri[8] - tri[2]};
    const float ap[3] = {p[0] - tri[0], p[1] - tri[1], p[2] - tri[2]};
    const float d1 = ab[0] * ap[0] + ab[1] * ap[1] + ab[2] * ap[2], d2 = ac[0] * ap[0] + ac[1] * ap[1] + ac[2] * ap[2];
    float q[3];
    int pt;
    if (d1 <= 0.f && d2 <= 0.f) { pt = 4; q[0] = ap[0]; q[1] = ap[1]; q[2] = ap[2]; }
    else {
        const float bp[3] = {p[0] - tri[3], p[1] - tri[4], p[2] - tri[5]};
        const float d3 = ab[0] * bp[0] + ab[1] * bp[1] + ab[2] * bp[2], d4 = ac[0] * bp[0] + ac[1] * bp[1] + ac[2] * bp[2];
        const float vc = d1 * d4 - d3 * d2;
        if (d3 >= 0.f && d4 <= d3) { pt = 5; q[0] = bp[0]; q[1] = bp[1]; q[2] = bp[2]; }
        else if (vc <= 0.f && d1 >= 0.f && d3 <= 0.f) {
            const float v = d1 / (d1 - d3);
            pt = 1;
            for (int k = 0; k < 3; ++k) q[k] = ap[k] - v * ab[k];
        } else {
            const float cp[3] = {p[0] - tri[6], p[1] - tri[7], p[2] - tri[8]};
            const float d5 = ab[0] * cp[0] + ab[1] * cp[1] + ab[2] * cp[2], d6 = ac[0] * cp[0] + ac[1] * cp[1] + ac[2] * cp[2];
            const float vb = d5 * d2 - d1 * d6, va = d3 * d6 - d5 * d4;
            if (d6 >= 0.f && d5 <= d6) { pt = 6; q[0] = cp[0]; q[1] = cp[1]; q[2] = cp[2]; }
            else if (vb <= 0.f && d2 >= 0.f && d6 <= 0.f) {
                const float w = d2 / (d2 - d6);
                pt = 3;
                for (int k = 0; k < 3; ++k) q[k] = ap[k] - w * ac[k];
            } else if (va <= 0.f && (d4 - d3) >= 0.f && (d5 - d6) >= 0.f) {
                const float w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
                pt = 2;
                for (int k = 0; k < 3; ++k) q[k] = bp[k] - w * (tri[6 + k] - tri[3 + k]);
            } else if (degenerate(ab, ac)) {
                return closest_on_edges(p, tri, part);
            } else {
                const float den = 1.f / (va + vb + vc), v = vb * den, w = vc * den;
                pt = 0;
                for (int k = 0; k < 3; ++k) q[k] = ap[k] - v * ab[k] - w * ac[k];
            }
        }
    }
    *part = pt;
    return q[0] * q[0] + q[1] * q[1] + q[2] * q[2];
}

__global__ void __launch_bounds__(kSamplesPerBlock)
nearest_kernel(const float *__restrict__ samples, int S, const float *__restrict__ soup, int T, int tris_per_block,
               unsigned long long *__restrict__ best) {
    __shared__ __align__(128) float tiles[2][kTileTris * kSoupFloats];
    __shared__ __align__(8) unsigned long long full[2];
    const int s = blockIdx.x * kSamplesPerBlock + threadIdx.x;
    const int t_begin = blockIdx.y * tris_per_block;
    int t_end = t_begin + tris_per_block;
    if (t_end > T) t_end = T;
    const int ntiles = (t_end - t_begin + kTileTris - 1) / kTileTris;
    float p[3] = {0.f, 0.f, 0.f};
    if (s < S) { p[0] = samples[3 * s]; p[1] = samples[3 * s + 1]; p[2] = samples[3 * s + 2]; }
    if (threadIdx.x == 0) {
        mbar_init(smem_addr(&full[0]), 1);
        mbar_init(smem_addr(&full[1]), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto issue = [&](int tile) {              // one thread: arm the stage's barrier with the byte count, start the bulk copy
        const int t0 = t_begin + tile * kTileTris;
        const int n = (t_end - t0 < kTileTris) ? t_end - t0 : kTileTris;
        const uint32_t bytes = uint32_t(n) * kSoupFloats * sizeof(float);
        const uint32_t bar = smem_addr(&full[tile & 1]);
        mbar_expect_tx(bar, bytes);
        bulk_g2s(smem_addr(&tiles[tile & 1][0]), soup + size_t(t0) * kSoupFloats, bytes, bar);
    };
    if (threadIdx.x == 0) {
        if (ntiles > 0) issue(0);
        if (ntiles > 1) issue(1);
    }
    float best_d = 3.0e38f;
    int best_t = 0, best_p = 0;
    for (int tile = 0; tile < ntiles; ++tile) {
        mbar_wait(smem_addr(&full[tile & 1]), (tile >> 1) & 1);
        const int t0 = t_begin + tile * kTileTris;
        const int n = (t_end - t0 < kTileTris) ? t_end - t0 : kTileTris;
        const float *tri = &tiles[tile & 1][0];
#pragma unroll 4
        for (int i = 0; i < n; ++i) {         // every lane reads the same triangle: a shared-memory broadcast
            int part;
            const float d = closest_part(p, tri + i * kSoupFloats, &part);
            if (d < best_d) { best_d = d; best_t = t0 + i; best_p = part; }
        }
        __syncthreads();                      // everybody is done with this stage
        if (threadIdx.x == 0 && tile + 2 < ntiles) issue(tile + 2);
    }
    if (s < S && ntiles > 0) {
        const unsigned long long key = (static_cast<unsigned long long>(__float_as_uint(best_d)) << 32) |
                                       (static_cast<unsigned long long>(uint32_t(best_t)) << 3) | uint32_t(best_p);
        atomicMin(best + s, key);             // distances are >= 0: their bit patterns order like the numbers
    }
}

__global__ void unpack_kernel(const unsigned long long *__restrict__ best, int S, int *__restrict__ tri, int *__restrict__ part) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const uint32_t lo = uint32_t(best[s] & 0xffffffffull);
    tri[s] = int(lo >> 3);
    part[s] = int(lo & 7u);
}

// ---- the reference's closed forms in float64 -------------------------------------------------------------------------
__device__ __forceinline__ void f_and_df(int kind, double sigma, double d, double *f, double *df) {     // robust.h:14-52
    if (kind == 0) { *f = d; *df = 1.0; }
    else if (kind == 1) { *f = d * d; *df = 2.0 * d; }
    else {
        const double s2 = sigma * sigma, x2 = d * d, q = s2 + x2;
        *f = s2 * x2 / q;
        *df = (s2 / q - s2 * x2 / (q * q)) * 2.0 * d;
    }
}
__device__ __forceinline__ void cross(const double *a, const double *b, double *o) {
    o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ double dot(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// |(x-a) x (x-b)| / |b-a| and its gradients (sample2meshdist.h:134-158); gradients are ADDED to dx, da, db
__device__ void point_line(int kind, double sigma, const double *x, const double *a, const double *b, double *val, double *dx,
                           double *da, double *db) {
    double xa[3], xb[3], ba[3], w[3];
    for (int k = 0; k < 3; ++k) { xa[k] = x[k] - a[k]; xb[k] = x[k] - b[k]; ba[k] = b[k] - a[k]; }
    cross(xa, xb, w);
    const double nw = sqrt(dot(w, w)), nab = sqrt(dot(ba, ba));
    double f, df;
    f_and_df(kind, sigma, nw / nab, &f, &df);
    double r[3], d[3], ab[3], bx[3], t[3];
    for (int k = 0; k < 3; ++k) { r[k] = w[k] / (nw * nab); d[k] = ba[k] * nw / (nab * nab * nab); ab[k] = -ba[k]; bx[k] = -xb[k]; }
    cross(ab, r, t);
    for (int k = 0; k < 3; ++k) dx[k] += df * t[k];
    cross(bx, r, t);
    for (int k = 0; k < 3; ++k) da[k] += df * (t[k] + d[k]);
    cross(xa, r, t);
    for (int k = 0; k < 3; ++k) db[k] += df * (t[k] - d[k]);
    *val = f;
}

__device__ void point_point(int kind, double sigma, const double *x, const double *a, double *val, double *dx, double *da) {
    double xa[3] = {x[0] - a[0], x[1] - a[1], x[2] - a[2]};
    const double dist = sqrt(dot(xa, xa));
    double f, df;
    f_and_df(kind, sigma, dist, &f, &df);
    for (int k = 0; k < 3; ++k) { dx[k] += df * xa[k] / dist; da[k] -= df * xa[k] / dist; }
    *val = f;
}

// det(x-a, b-a, c-b) / |(b-a) x (c-b)| and its gradients (sample2meshdist.h:67-100)
__device__ void point_plane(int kind, double sigma, const double *x, const double *a, const double *b, const double *c, double *val,
                            double *dx, double *da, double *db, double *dc) {
    double A[3][3];
    for (int k = 0; k < 3; ++k) { A[0][k] = x[k] - a[k]; A[1][k] = b[k] - a[k]; A[2][k] = c[k] - b[k]; }
    const double det = A[0][0] * (A[1][1] * A[2][2] - A[2][1] * A[1][2]) - A[1][0] * (A[0][1] * A[2][2] - A[2][1] * A[0][2]) +
                       A[2][0] * (A[0][1] * A[1][2] - A[1][1] * A[0][2]);
    // adjugate: column j = d det / d (row j of A)
    const double J[3][3] = {
        {A[2][2] * A[1][1] - A[2][1] * A[1][2], A[0][2] * A[2][1] - A[0][1] * A[2][2], A[0][1] * A[1][2] - A[0][2] * A[1][1]},
        {A[1][2] * A[2][0] - A[1][0] * A[2][2], A[0][0] * A[2][2] - A[0][2] * A[2][0], A[0][2] * A[1][0] - A[0][0] * A[1][2]},
        {A[1][0] * A[2][1] - A[1][1] * A[2][0], A[0][1] * A[2][0] - A[0][0] * A[2][1], A[0][0] * A[1][1] - A[0][1] * A[1][0]}};
    const double *z = A[1], *y = A[2];
    double n[3];
    cross(z, y, n);
    const double s = sqrt(dot(n, n)), zy = dot(z, y), yy = dot(y, y), zz = dot(z, z);
    double f, df;
    f_and_df(kind, sigma, det / s, &f, &df);
    const double s2 = s * s;
    for (int k = 0; k < 3; ++k) {
        const double ds_a = -(z[k] * yy - y[k] * zy) / s, ds_c = (y[k] * zz - z[k] * zy) / s, ds_b = -ds_a - ds_c;
        dx[k] += df * (J[k][0] / s);
        da[k] += df * ((-J[k][0] - J[k][1]) / s - ds_a * (det / s2));
        db[k] += df * ((J[k][1] - J[k][2]) / s - ds_b * (det / s2));
        dc[k] += df * (J[k][2] / s - ds_c * (det / s2));
    }
    *val = f;
}

// Distance<F>::tri (sample2meshdist.h:182-195) for every sample's (triangle, part)
__global__ void evaluate_kernel(int kind, double sigma, const double *__restrict__ samples, int S, const double *__restrict__ verts,
                                const int *__restrict__ faces, const int *__restrict__ tri, const int *__restrict__ part,
                                double *__restrict__ value, double *__restrict__ d_sample, double *__restrict__ d_tri) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const int t = tri[s], pt = part[s];
    double x[3], a[3], b[3], c[3];
    for (int k = 0; k < 3; ++k) {
        x[k] = samples[3 * s + k];
        a[k] = verts[3 * size_t(faces[3 * t]) + k];
        b[k] = verts[3 * size_t(faces[3 * t + 1]) + k];
        c[k] = verts[3 * size_t(faces[3 * t + 2]) + k];
    }
    double dx[3] = {0, 0, 0}, da[3] = {0, 0, 0}, db[3] = {0, 0, 0}, dc[3] = {0, 0, 0}, val = 0;
    switch (pt) {
        case 0: point_plane(kind, sigma, x, a, b, c, &val, dx, da, db, dc); break;
        case 1: point_line(kind, sigma, x, a, b, &val, dx, da, db); break;
        case 2: point_line(kind, sigma, x, b, c, &val, dx, db, dc); break;
        case 3: point_line(kind, sigma, x, c, a, &val, dx, dc, da); break;
        case 4: point_point(kind, sigma, x, a, &val, dx, da); break;
        case 5: point_point(kind, sigma, x, b, &val, dx, db); break;
        default: point_point(kind, sigma, x, c, &val, dx, dc); break;
    }
    value[s] = val;
    for (int k = 0; k < 3; ++k) {
        d_sample[3 * s + k] = dx[k];
        d_tri[9 * s + k] = da[k];
        d_tri[9 * s + 3 + k] = db[k];
        d_tri[9 * s + 6 + k] = dc[k];
    }
}

}  // namespace mosh2_md
