// A pixel's simplex in the permutohedral lattice (permutohedral.cpp:191-242): features, elevation, the closest
// remainder-0 vertex and the ranks, in the reference's float32 operation order (every op an explicit __f*_rn
// intrinsic, no FMA contraction).  The lattice build (lattice.cu: k_lattice_insert) and the kernel-bandwidth gradient
// (meanfield.cu: k_kg_pass) share it, so the gradient rotates by exactly the ranks the build hashed.
#pragma once
#include <cstdint>

namespace dsrg {

// x/sigma_x, y/sigma_y and, for the bilateral lattice (D = 5), r/sigma_r, g/sigma_g, b/sigma_b of pixel i of image b
// of `image` ([B][N][3] uint8) (densecrf.cpp:65-78)
template <int D>
__device__ __forceinline__ void lattice_features(int x, int y, const uint8_t *image, int b, int N, int i,
                                                 const float *sigma, float *f) {
    f[0] = __fdiv_rn((float)x, sigma[0]);
    f[1] = __fdiv_rn((float)y, sigma[1]);
    if (D == 5) {
        const uint8_t *px = image + ((size_t)b * N + i) * 3;
        f[2] = __fdiv_rn((float)px[0], sigma[2]);
        f[3] = __fdiv_rn((float)px[1], sigma[3]);
        f[4] = __fdiv_rn((float)px[2], sigma[4]);
    }
}

// elevate f, find the remainder-0 vertex rem0 and the ranks, back onto the plane; el, rem0, rank are [D + 1]
template <int D>
__device__ __forceinline__ void lattice_simplex(const float *f, const float *scale, float *el, float *rem0,
                                                int *rank) {
    // elevate (:201-207)
    float sm = 0.0f;
#pragma unroll
    for (int j = D; j > 0; j--) {
        float cf = __fmul_rn(f[j - 1], scale[j - 1]);
        el[j] = __fsub_rn(sm, __fmul_rn((float)j, cf));
        sm = __fadd_rn(sm, cf);
    }
    el[0] = sm;
    // closest 0-coloured simplex (:210-220); cvtps_epi32 under MXCSR-nearest == rintf
    const float inv = __fdiv_rn(1.0f, (float)(D + 1));
    const float dp1 = (float)(D + 1);
    int isum = 0;
#pragma unroll
    for (int k = 0; k <= D; k++) {
        float v = rintf(__fmul_rn(inv, el[k]));
        rem0[k] = __fmul_rn(v, dp1);
        isum += (int)v;
    }
    // rank (:223-233): strict <, ties increment the later coordinate
#pragma unroll
    for (int k = 0; k <= D; k++) rank[k] = 0;
#pragma unroll
    for (int k = 0; k < D; k++) {
        float di = __fsub_rn(el[k], rem0[k]);
#pragma unroll
        for (int j = k + 1; j <= D; j++) {
            float dj = __fsub_rn(el[j], rem0[j]);
            if (di < dj) rank[k]++; else rank[j]++;
        }
    }
    // back onto the plane (:236-242)
#pragma unroll
    for (int k = 0; k <= D; k++) {
        rank[k] += isum;
        if (rank[k] < 0) {
            rank[k] += D + 1;
            rem0[k] = __fadd_rn(rem0[k], dp1);
        } else if (rank[k] >= D + 1) {
            rank[k] -= D + 1;
            rem0[k] = __fsub_rn(rem0[k], dp1);
        }
    }
}

}  // namespace dsrg
