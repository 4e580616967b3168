// The kernel-bandwidth and feature gradient's shared pieces (the math: the comment above them in meanfield.cu), used
// by the fused backward (meanfield.cu) and the label-chunked one (meanfield_wide.cu).
#pragma once
#include "common.cuh"
#include "simplex.cuh"

namespace dsrg {

struct KgLat {
    const int32_t *off;      // [nimg][d+1][N]
    const float *bary, *wn;  // [nimg][d+1][N]
    const float *norm;       // [nimg][N]
    const int32_t *rowbase;
    int shared;
    float alpha;
    float sigma[5], scale[5];
};
struct KgArgs {
    KgLat sp, bi;
    const uint8_t *image;  // [B][N][3]
    const float *potts;    // {w1, w2} on the device, or nullptr: w1, w2
    float w1, w2;
    float *part;           // [B][nblk][8] per-block sums of dL/dp in theta order
    float *csum;           // [2][B][N] c per pixel: spatial, bilateral
    int M, N, W, nblk;
};

// per-incidence s_r of one lattice -> the pixel's dL/dp over that lattice's features (added to dp), scaled by sign.
// FEAT: the features are the caller's (feat [B][D][N]), and the pixel's dL/df also goes to gfeat [B][D][N] (written
// when `first`, else added).
template <int D, bool FEAT = false>
__device__ __forceinline__ void kg_features(const KgLat &L, int x, int y, const uint8_t *image, int b, int N,
                                            int i, const float *s, float sign, float *dp, const float *feat = nullptr,
                                            float *gfeat = nullptr, bool first = false) {
    float f[D], el[D + 1], rem0[D + 1];
    int rank[D + 1];
    if constexpr (FEAT) {
#pragma unroll
        for (int j = 0; j < D; j++) f[j] = __ldg(feat + ((size_t)b * D + j) * N + i);
    } else {
        lattice_features<D>(x, y, image, b, N, i, L.sigma, f);
    }
    lattice_simplex<D>(f, L.scale, el, rem0, rank);
    const float c = sign * L.alpha / (float)(D + 1);
    float gel[D + 1];
#pragma unroll
    for (int j = 0; j <= D; j++) {
        const int r0 = D - rank[j], r1 = r0 == D ? 0 : r0 + 1;
        float a = 0.0f, b = 0.0f;
#pragma unroll
        for (int r = 0; r <= D; r++) {
            if (r == r0) a = s[r];
            if (r == r1) b = s[r];
        }
        gel[j] = c * (a - b);
    }
    float sm = gel[0];
#pragma unroll
    for (int j = 1; j <= D; j++) {
        const float df = L.scale[j - 1] * (sm - (float)j * gel[j]);   // dL/df_{j-1}
        dp[j - 1] = fmaf(f[j - 1], df, dp[j - 1]);
        if constexpr (FEAT) {
            float *o = gfeat + ((size_t)b * D + j - 1) * N + i;
            *o = first ? df : *o + df;
        }
        sm += gel[j];
    }
}

// the block's seven sums into part[b][block] (written when `first`, else added), in a fixed order
__device__ __forceinline__ void kg_block_sum(const KgArgs &a, int b, const float *dp, bool first) {
    __shared__ float red[kThreads / 32][7];
    float v[7];
#pragma unroll
    for (int k = 0; k < 7; k++) {
        v[k] = dp[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], o);
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 7; k++) red[threadIdx.x >> 5][k] = v[k];
    }
    __syncthreads();
    if (threadIdx.x < 7) {
        float acc = 0.0f;
        for (int w = 0; w < kThreads / 32; w++) acc += red[w][threadIdx.x];
        float *pp = a.part + ((size_t)b * a.nblk + blockIdx.x) * 8 + threadIdx.x;
        *pp = first ? acc : *pp + acc;
    }
}

// host side (meanfield.cu): a lattice's view for the passes, and the normalisation term and the per-image reductions
// after the loop (nothing in them has a label dimension)
KgLat kg_lat(const Lattice &L);
void kg_finish(Engine *e, const KgArgs &ka, int B, float *g_theta, int bgrid, cudaStream_t s, const float *feat,
               float *gfeat, int tag);

}  // namespace dsrg
