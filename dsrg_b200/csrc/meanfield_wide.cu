// Mean-field inference for label counts above DSRG_MAX_LABELS (32): the generic, label-chunked path.
//
// The reference's DenseCRF(W, H, nlabels) is generic in the label count (CRF/krahenbuhl2013/wrapper.pyx:23) and its
// COCO tool drives it with 81 labels (training/tools/test-coco.py).  The fused tile kernel keeps a pixel's whole
// label vector in registers, which stops at 32; beyond that the same arithmetic runs un-fused, one thread per
// (pixel, label quad): splat (pairwise.cpp:66, permutohedral.cpp:545-553), the per-axis blur (:556-569), slice +
// update (:574-584, pairwise.cpp:79, labelcompatibility.cpp:46-48) into the energies, and a soft-max over all
// labels (densecrf.cpp:98-106).  It moves every value through L2 and is several times slower per label than the
// fused path -- it exists so that the boundary has no hole, not for the 21-class hot path.
#include "common.cuh"

namespace dsrg {

// wn = bary * norm (the fused path gets it from the tile build)
__global__ void __launch_bounds__(kThreads)
k_wide_weights(const float *bary, const float *norm, float *wn, int N, int dp1) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const float nrm = norm[(size_t)b * N + i];
    for (int r = 0; r < dp1; r++) {
        const size_t at = ((size_t)b * dp1 + r) * N + i;
        wn[at] = __fmul_rn(bary[at], nrm);
    }
}

int wide_weights(Engine *e, Lattice &L, int nb, cudaStream_t s) {
    dim3 g(cdiv(L.N, kThreads), nb);
    DSRG_LAUNCH(e, T_LAT_MISC, s, k_wide_weights<<<g, kThreads, 0, s>>>(L.bary, L.norm, L.wn, L.N, L.d + 1));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

// unary (any layout) -> U planar (optionally clamped in place); Q = softmax(U)   (densecrf.cpp:120)
__global__ void __launch_bounds__(kThreads)
k_wide_init(const float *unary, float *unary_rw, int layout, int clamp, float *U, float *Q, int M, int N) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    float mx = -INFINITY;
    for (int k = 0; k < M; k++) {
        const size_t at = (layout == DSRG_LAYOUT_NCHW) ? ((size_t)b * M + k) * N + i : ((size_t)b * N + i) * M + k;
        float v = unary[at];
        if (clamp && v < kMinProb) {
            v = kMinProb;
            unary_rw[at] = v;
        }
        U[((size_t)b * M + k) * N + i] = v;
        mx = fmaxf(mx, v);
    }
    float sum = 0.0f;
    for (int k = 0; k < M; k++) {
        const size_t at = ((size_t)b * M + k) * N + i;
        const float ev = expf(U[at] - mx);
        Q[at] = ev;
        sum += ev;
    }
    for (int k = 0; k < M; k++) Q[((size_t)b * M + k) * N + i] /= sum;
}

struct WideLat {
    const int32_t *off;      // [nimg][dp1][N] local row (1-based)
    const float *wn;         // [nimg][dp1][N]
    const int32_t *rowbase;  // [B+1]
    float *val;              // [rows][MP]
    int shared, dp1;
};

__global__ void __launch_bounds__(kThreads)
k_wide_zero(float4 *a, const int32_t *rowbase_a, float4 *c, const int32_t *rowbase_c, int B, int CH) {
    const long long na = (long long)rowbase_a[B] * CH, nc = (long long)rowbase_c[B] * CH;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < na + nc; t += (long long)gridDim.x * blockDim.x) {
        if (t < na) a[t] = z; else c[t - na] = z;
    }
}

// one thread per (pixel, label quad): values[row_r] += wn_r * Q   for the d+1 vertices of both lattices
__global__ void __launch_bounds__(kThreads)
k_wide_splat(const float *Q, WideLat sp, WideLat bi, int M, int N, int CH) {
    const int b = blockIdx.z, c = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    float q[4];
#pragma unroll
    for (int k = 0; k < 4; k++) q[k] = (4 * c + k < M) ? Q[((size_t)b * M + 4 * c + k) * N + i] : 0.0f;
    for (int l = 0; l < 2; l++) {
        const WideLat &L = l ? bi : sp;
        const size_t px = (size_t)(L.shared ? 0 : b) * L.dp1 * N + i;
        const int base = L.rowbase[b];
        float4 *val = reinterpret_cast<float4 *>(L.val);
        for (int r = 0; r < L.dp1; r++) {
            const float w = L.wn[px + (size_t)r * N];
            const int row = base + L.off[px + (size_t)r * N];
            atomicAdd(val + (size_t)row * CH + c, make_float4(w * q[0], w * q[1], w * q[2], w * q[3]));
        }
    }
}

// one lattice axis, every image: thread per (row, label quad)
__global__ void __launch_bounds__(kThreads)
k_wide_blur(const float4 *in, float4 *out, const int2 *nbr, const int32_t *rowbase, int B, int shared, int CH) {
    const long long rows = rowbase[B];
    const int rows_img = shared ? rowbase[1] : 0;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < rows * CH; t += (long long)gridDim.x * blockDim.x) {
        const long long g = t / CH;
        const int c = (int)(t - g * CH);
        long long n1, n2;
        if (shared) {
            const long long img0 = (g / rows_img) * rows_img;
            const int2 n = nbr[g - img0];
            n1 = img0 + n.x;
            n2 = img0 + n.y;
        } else {
            const int2 n = nbr[g];
            n1 = n.x;
            n2 = n.y;
        }
        const float4 o = in[g * CH + c], a = in[n1 * CH + c], d = in[n2 * CH + c];
        out[g * CH + c] = make_float4(o.x + 0.5f * (a.x + d.x), o.y + 0.5f * (a.y + d.y), o.z + 0.5f * (a.z + d.z),
                                      o.w + 0.5f * (a.w + d.w));
    }
}

// t = U + c_sp * sum_r wn_r row_r (spatial) + c_bi * sum_r wn_r row_r (bilateral), written over Q
__global__ void __launch_bounds__(kThreads)
k_wide_slice(const float *U, float *T, WideLat sp, WideLat bi, float c_sp, float c_bi, int M, int N, int CH) {
    const int b = blockIdx.z, c = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    float t[4];
#pragma unroll
    for (int k = 0; k < 4; k++) t[k] = (4 * c + k < M) ? U[((size_t)b * M + 4 * c + k) * N + i] : 0.0f;
    for (int l = 0; l < 2; l++) {
        const WideLat &L = l ? bi : sp;
        const float coef = l ? c_bi : c_sp;
        const size_t px = (size_t)(L.shared ? 0 : b) * L.dp1 * N + i;
        const int base = L.rowbase[b];
        const float4 *val = reinterpret_cast<const float4 *>(L.val);
        for (int r = 0; r < L.dp1; r++) {
            const float wr = coef * L.wn[px + (size_t)r * N];
            const float4 v = val[(size_t)(base + L.off[px + (size_t)r * N]) * CH + c];
            t[0] = fmaf(wr, v.x, t[0]);
            t[1] = fmaf(wr, v.y, t[1]);
            t[2] = fmaf(wr, v.z, t[2]);
            t[3] = fmaf(wr, v.w, t[3]);
        }
    }
#pragma unroll
    for (int k = 0; k < 4; k++)
        if (4 * c + k < M) T[((size_t)b * M + 4 * c + k) * N + i] = t[k];
}

// Q = softmax(T) in place (expAndNormalize, densecrf.cpp:98-106)
__global__ void __launch_bounds__(kThreads)
k_wide_softmax(float *T, int M, int N) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    float *p = T + (size_t)b * M * N + i;
    float mx = -INFINITY;
    for (int k = 0; k < M; k++) mx = fmaxf(mx, p[(size_t)k * N]);
    float sum = 0.0f;
    for (int k = 0; k < M; k++) {
        const float ev = expf(p[(size_t)k * N] - mx);
        p[(size_t)k * N] = ev;
        sum += ev;
    }
    for (int k = 0; k < M; k++) p[(size_t)k * N] /= sum;
}

int meanfield_run_wide(Engine *e, int B, const float *unary, int layout, bool clamp, float *unary_rw,
                       const dsrg_crf_params &p, cudaStream_t s) {
    const int M = e->M, N = e->N, CH = e->MP / 4, T = p.n_iters;
    dim3 gp(cdiv(N, kThreads), B), gq(cdiv(N, kThreads), CH, B);
    DSRG_LAUNCH(e, T_MF_INIT, s, k_wide_init<<<gp, kThreads, 0, s>>>(unary, unary_rw, layout, clamp ? 1 : 0, e->U, e->Q0, M, N));
    if (T == 0) return DSRG_OK;
    const float alpha_sp = 1.0f / (1 + powf(2, -e->sp.d)), alpha_bi = 1.0f / (1 + powf(2, -e->bi.d));  // permutohedral.cpp:571
    const float c_sp = p.w2 * alpha_sp, c_bi = p.w1 * alpha_bi;
    const int grid = 8 * e->sm_count;
    float *spY = e->spA, *spZ = e->spB, *biY = e->biA, *biZ = e->biB;
    for (int it = 0; it < T; it++) {
        DSRG_LAUNCH(e, T_MF_ZERO, s, k_wide_zero<<<grid, kThreads, 0, s>>>((float4 *)spY, e->sp.rowbase, (float4 *)biY, e->bi.rowbase, B, CH));
        WideLat sp{e->sp.off, e->sp.wn, e->sp.rowbase, spY, e->sp.shared, e->sp.d + 1};
        WideLat bi{e->bi.off, e->bi.wn, e->bi.rowbase, biY, e->bi.shared, e->bi.d + 1};
        DSRG_LAUNCH(e, T_MF_TILE, s, k_wide_splat<<<gq, kThreads, 0, s>>>(e->Q0, sp, bi, M, N, CH));
        for (int l = 0; l < 2; l++) {
            Lattice &L = l ? e->bi : e->sp;
            float *&src = l ? biY : spY, *&dst = l ? biZ : spZ;
            for (int j = 0; j <= L.d; j++) {
                DSRG_LAUNCH(e, T_MF_BLUR_BI, s,
                            k_wide_blur<<<grid, kThreads, 0, s>>>((const float4 *)src, (float4 *)dst, L.nbr + (size_t)j * L.nbr_stride,
                                                                  L.rowbase, B, L.shared, CH));
                float *t = src; src = dst; dst = t;
            }
        }
        sp.val = spY;
        bi.val = biY;
        DSRG_LAUNCH(e, T_MF_TILE, s, k_wide_slice<<<gq, kThreads, 0, s>>>(e->U, e->Q0, sp, bi, c_sp, c_bi, M, N, CH));
        DSRG_LAUNCH(e, T_MF_TILE, s, k_wide_softmax<<<gp, kThreads, 0, s>>>(e->Q0, M, N));
    }
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

}  // namespace dsrg
