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
#include "kgrad.cuh"

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

// ---------------------------------------------------------------------------------------------
// Training above 32 labels: the forward keeping Q_0..Q_T, and the backward of the mean field (DenseCRF::gradient,
// densecrf.cpp:238-297) on the label-chunked kernels.  With F(X) = alpha n K(n X) (wn = bary * norm, alpha on the
// slice):
//   Potts forward : t = U + w2 F_sp(Q) + w1 F_bi(Q)
//   matrix forward: t = U - mu_sp F_sp(Q) - mu_bi F_bi(Q)      (compat = {mu_bi, mu_sp} [2][M][M])
//   backward, t = T..0: g_t = Q_t (G_t - <G_t, Q_t>), grad_U += g_t, G_T = dL/dQ_T; for t > 0 splat wn g_t, blur
//   the axes d..0 (K^T: every single-axis blur is symmetric), slice S_k = F_k^T(g_t) and form
//     Potts : G_{t-1} = w2 S_sp + w1 S_bi,            dL/dw_k  += <S_k, Q_{t-1}>
//     matrix: G_{t-1} = -(mu_sp^T S_sp + mu_bi^T S_bi), dL/dmu_k += -sum_i S_k,i (x) Q_{t-1},i
// The parameter sums are kept per block (Potts) or per (image, pixel chunk) (matrices) and reduced in a fixed order:
// no float atomics outside the splat.  The slices and mat-vecs run in meanfield.cu's operation order (fma chains
// from zero with weights alpha wn, the spatial lattice first, labels ascending).
// ---------------------------------------------------------------------------------------------

// the quad c of pixel i: t += coef * wn_r * row_r over the d+1 vertices of L
__device__ __forceinline__ void wide_slice_quad(const WideLat &L, float coef, int b, int i, int c, int N, int CH,
                                                float t[4]) {
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

// k_wide_slice with the Potts weights read on the device (potts = {w1, w2})
__global__ void __launch_bounds__(kThreads)
k_wide_slice_dev(const float *U, float *T, WideLat sp, WideLat bi, const float *potts, float a_sp, float a_bi, int M,
                 int N, int CH) {
    const int b = blockIdx.z, c = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const float c_sp = __ldg(potts + 1) * a_sp, c_bi = __ldg(potts) * a_bi;
    float t[4];
#pragma unroll
    for (int k = 0; k < 4; k++) t[k] = (4 * c + k < M) ? U[((size_t)b * M + 4 * c + k) * N + i] : 0.0f;
    wide_slice_quad(sp, c_sp, b, i, c, N, CH, t);
    wide_slice_quad(bi, c_bi, b, i, c, N, CH, t);
#pragma unroll
    for (int k = 0; k < 4; k++)
        if (4 * c + k < M) T[((size_t)b * M + 4 * c + k) * N + i] = t[k];
}

// S_sp = F_sp(.), S_bi = F_bi(.) of the blurred values, each sliced from zero, planar [B][M][N]
__global__ void __launch_bounds__(kThreads)
k_wide_slice_planar(float *S_sp, float *S_bi, WideLat sp, WideLat bi, float a_sp, float a_bi, int M, int N, int CH) {
    const int b = blockIdx.z, c = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    float t[4] = {0.0f, 0.0f, 0.0f, 0.0f}, u[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    wide_slice_quad(sp, a_sp, b, i, c, N, CH, t);
    wide_slice_quad(bi, a_bi, b, i, c, N, CH, u);
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (4 * c + k < M) {
            S_sp[((size_t)b * M + 4 * c + k) * N + i] = t[k];
            S_bi[((size_t)b * M + 4 * c + k) * N + i] = u[k];
        }
    }
}

// out[l] = U[l] - sum_l' mu_sp[l, l'] S_sp[l'] - sum_l' mu_bi[l, l'] S_bi[l']  (U == nullptr: from zero), or with
// mu^T (TRANSPOSE: the backward's G).  One thread per (pixel, label quad); the block's quad needs four rows (columns)
// of each matrix, 8 M floats in shared memory (both whole matrices would not fit above 80 labels).
template <bool TRANSPOSE>
__global__ void __launch_bounds__(kThreads)
k_wide_compat_msg(const float *U, const float *S_sp, const float *S_bi, const float *compat, float *out, int M, int N) {
    extern __shared__ float mus[];   // [2 = sp, bi][4][M]
    const int b = blockIdx.z, c = blockIdx.y;
    for (int e = threadIdx.x; e < 8 * M; e += blockDim.x) {
        const int m = e / (4 * M), k = (e / M) & 3, l2 = e % M, l = 4 * c + k;
        const float *mu = compat + (m ? 0 : (size_t)M * M);   // compat = {mu_bi, mu_sp}
        mus[e] = l < M ? (TRANSPOSE ? mu[(size_t)l2 * M + l] : mu[(size_t)l * M + l2]) : 0.0f;
    }
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    float t[4];
#pragma unroll
    for (int k = 0; k < 4; k++) t[k] = (U && 4 * c + k < M) ? U[((size_t)b * M + 4 * c + k) * N + i] : 0.0f;
#pragma unroll
    for (int m = 0; m < 2; m++) {
        const float *S = (m ? S_bi : S_sp) + (size_t)b * M * N + i;
        const float *mu = mus + m * 4 * M;
        for (int l2 = 0; l2 < M; l2++) {
            const float s = S[(size_t)l2 * N];
#pragma unroll
            for (int k = 0; k < 4; k++) t[k] = fmaf(-mu[k * M + l2], s, t[k]);
        }
    }
#pragma unroll
    for (int k = 0; k < 4; k++)
        if (4 * c + k < M) out[((size_t)b * M + 4 * c + k) * N + i] = t[k];
}

// g = Q (G - <G, Q>) per pixel over all labels; gU = g (first) or gU += g; g also to gout when given (gout may be G)
__global__ void __launch_bounds__(kThreads)
k_wide_vjp(const float *G, const float *Q, float *gU, float *gout, int first, int M, int N) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const size_t at = (size_t)b * M * N + i;
    float dot = 0.0f;
    for (int k = 0; k < M; k++) dot = fmaf(G[at + (size_t)k * N], Q[at + (size_t)k * N], dot);
    for (int k = 0; k < M; k++) {
        const size_t a = at + (size_t)k * N;
        const float g = Q[a] * (G[a] - dot);
        gU[a] = first ? g : gU[a] + g;
        if (gout) gout[a] = g;
    }
}

// Potts: G = w2 S_sp + w1 S_bi per (pixel, label quad) with the block's {<S_sp, Q>, <S_bi, Q>} to
// part[b][c][block] (first: written, else added)
__global__ void __launch_bounds__(kThreads)
k_wide_potts_bwd(const float *Qt, float *G, WideLat sp, WideLat bi, const float *potts, float w1, float w2,
                 float a_sp, float a_bi, float2 *part, int first, int M, int N, int CH) {
    __shared__ float2 red[kThreads / 32];
    const int b = blockIdx.z, c = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (potts) {
        w1 = __ldg(potts);
        w2 = __ldg(potts + 1);
    }
    float p_sp = 0.0f, p_bi = 0.0f;
    if (i < N) {
        float q[4], s[4] = {0.0f, 0.0f, 0.0f, 0.0f}, g[4];
#pragma unroll
        for (int k = 0; k < 4; k++) q[k] = (4 * c + k < M) ? Qt[((size_t)b * M + 4 * c + k) * N + i] : 0.0f;
        wide_slice_quad(sp, a_sp, b, i, c, N, CH, s);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            p_sp = fmaf(s[k], q[k], p_sp);
            g[k] = w2 * s[k];
            s[k] = 0.0f;
        }
        wide_slice_quad(bi, a_bi, b, i, c, N, CH, s);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            p_bi = fmaf(s[k], q[k], p_bi);
            g[k] = fmaf(w1, s[k], g[k]);
            if (4 * c + k < M) G[((size_t)b * M + 4 * c + k) * N + i] = g[k];
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        p_sp += __shfl_down_sync(0xffffffffu, p_sp, o);
        p_bi += __shfl_down_sync(0xffffffffu, p_bi, o);
    }
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = make_float2(p_sp, p_bi);
    __syncthreads();
    if (threadIdx.x == 0) {
        float2 a = make_float2(0.0f, 0.0f);
#pragma unroll
        for (int w = 0; w < kThreads / 32; w++) {
            a.x += red[w].x;
            a.y += red[w].y;
        }
        float2 *pp = part + ((size_t)b * CH + c) * gridDim.x + blockIdx.x;
        if (!first) {
            a.x += pp->x;
            a.y += pp->y;
        }
        *pp = a;
    }
}

// The matrices' outer products, an FP32 tiled GEMM per image: part[b][chunk][k][l][l'] (+)= sum over the chunk's
// pixels of S_k[l] Q[l'] (k = 0: bilateral, 1: spatial).  A CTA owns a 32 x 32 block of (l, l') over one pixel chunk
// and stages 32-pixel slabs of S and Q; each thread owns 2 x 2 entries and sums a slab, then adds the slab to its
// total, so a sum's depth stays near 32 + N / (32 kWideChunks) rather than N / kWideChunks.
constexpr int kWideOuterTile = 32;
__global__ void __launch_bounds__(kThreads)
k_wide_outer(const float *S_sp, const float *S_bi, const float *Qt, float *part, int first, int M, int N,
             int chunk_px) {
    constexpr int TL = kWideOuterTile;
    __shared__ float ss[TL][TL + 1], qs[TL][TL + 1];   // [pixel][label]
    const int tl = (M + TL - 1) / TL;
    const int l0 = (blockIdx.x / tl) * TL, m0 = (blockIdx.x % tl) * TL;
    const int k = blockIdx.y / kWideChunks, chunk = blockIdx.y % kWideChunks, b = blockIdx.z;
    const float *S = (k ? S_sp : S_bi) + (size_t)b * M * N, *Q = Qt + (size_t)b * M * N;
    const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
    const int p_beg = chunk * chunk_px, p_end = min(N, p_beg + chunk_px);
    float acc[2][2] = {{0.0f, 0.0f}, {0.0f, 0.0f}};
    for (int p0 = p_beg; p0 < p_end; p0 += TL) {
        __syncthreads();
        for (int e = tid; e < TL * TL; e += kThreads) {
            const int r = e / TL, px = e % TL, p = p0 + px;
            const bool pin = p < p_end;
            ss[px][r] = (pin && l0 + r < M) ? S[(size_t)(l0 + r) * N + p] : 0.0f;
            qs[px][r] = (pin && m0 + r < M) ? Q[(size_t)(m0 + r) * N + p] : 0.0f;
        }
        __syncthreads();
        float sl[2][2] = {{0.0f, 0.0f}, {0.0f, 0.0f}};
#pragma unroll 8
        for (int px = 0; px < TL; px++) {
            const float a0 = ss[px][2 * ty], a1 = ss[px][2 * ty + 1], q0 = qs[px][2 * tx], q1 = qs[px][2 * tx + 1];
            sl[0][0] = fmaf(a0, q0, sl[0][0]);
            sl[0][1] = fmaf(a0, q1, sl[0][1]);
            sl[1][0] = fmaf(a1, q0, sl[1][0]);
            sl[1][1] = fmaf(a1, q1, sl[1][1]);
        }
#pragma unroll
        for (int u = 0; u < 2; u++)
#pragma unroll
            for (int v = 0; v < 2; v++) acc[u][v] += sl[u][v];
    }
    float *pp = part + (((size_t)b * kWideChunks + chunk) * 2 + k) * M * M;
#pragma unroll
    for (int u = 0; u < 2; u++)
#pragma unroll
        for (int v = 0; v < 2; v++) {
            const int l = l0 + 2 * ty + u, l2 = m0 + 2 * tx + v;
            if (l < M && l2 < M) {
                float *o = pp + (size_t)l * M + l2;
                *o = first ? acc[u][v] : *o + acc[u][v];
            }
        }
}

// ---------------------------------------------------------------------------------------------
// The kernel-bandwidth and feature gradient above 32 labels: the math of the fused path (kgrad.cuh, the comment above
// KgLat in meanfield.cu) with the label dimension chunked into quads.  Iteration it (T down to 1) pairs g_it with
// Q_{it-1}, as kg_iter pairs g_{t+1} with Q_t: Vg = B^T S(n g_it) is the reverse-blurred buffer the backward slices,
// Vy = B S(n Q_{it-1}) a forward splat and blur into the buffers Vg leaves free, and per lattice
//   Potts : x = g_it, u = Q_{it-1}, and the lattice's weight w
//   matrix: x = -mu^T g_it, u = -mu Q_{it-1} (k_wide_compat_xu), w = 1
// k_wide_kg_pass forms s_r at every incidence and the pixel's c, then kg_features rotates s into dL/dp (and for
// caller-given features dL/df).  The normalisation term and the per-image sums after the loop are kg_finish's.
// ---------------------------------------------------------------------------------------------

// x = -mu^T g and u = -mu Q for one matrix mu ([M][M]), planar [B][M][N], one thread per (pixel, label quad); the
// block's quad needs four columns and four rows of mu, 8 M floats in shared memory (as k_wide_compat_msg)
__global__ void __launch_bounds__(kThreads)
k_wide_compat_xu(const float *g, const float *Q, const float *mu, float *x, float *u, int M, int N) {
    extern __shared__ float mus[];   // [2 = mu^T, mu][4][M]
    const int b = blockIdx.z, c = blockIdx.y;
    for (int e = threadIdx.x; e < 8 * M; e += blockDim.x) {
        const int m = e / (4 * M), k = (e / M) & 3, l2 = e % M, l = 4 * c + k;
        mus[e] = l < M ? (m ? mu[(size_t)l * M + l2] : mu[(size_t)l2 * M + l]) : 0.0f;
    }
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const float *gp = g + (size_t)b * M * N + i, *qp = Q + (size_t)b * M * N + i;
    float xa[4] = {0.0f, 0.0f, 0.0f, 0.0f}, ua[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    for (int l2 = 0; l2 < M; l2++) {
        const float gv = gp[(size_t)l2 * N], qv = qp[(size_t)l2 * N];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            xa[k] = fmaf(-mus[k * M + l2], gv, xa[k]);
            ua[k] = fmaf(-mus[(4 + k) * M + l2], qv, ua[k]);
        }
    }
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (4 * c + k < M) {
            x[((size_t)b * M + 4 * c + k) * N + i] = xa[k];
            u[((size_t)b * M + 4 * c + k) * N + i] = ua[k];
        }
    }
}

// s_r = n w sum over the label quads, ascending, of x . Vy[r] + u . Vg[r] at the D + 1 incidences of one lattice;
// returns c = 1/2 n^2 alpha sum_r bary_r s_r (kg_incidences with the labels chunked)
template <int D>
__device__ __forceinline__ float wide_kg_incidences(const KgLat &L, int b, int i, int M, int N, int CH, const float *x,
                                                    const float *u, float w, const float4 *vy, const float4 *vg,
                                                    float *s) {
    const size_t at = (size_t)(L.shared ? 0 : b) * (D + 1) * N + i;
    const int base = L.rowbase[b];
    const float n = __ldg(L.norm + (size_t)(L.shared ? 0 : b) * N + i);
    size_t row[D + 1];
    float acc[D + 1];
#pragma unroll
    for (int r = 0; r <= D; r++) {
        row[r] = (size_t)(base + __ldg(L.off + at + (size_t)r * N)) * CH;
        acc[r] = 0.0f;
    }
    const float *xp = x + (size_t)b * M * N + i, *up = u + (size_t)b * M * N + i;
    for (int c = 0; c < CH; c++) {
        float xv[4], uv[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int l = 4 * c + k;
            xv[k] = l < M ? __ldg(xp + (size_t)l * N) : 0.0f;
            uv[k] = l < M ? __ldg(up + (size_t)l * N) : 0.0f;
        }
#pragma unroll
        for (int r = 0; r <= D; r++) {
            const float4 a = vy[row[r] + c], g = vg[row[r] + c];
            float t = acc[r];
            t = fmaf(xv[0], a.x, t);
            t = fmaf(xv[1], a.y, t);
            t = fmaf(xv[2], a.z, t);
            t = fmaf(xv[3], a.w, t);
            t = fmaf(uv[0], g.x, t);
            t = fmaf(uv[1], g.y, t);
            t = fmaf(uv[2], g.z, t);
            t = fmaf(uv[3], g.w, t);
            acc[r] = t;
        }
    }
    float cs = 0.0f;
#pragma unroll
    for (int r = 0; r <= D; r++) {
        s[r] = n * w * acc[r];
        cs = fmaf(__ldg(L.bary + at + (size_t)r * N), s[r], cs);
    }
    return 0.5f * n * n * L.alpha * cs;
}

// One thread per pixel, for each lattice whose x is given (the Potts pass runs both, the matrices one per launch):
// s_r and c (added to csum), the rotation to dL/dp (FEAT: the bilateral features are feat's and the pixel's dL/df goes
// to gfeat), then the block's sums to part.  `first`: csum and gfeat of the given lattices are written, not added;
// `part_first`: the same for part.  The weights are a.potts ({w1, w2}, device) or a.w1 / a.w2 (1 for the matrices).
template <bool FEAT>
__global__ void __launch_bounds__(kThreads)
k_wide_kg_pass(KgArgs a, const float *x_sp, const float *u_sp, const float *x_bi, const float *u_bi,
               const float4 *vy_sp, const float4 *vg_sp, const float4 *vy_bi, const float4 *vg_bi, int CH, int first,
               int part_first, const float *feat, float *gfeat) {
    const int b = blockIdx.y, i = blockIdx.x * kThreads + threadIdx.x;
    float dp[7];
#pragma unroll
    for (int k = 0; k < 7; k++) dp[k] = 0.0f;
    if (i < a.N) {
        const int x = i % a.W, y = i / a.W;
        float s[6];
        float *csum_sp = a.csum + (size_t)b * a.N + i, *csum_bi = csum_sp + (size_t)gridDim.y * a.N;
        if (x_sp) {
            const float w = a.potts ? __ldg(a.potts + 1) : a.w2;
            const float c = wide_kg_incidences<2>(a.sp, b, i, a.M, a.N, CH, x_sp, u_sp, w, vy_sp, vg_sp, s);
            kg_features<2>(a.sp, x, y, a.image, b, a.N, i, s, 1.0f, dp + 5);
            *csum_sp = first ? c : *csum_sp + c;
        }
        if (x_bi) {
            const float w = a.potts ? __ldg(a.potts) : a.w1;
            const float c = wide_kg_incidences<5>(a.bi, b, i, a.M, a.N, CH, x_bi, u_bi, w, vy_bi, vg_bi, s);
            kg_features<5, FEAT>(a.bi, x, y, a.image, b, a.N, i, s, 1.0f, dp, feat, gfeat, first != 0);
            *csum_bi = first ? c : *csum_bi + c;
        }
    }
    kg_block_sum(a, b, dp, part_first != 0);
}

// With `compat` the messages are the matrices' (the training forward's slice_planar + compat_msg, below): S_sp, S_bi
// to two [B][M][N] planes, then t = U - mu_sp S_sp - mu_bi S_bi over Q, whose values the splat has consumed by then.
// The planes live in e->biC, which this loop never touches (it ping-pongs spA / spB and biA / biB) and which holds
// maxB * (6 (Ncap + P) + 1) * MP >= 2 * B * M * N floats: the matrices cost no memory beyond the Potts inference.
int meanfield_run_wide(Engine *e, int B, const float *unary, int layout, bool clamp, float *unary_rw,
                       const dsrg_crf_params &p, cudaStream_t s, const float *compat) {
    const int M = e->M, N = e->N, CH = e->MP / 4, T = p.n_iters;
    float *s_sp = e->biC, *s_bi = e->biC + (size_t)B * M * N;
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
        if (compat) {
            DSRG_LAUNCH(e, T_MF_TILE, s,
                        k_wide_slice_planar<<<gq, kThreads, 0, s>>>(s_sp, s_bi, sp, bi, alpha_sp, alpha_bi, M, N, CH));
            DSRG_LAUNCH(e, T_MF_TILE, s,
                        k_wide_compat_msg<false><<<gq, kThreads, 8 * M * sizeof(float), s>>>(e->U, s_sp, s_bi, compat,
                                                                                            e->Q0, M, N));
        } else {
            DSRG_LAUNCH(e, T_MF_TILE, s, k_wide_slice<<<gq, kThreads, 0, s>>>(e->U, e->Q0, sp, bi, c_sp, c_bi, M, N, CH));
        }
        DSRG_LAUNCH(e, T_MF_TILE, s, k_wide_softmax<<<gp, kThreads, 0, s>>>(e->Q0, M, N));
    }
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

static WideLat wide_lat(const Lattice &L, float *val) { return WideLat{L.off, L.wn, L.rowbase, val, L.shared, L.d + 1}; }

// blur every axis of L (d..0 when `reverse`, K^T) ping-ponging between *src and *dst; afterwards *src holds the
// result and *dst is free
static void wide_blur_axes(Engine *e, const Lattice &L, int B, bool reverse, int tag, cudaStream_t s, float **src,
                           float **dst) {
    const int CH = e->MP / 4, grid = 8 * e->sm_count;
    for (int p = 0; p <= L.d; p++) {
        const int j = reverse ? L.d - p : p;
        DSRG_LAUNCH(e, tag, s,
                    k_wide_blur<<<grid, kThreads, 0, s>>>((const float4 *)*src, (float4 *)*dst, L.nbr + (size_t)j * L.nbr_stride,
                                                          L.rowbase, B, L.shared, CH));
        float *t = *src; *src = *dst; *dst = t;
    }
}

// zero Y, splat X planar into it, blur every axis (d..0 when `reverse`, K^T) ping-ponging with Z; returns the
// blurred buffers
static void wide_filter_to(Engine *e, int B, const float *X, bool reverse, int tag, cudaStream_t s, float *spY,
                           float *spZ, float *biY, float *biZ, float **sp_out, float **bi_out) {
    const int M = e->M, N = e->N, CH = e->MP / 4, grid = 8 * e->sm_count;
    const dim3 gq(cdiv(N, kThreads), CH, B);
    DSRG_LAUNCH(e, tag, s, k_wide_zero<<<grid, kThreads, 0, s>>>((float4 *)spY, e->sp.rowbase, (float4 *)biY, e->bi.rowbase, B, CH));
    DSRG_LAUNCH(e, tag, s, k_wide_splat<<<gq, kThreads, 0, s>>>(X, wide_lat(e->sp, spY), wide_lat(e->bi, biY), M, N, CH));
    wide_blur_axes(e, e->sp, B, reverse, tag, s, &spY, &spZ);
    wide_blur_axes(e, e->bi, B, reverse, tag, s, &biY, &biZ);
    *sp_out = spY;
    *bi_out = biY;
}

// wide_filter_to on the mean-field buffers spA / spB and biA / biB
static void wide_filter(Engine *e, int B, const float *X, bool reverse, int tag, cudaStream_t s, float **sp_out,
                        float **bi_out) {
    wide_filter_to(e, B, X, reverse, tag, s, e->spA, e->spB, e->biA, e->biB, sp_out, bi_out);
}

static float wide_alpha(const Lattice &L) { return 1.0f / (1 + powf(2, -L.d)); }   // permutohedral.cpp:571

int meanfield_run_train_wide(Engine *e, int B, const CrfTrainIo &io, const dsrg_crf_params &p, cudaStream_t s) {
    const int M = e->M, N = e->N, CH = e->MP / 4, T = p.n_iters;
    const float *unary = io.unary, *potts = io.potts, *compat = io.compat;
    float *q_hist = io.q_out;
    const size_t slab = (size_t)B * M * N;
    const dim3 gp(cdiv(N, kThreads), B), gq(cdiv(N, kThreads), CH, B);
    const float a_sp = wide_alpha(e->sp), a_bi = wide_alpha(e->bi);
    DSRG_LAUNCH(e, T_WIDE_GRAD, s, k_wide_init<<<gp, kThreads, 0, s>>>(unary, nullptr, DSRG_LAYOUT_NCHW, 0, e->U, q_hist, M, N));
    for (int it = 1; it <= T; it++) {
        float *spV, *biV, *qt = q_hist + (size_t)it * slab;
        wide_filter(e, B, q_hist + (size_t)(it - 1) * slab, false, T_WIDE_GRAD, s, &spV, &biV);
        const WideLat sp = wide_lat(e->sp, spV), bi = wide_lat(e->bi, biV);
        if (compat) {   // e->U and e->Q0 hold S_sp and S_bi
            DSRG_LAUNCH(e, T_WIDE_GRAD, s, k_wide_slice_planar<<<gq, kThreads, 0, s>>>(e->U, e->Q0, sp, bi, a_sp, a_bi, M, N, CH));
            DSRG_LAUNCH(e, T_WIDE_GRAD, s,
                        k_wide_compat_msg<false><<<gq, kThreads, 8 * M * sizeof(float), s>>>(unary, e->U, e->Q0, compat, qt, M, N));
        } else if (potts) {
            DSRG_LAUNCH(e, T_WIDE_GRAD, s, k_wide_slice_dev<<<gq, kThreads, 0, s>>>(unary, qt, sp, bi, potts, a_sp, a_bi, M, N, CH));
        } else {
            DSRG_LAUNCH(e, T_WIDE_GRAD, s,
                        k_wide_slice<<<gq, kThreads, 0, s>>>(unary, qt, sp, bi, p.w2 * a_sp, p.w1 * a_bi, M, N, CH));
        }
        DSRG_LAUNCH(e, T_WIDE_GRAD, s, k_wide_softmax<<<gp, kThreads, 0, s>>>(qt, M, N));
    }
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int meanfield_backward_wide(Engine *e, int B, const CrfTrainIo &io, const dsrg_crf_params &p, cudaStream_t s) {
    const int M = e->M, N = e->N, CH = e->MP / 4, T = p.n_iters;
    const float *q_hist = io.q_hist, *potts = io.potts, *compat = io.compat, *feat = io.features;
    float *grad_feat = io.grad_features;
    const size_t slab = (size_t)B * M * N;
    const int nblk = cdiv(N, kThreads);
    const dim3 gp(nblk, B), gq(nblk, CH, B);
    const float a_sp = wide_alpha(e->sp), a_bi = wide_alpha(e->bi);
    // the kernel-bandwidth gradient (grad_theta), or the feature gradient (grad_feat) with the spatial sums to
    // grad_theta_sp: per iteration Vy into the buffers Vg leaves free and k_wide_kg_pass, kg_finish after the loop
    float *grad_theta = grad_feat ? io.grad_theta_sp : io.grad_theta;
    const bool kg = grad_theta || grad_feat;
    const int kg_tag = grad_feat ? T_FGRAD : T_KGRAD;
    KgArgs ka{};
    if (kg) {
        ka.sp = kg_lat(e->sp);
        ka.bi = kg_lat(e->bi);
        ka.image = io.image;
        ka.potts = compat ? nullptr : potts;
        ka.w1 = compat ? 1.0f : p.w1;   // the matrices' x and u carry mu
        ka.w2 = compat ? 1.0f : p.w2;
        ka.part = e->kg_part;
        ka.csum = e->kg_csum;
        ka.M = M;
        ka.N = N;
        ka.W = e->W;
        ka.nblk = nblk;
    }
    // e->Q0: g_t, then S_sp (matrices) or G_{t-1} (Potts); e->U: S_bi; e->wide_g: the matrices' G_{t-1}.  With kg and
    // matrices, e->U and e->wide_g hold x and u of one lattice before the slice (G_t was read by the VJP by then).
    float *X = e->Q0;
    const float *G = io.grad_q;
    const int tl = (M + kWideOuterTile - 1) / kWideOuterTile;
    const int chunk_px = cdiv(cdiv(N, kWideChunks), kWideOuterTile) * kWideOuterTile;
    for (int it = T; it > 0; it--) {
        const float *qt = q_hist + (size_t)it * slab, *qp = q_hist + (size_t)(it - 1) * slab;
        const int first = it == T;
        DSRG_LAUNCH(e, T_WIDE_GRAD, s, k_wide_vjp<<<gp, kThreads, 0, s>>>(G, qt, io.grad_unary, X, first, M, N));
        float *spV, *biV;
        wide_filter(e, B, X, true, T_WIDE_GRAD, s, &spV, &biV);
        if (kg) {
            // Vy = B S(n Q_{it-1}) in the mean-field buffer Vg does not hold and spC / biC
            float *vy_sp, *vy_bi;
            wide_filter_to(e, B, qp, false, kg_tag, s, spV == e->spA ? e->spB : e->spA, e->spC,
                           biV == e->biA ? e->biB : e->biA, e->biC, &vy_sp, &vy_bi);
            const float4 *ysp = (const float4 *)vy_sp, *ybi = (const float4 *)vy_bi;
            const float4 *gsp = (const float4 *)spV, *gbi = (const float4 *)biV;
#define DSRG_KG_PASS(XS, US, XB, UB, PF)                                                                              \
    do {                                                                                                              \
        if (feat)                                                                                                     \
            DSRG_LAUNCH(e, kg_tag, s,                                                                                 \
                        k_wide_kg_pass<true><<<gp, kThreads, 0, s>>>(ka, XS, US, XB, UB, ysp, gsp, ybi, gbi, CH,      \
                                                                     first, PF, feat, grad_feat));                    \
        else                                                                                                          \
            DSRG_LAUNCH(e, kg_tag, s,                                                                                 \
                        k_wide_kg_pass<false><<<gp, kThreads, 0, s>>>(ka, XS, US, XB, UB, ysp, gsp, ybi, gbi, CH,     \
                                                                      first, PF, nullptr, nullptr));                  \
    } while (0)
            if (compat) {   // one lattice per launch: x, u of the spatial matrix, then of the bilateral one
                const size_t smem = 8 * M * sizeof(float);
                DSRG_LAUNCH(e, kg_tag, s,
                            k_wide_compat_xu<<<gq, kThreads, smem, s>>>(X, qp, compat + (size_t)M * M, e->U, e->wide_g, M, N));
                DSRG_KG_PASS(e->U, e->wide_g, nullptr, nullptr, first);
                DSRG_LAUNCH(e, kg_tag, s, k_wide_compat_xu<<<gq, kThreads, smem, s>>>(X, qp, compat, e->U, e->wide_g, M, N));
                DSRG_KG_PASS(nullptr, nullptr, e->U, e->wide_g, 0);
            } else {
                DSRG_KG_PASS(X, qp, X, qp, first);
            }
#undef DSRG_KG_PASS
        }
        const WideLat sp = wide_lat(e->sp, spV), bi = wide_lat(e->bi, biV);
        if (compat) {
            DSRG_LAUNCH(e, T_WIDE_GRAD, s, k_wide_slice_planar<<<gq, kThreads, 0, s>>>(X, e->U, sp, bi, a_sp, a_bi, M, N, CH));
            DSRG_LAUNCH(e, T_WIDE_GRAD, s,
                        k_wide_compat_msg<true><<<gq, kThreads, 8 * M * sizeof(float), s>>>(nullptr, X, e->U, compat, e->wide_g, M, N));
            if (io.grad_compat)
                DSRG_LAUNCH(e, T_WIDE_GRAD, s,
                            k_wide_outer<<<dim3(tl * tl, 2 * kWideChunks, B), kThreads, 0, s>>>(X, e->U, qp, e->wide_cpart,
                                                                                               first, M, N, chunk_px));
            G = e->wide_g;
        } else {
            DSRG_LAUNCH(e, T_WIDE_GRAD, s,
                        k_wide_potts_bwd<<<gq, kThreads, 0, s>>>(qp, X, sp, bi, potts, p.w1, p.w2, a_sp, a_bi, e->wide_ppart,
                                                                 first, M, N, CH));
            G = X;
        }
    }
    DSRG_LAUNCH(e, T_WIDE_GRAD, s, k_wide_vjp<<<gp, kThreads, 0, s>>>(G, q_hist, io.grad_unary, nullptr, T == 0, M, N));
    if (T == 0) {
        if (io.grad_potts) DSRG_CUDA_TRY(cudaMemsetAsync(io.grad_potts, 0, sizeof(float) * 2 * B, s));
        if (io.grad_compat) DSRG_CUDA_TRY(cudaMemsetAsync(io.grad_compat, 0, sizeof(float) * 2 * M * M * B, s));
        if (grad_feat) DSRG_CUDA_TRY(cudaMemsetAsync(grad_feat, 0, sizeof(float) * 5 * N * B, s));
        if (grad_theta) DSRG_CUDA_TRY(cudaMemsetAsync(grad_theta, 0, sizeof(float) * (grad_feat ? 2 : 7) * B, s));
    } else {
        if (io.grad_potts) {
            potts_reduce(e, e->wide_ppart, io.grad_potts, CH * nblk, B, T_WIDE_GRAD, s);
        } else if (io.grad_compat) {
            compat_reduce(e, e->wide_cpart, io.grad_compat, kWideChunks, 2 * M * M, B, T_WIDE_GRAD, s);
        }
        if (kg) kg_finish(e, ka, B, grad_theta, 8 * e->sm_count, s, feat, grad_feat, kg_tag);
    }
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

// ---------------------------------------------------------------------------------------------
// The energy above 32 labels: the fused energy's definition and operation order (the comment above EnergyArgs in
// meanfield.cu) with the labels chunked into quads.  wn q is splatted once into spA / biA (the backward copies the
// splat to spC / biC) and blurred in K's order, the copy in K^T's.  Then
//   Potts   : one per-pixel pass slices each quad of each lattice and forms the terms or grad_q, with no planes;
//   matrices: the forward slices F_sp / F_bi into e->U / e->Q0 and mixes them with mu per pixel; the backward slices
//             F_k and F_k^T of one lattice at a time into those planes and forms g_k (mu_k F_k + mu_k^T F_k^T), the
//             spatial launch writing grad_q and the bilateral one adding to it.
// The forward's per-pixel terms go to per-block double sums e->en_part [B][nblk][4], which k_crf_energy_reduce adds in
// block order: no float atomics outside the splat, and no device memory beyond the fused energy's.
// ---------------------------------------------------------------------------------------------
struct WideEnergyArgs {
    WideLat sp, bi;             // values K S(wn q)
    WideLat spt, bit;           // values K^T S(wn q) (the backward)
    const float *q, *unary;     // [B][M][N]; unary may be nullptr
    const float *potts;         // {w1, w2} on the device, or nullptr: w1, w2
    float w1, w2, a_sp, a_bi;
    const float *grad_terms;    // [B][4] (the backward)
    float *grad_q, *grad_unary; // [B][M][N]; grad_unary may be nullptr
    double *part;               // [B][nblk][4] (the forward)
    int M, N, CH;
};

// the entropy and unary terms of one label (q at `at`) into acc[0..1]; BWD: returns the start of its grad_q and
// writes its grad_unary
template <bool BWD>
__device__ __forceinline__ float wide_energy_local(const WideEnergyArgs &a, size_t at, float q, float g0, float g1,
                                                   float acc[4]) {
    const float u = a.unary ? __ldg(a.unary + at) : 0.0f;
    const float lq = logf(fmaxf(q, 1e-20f));
    acc[0] = fmaf(q, lq, acc[0]);
    acc[1] = fmaf(-u, q, acc[1]);
    if constexpr (BWD) {
        if (a.grad_unary) a.grad_unary[at] = -g1 * q;
        return fmaf(-g1, u, g0 * (q > 1e-20f ? lq + 1.0f : lq));
    }
    return 0.0f;
}

// the block's per-pixel terms summed in double to part[b][block][4] (k_crf_energy's reduction)
__device__ __forceinline__ void wide_energy_block_sum(const float acc[4], double *part, int b) {
    __shared__ double red[kThreads / 32][4];
    double v[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        v[k] = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], o);
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 4; k++) red[threadIdx.x >> 5][k] = v[k];
    }
    __syncthreads();
    if (threadIdx.x < 4) {
        double s = 0.0;
        for (int w = 0; w < kThreads / 32; w++) s += red[w][threadIdx.x];
        part[((size_t)b * gridDim.x + blockIdx.x) * 4 + threadIdx.x] = s;
    }
}

// Potts, one thread per pixel over the label quads: the terms to the block sums or (BWD) grad_q = the local part
// + g_2 (-w2 F_sp) + g_2 (-w2 F_sp^T) + g_3 (-w1 F_bi) + g_3 (-w1 F_bi^T), in k_crf_energy's order
template <bool BWD>
__global__ void __launch_bounds__(kThreads)
k_wide_energy_potts(WideEnergyArgs a) {
    const int b = blockIdx.y, i = blockIdx.x * kThreads + threadIdx.x;
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (i < a.N) {
        const float w1 = a.potts ? __ldg(a.potts) : a.w1, w2 = a.potts ? __ldg(a.potts + 1) : a.w2;
        float g0 = 0.0f, g1 = 0.0f, g2 = 0.0f, g3 = 0.0f;
        if constexpr (BWD) {
            g0 = __ldg(a.grad_terms + 4 * b);
            g1 = __ldg(a.grad_terms + 4 * b + 1);
            g2 = __ldg(a.grad_terms + 4 * b + 2);
            g3 = __ldg(a.grad_terms + 4 * b + 3);
        }
        for (int c = 0; c < a.CH; c++) {
            float q[4], g[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int l = 4 * c + k;
                const size_t at = ((size_t)b * a.M + l) * a.N + i;
                q[k] = l < a.M ? __ldg(a.q + at) : 0.0f;
                g[k] = l < a.M ? wide_energy_local<BWD>(a, at, q[k], g0, g1, acc) : 0.0f;
            }
#pragma unroll
            for (int kk = 0; kk < 2; kk++) {
                const float w = kk == 0 ? w2 : w1, gk = kk == 0 ? g2 : g3;
                float f[4] = {0.0f, 0.0f, 0.0f, 0.0f};
                wide_slice_quad(kk == 0 ? a.sp : a.bi, kk == 0 ? a.a_sp : a.a_bi, b, i, c, a.N, a.CH, f);
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const float m = -w * f[k];
                    acc[2 + kk] = fmaf(q[k], m, acc[2 + kk]);
                    if constexpr (BWD) g[k] = fmaf(gk, m, g[k]);
                }
                if constexpr (BWD) {
                    float t[4] = {0.0f, 0.0f, 0.0f, 0.0f};
                    wide_slice_quad(kk == 0 ? a.spt : a.bit, kk == 0 ? a.a_sp : a.a_bi, b, i, c, a.N, a.CH, t);
#pragma unroll
                    for (int k = 0; k < 4; k++) g[k] = fmaf(gk, -w * t[k], g[k]);
                }
            }
            if constexpr (BWD) {
#pragma unroll
                for (int k = 0; k < 4; k++)
                    if (4 * c + k < a.M) a.grad_q[((size_t)b * a.M + 4 * c + k) * a.N + i] = g[k];
            }
        }
    }
    if constexpr (!BWD) wide_energy_block_sum(acc, a.part, b);
}

// Matrices, the forward: one thread per pixel, terms 0 / 1 over the labels and e_k = sum_l q_l (mu_k F_k)_l with
// (mu F)_l an fma chain over l' from zero, labels ascending.  mu's rows are staged kWideEnergyRows at a time, transposed
// ([l'][row]), so a stage reads each F_k[l'] once for all of its rows; any label count fits.  F_sp, F_bi [B][M][N].
constexpr int kWideEnergyRows = 16;
__global__ void __launch_bounds__(kThreads)
k_wide_energy_mat(WideEnergyArgs a, const float *compat, const float *F_sp, const float *F_bi) {
    constexpr int R = kWideEnergyRows;
    extern __shared__ float4 mus4[];   // [M][R / 4]
    const int b = blockIdx.y, i = blockIdx.x * kThreads + threadIdx.x, M = a.M, N = a.N;
    const bool in = i < N;
    const size_t px = (size_t)b * M * N + i;
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (in)
        for (int l = 0; l < M; l++) wide_energy_local<false>(a, px + (size_t)l * N, __ldg(a.q + px + (size_t)l * N), 0.0f, 0.0f, acc);
#pragma unroll 1
    for (int kk = 0; kk < 2; kk++) {
        const float *mu = compat + (kk == 0 ? (size_t)M * M : 0);   // compat = {mu_bi, mu_sp}
        const float *F = (kk == 0 ? F_sp : F_bi) + px;
        float ek = 0.0f;
        for (int l0 = 0; l0 < M; l0 += R) {
            __syncthreads();
            for (int e = threadIdx.x; e < R * M; e += kThreads) {
                const int l2 = e / R, r = e % R;
                reinterpret_cast<float *>(mus4)[e] = l0 + r < M ? __ldg(mu + (size_t)(l0 + r) * M + l2) : 0.0f;
            }
            __syncthreads();
            if (!in) continue;
            float m[R];
#pragma unroll
            for (int r = 0; r < R; r++) m[r] = 0.0f;
            for (int l2 = 0; l2 < M; l2++) {
                const float f = __ldg(F + (size_t)l2 * N);
#pragma unroll
                for (int r4 = 0; r4 < R / 4; r4++) {
                    const float4 v = mus4[l2 * (R / 4) + r4];
                    m[4 * r4] = fmaf(v.x, f, m[4 * r4]);
                    m[4 * r4 + 1] = fmaf(v.y, f, m[4 * r4 + 1]);
                    m[4 * r4 + 2] = fmaf(v.z, f, m[4 * r4 + 2]);
                    m[4 * r4 + 3] = fmaf(v.w, f, m[4 * r4 + 3]);
                }
            }
#pragma unroll
            for (int r = 0; r < R; r++)
                if (l0 + r < M) ek = fmaf(__ldg(a.q + px + (size_t)(l0 + r) * N), m[r], ek);
        }
        acc[2 + kk] = ek;
    }
    wide_energy_block_sum(acc, a.part, b);
}

// Matrices, the backward of one lattice (first: the spatial one, g_2, writing grad_q; else the bilateral one, g_3,
// adding to it): grad_q_l += g_k (mu F)_l, then mu[l'][l] (g_k F^T_l') over l' ascending, k_crf_energy's order.  One
// thread per (pixel, label quad); the quad's four rows and four columns of mu, 8 M floats in shared memory
// ([2 = rows, columns][M][4]).  F, Ft [B][M][N].
__global__ void __launch_bounds__(kThreads)
k_wide_energy_mat_bwd(WideEnergyArgs a, const float *mu, const float *F, const float *Ft, int first) {
    extern __shared__ float4 mq[];
    const int b = blockIdx.z, c = blockIdx.y, M = a.M, N = a.N;
    for (int e = threadIdx.x; e < 8 * M; e += blockDim.x) {
        const int m = e / (4 * M), l2 = (e / 4) % M, k = e & 3, l = 4 * c + k;
        reinterpret_cast<float *>(mq)[e] = l < M ? __ldg(m ? mu + (size_t)l2 * M + l : mu + (size_t)l * M + l2) : 0.0f;
    }
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const float gk = __ldg(a.grad_terms + 4 * b + (first ? 2 : 3));
    float g[4], m[4] = {0.0f, 0.0f, 0.0f, 0.0f}, unused[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int l = 4 * c + k;
        const size_t at = ((size_t)b * M + l) * N + i;
        if (l >= M)
            g[k] = 0.0f;
        else if (first)
            g[k] = wide_energy_local<true>(a, at, __ldg(a.q + at), __ldg(a.grad_terms + 4 * b),
                                           __ldg(a.grad_terms + 4 * b + 1), unused);
        else
            g[k] = a.grad_q[at];
    }
    const float *fp = F + (size_t)b * M * N + i, *tp = Ft + (size_t)b * M * N + i;
    for (int l2 = 0; l2 < M; l2++) {
        const float f = __ldg(fp + (size_t)l2 * N);
        const float4 r = mq[l2];
        m[0] = fmaf(r.x, f, m[0]);
        m[1] = fmaf(r.y, f, m[1]);
        m[2] = fmaf(r.z, f, m[2]);
        m[3] = fmaf(r.w, f, m[3]);
    }
#pragma unroll
    for (int k = 0; k < 4; k++) g[k] = fmaf(gk, m[k], g[k]);
    for (int l2 = 0; l2 < M; l2++) {
        const float t = gk * __ldg(tp + (size_t)l2 * N);
        const float4 r = mq[M + l2];
        g[0] = fmaf(r.x, t, g[0]);
        g[1] = fmaf(r.y, t, g[1]);
        g[2] = fmaf(r.z, t, g[2]);
        g[3] = fmaf(r.w, t, g[3]);
    }
#pragma unroll
    for (int k = 0; k < 4; k++)
        if (4 * c + k < M) a.grad_q[((size_t)b * M + 4 * c + k) * N + i] = g[k];
}

// copy the B images' rows of both lattices' splat targets (row counts device-resident, as k_wide_zero)
__global__ void __launch_bounds__(kThreads)
k_wide_energy_copy(const float4 *a, float4 *a2, const int32_t *rowbase_a, const float4 *c, float4 *c2,
                   const int32_t *rowbase_c, int B, int CH) {
    const long long na = (long long)rowbase_a[B] * CH, nc = (long long)rowbase_c[B] * CH;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < na + nc; t += (long long)gridDim.x * blockDim.x) {
        if (t < na) a2[t] = a[t]; else c2[t - na] = c[t - na];
    }
}

int meanfield_energy_wide(Engine *e, int B, const float *q, const float *unary, const float *potts, const float *compat,
                          const dsrg_crf_params &p, float *terms, const float *grad_terms, float *grad_q,
                          float *grad_unary, cudaStream_t s) {
    const int M = e->M, N = e->N, CH = e->MP / 4, nblk = cdiv(N, kThreads), grid = 8 * e->sm_count;
    const bool bwd = grad_terms != nullptr;
    const dim3 gp(nblk, B), gq(nblk, CH, B);
    const float a_sp = wide_alpha(e->sp), a_bi = wide_alpha(e->bi);
    const int tag = T_CRF_ENERGY;
    // S(wn q) into A, and for the gradient a copy in C.  K S(wn q) from A with B as scratch; K^T S(wn q) from C with
    // whichever of A / B the first result left free
    DSRG_LAUNCH(e, tag, s, k_wide_zero<<<grid, kThreads, 0, s>>>((float4 *)e->spA, e->sp.rowbase, (float4 *)e->biA, e->bi.rowbase, B, CH));
    DSRG_LAUNCH(e, tag, s, k_wide_splat<<<gq, kThreads, 0, s>>>(q, wide_lat(e->sp, e->spA), wide_lat(e->bi, e->biA), M, N, CH));
    if (bwd)
        DSRG_LAUNCH(e, tag, s,
                    k_wide_energy_copy<<<grid, kThreads, 0, s>>>((const float4 *)e->spA, (float4 *)e->spC, e->sp.rowbase,
                                                                 (const float4 *)e->biA, (float4 *)e->biC, e->bi.rowbase,
                                                                 B, CH));
    float *vf_sp = e->spA, *free_sp = e->spB, *vf_bi = e->biA, *free_bi = e->biB, *vt_sp = e->spC, *vt_bi = e->biC;
    wide_blur_axes(e, e->sp, B, false, tag, s, &vf_sp, &free_sp);
    wide_blur_axes(e, e->bi, B, false, tag, s, &vf_bi, &free_bi);
    if (bwd) {
        wide_blur_axes(e, e->sp, B, true, tag, s, &vt_sp, &free_sp);
        wide_blur_axes(e, e->bi, B, true, tag, s, &vt_bi, &free_bi);
    }
    const WideEnergyArgs a{wide_lat(e->sp, vf_sp), wide_lat(e->bi, vf_bi), wide_lat(e->sp, vt_sp),
                           wide_lat(e->bi, vt_bi), q, unary, potts, p.w1, p.w2, a_sp, a_bi, grad_terms, grad_q,
                           grad_unary, e->en_part, M, N, CH};
    if (!compat) {
        if (bwd)
            DSRG_LAUNCH(e, tag, s, k_wide_energy_potts<true><<<gp, kThreads, 0, s>>>(a));
        else
            DSRG_LAUNCH(e, tag, s, k_wide_energy_potts<false><<<gp, kThreads, 0, s>>>(a));
    } else if (!bwd) {   // e->U, e->Q0: F_sp, F_bi
        DSRG_LAUNCH(e, tag, s, k_wide_slice_planar<<<gq, kThreads, 0, s>>>(e->U, e->Q0, a.sp, a.bi, a_sp, a_bi, M, N, CH));
        DSRG_LAUNCH(e, tag, s,
                    k_wide_energy_mat<<<gp, kThreads, kWideEnergyRows * M * sizeof(float), s>>>(a, compat, e->U, e->Q0));
    } else {             // per lattice, e->U, e->Q0: F_k, F_k^T
        for (int kk = 0; kk < 2; kk++) {
            const float al = kk == 0 ? a_sp : a_bi;
            DSRG_LAUNCH(e, tag, s,
                        k_wide_slice_planar<<<gq, kThreads, 0, s>>>(e->U, e->Q0, kk == 0 ? a.sp : a.bi,
                                                                    kk == 0 ? a.spt : a.bit, al, al, M, N, CH));
            DSRG_LAUNCH(e, tag, s,
                        k_wide_energy_mat_bwd<<<gq, kThreads, 8 * M * sizeof(float), s>>>(
                            a, compat + (kk == 0 ? (size_t)M * M : 0), e->U, e->Q0, kk == 0));
        }
    }
    if (!bwd) DSRG_LAUNCH(e, tag, s, k_crf_energy_reduce<<<B, 32, 0, s>>>(e->en_part, nblk, terms));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

}  // namespace dsrg
