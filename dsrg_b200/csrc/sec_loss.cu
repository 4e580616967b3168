// SEC's seeding and expansion losses (Kolesnikov & Lampert, ECCV 2016) on the device (sm_90a); replaces the
// Theano graphs of SeedLossLayer (pylayers/pylayers/pylayers.py:95-118) and ExpandLossLayer (:183-233).
//
// SeedLossLayer:   loss = -mean_n( sum_{c,h,w} lab log p / sum lab )     (no max(count, 1e-4) floor)
// ExpandLossLayer: loss = loss_1 + loss_2 + loss_3 over the present (s_k = stat_k > 0.5) and absent fg classes:
//   loss_1 = -mean_n sum_k s_k log G_fg(p_k) / P,  loss_2 = -mean_n sum_k (1-s_k) log(1 - max p_k) / A,
//   loss_3 = -mean_n log G_bg(p_0),  G_q(x) = sum_i sort(x)_i q^(n-1-i) / Z,  Z = sum_i q^i     (:198-218)
// Global weighted rank pooling (GWRP) runs one CTA per (image, class plane): the plane is sorted in shared
// memory (bitonic network on (float key, pixel index) pairs), the rank-weighted sum is formed in float64 and the
// plane max is the last sorted value.  Every reduction has a fixed order and there are no float atomics, so two
// identical calls give bit-identical losses and gradients.
//
// Backward follows what Theano 0.8.2's T.grad builds (restated from its source; not pinned against Theano itself):
// the gradient of a sorted position goes to the element argsort put there (SortOp.grad), and the gradient of the
// plane max goes IN FULL to every element equal to the max (MaxAndArgmax.grad: eq(xmax, x) * g_max).  With P = 0
// or A = 0 the coefficient is 0/0 = NaN and eq(...) * NaN makes the whole foreground plane NaN, as in Theano.
#include <math.h>

#include "common.cuh"

namespace dsrg {

namespace {

constexpr int kSortThreads = 512;
constexpr int kPlainChunks = kSecPlainChunks;

__device__ __forceinline__ uint32_t float_key(float f) {  // order-preserving map of float bits to uint32
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float key_float(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// fixed-order block sum (blockDim.x a multiple of 32, <= 1024); every thread gets the result
__device__ double block_sum_d(double v, double *scratch /* [33] */) {
    v = warp_sum_d(v);
    const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();  // scratch may still be read from a previous call
    if ((threadIdx.x & 31) == 0) scratch[w] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int k = 0; k < nw; k++) s += scratch[k];
        scratch[32] = s;
    }
    __syncthreads();
    return scratch[32];
}

// Stage plane `x` (n values) as (key << 32 | pixel index) in `s`, pad to n2 (a power of two) with keys above any
// float, sort ascending.  Equal values end up in ascending pixel order.
__device__ void sort_plane(const float *__restrict__ x, int n, int n2, unsigned long long *s) {
    for (int i = threadIdx.x; i < n2; i += blockDim.x)
        s[i] = i < n ? ((unsigned long long)float_key(x[i]) << 32) | (unsigned)i : ~0ull;
    __syncthreads();
    for (int k = 2; k <= n2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < (n2 >> 1); t += blockDim.x) {
                const int i = 2 * t - (t & (j - 1)), l = i + j;
                const unsigned long long a = s[i], b = s[l];
                if ((a > b) == ((i & k) == 0)) {
                    s[i] = b;
                    s[l] = a;
                }
            }
            __syncthreads();
        }
    }
}

// G = sum_i (sort(x)_i * w_i) / Z in float64 (the reference divides each product by Z before the sum, :205)
__device__ double gwrp_sum(const unsigned long long *s, int n, const double *__restrict__ w, double Z,
                           double *scratch) {
    double acc = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) acc += ((double)key_float((uint32_t)(s[i] >> 32)) * w[i]) / Z;
    return block_sum_d(acc, scratch);
}

struct GwrpArgs {
    const float *probs;   // [B][M][n]
    const float *labels;  // [B][M]: stat (the labels blob, N x 1 x 1 x M)
    const double *w_fg, *w_bg;  // [n] q^(n-1-i)
    double z_fg, z_bg;
    int M, n, n2;
};

__device__ __forceinline__ void image_counts(const float *lab, int M, int *P, int *A) {
    int p = 0;
    for (int k = 1; k < M; k++) p += lab[k] > 0.5f;
    *P = p;
    *A = (M - 1) - p;
}

// grid (M, B): one record per plane, rec = (G, max)
__global__ void __launch_bounds__(kSortThreads)
k_gwrp_fwd(GwrpArgs a, double2 *rec) {
    extern __shared__ unsigned long long sh_keys[];
    __shared__ double scratch[33];
    const int k = blockIdx.x, b = blockIdx.y;
    sort_plane(a.probs + ((size_t)b * a.M + k) * a.n, a.n, a.n2, sh_keys);
    const double G = gwrp_sum(sh_keys, a.n, k == 0 ? a.w_bg : a.w_fg, k == 0 ? a.z_bg : a.z_fg, scratch);
    if (threadIdx.x == 0) rec[(size_t)b * a.M + k] = make_double2(G, (double)key_float((uint32_t)(sh_keys[a.n - 1] >> 32)));
}

// One CTA: image b's three sums over its planes in class order, then the batch sums in image order.
//   terms[0] = sum_n sum_k s_k log G_k / P,  terms[1] = sum_n sum_k (1-s_k) log(1 - max_k) / A,
//   terms[2] = sum_n log G_bg;  loss = -(terms[0] + terms[1] + terms[2]) / N.
__global__ void k_gwrp_final(const double2 *rec, const float *labels, double *img, float *terms, int B, int M) {
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const float *lab = labels + (size_t)b * M;
        int P, A;
        image_counts(lab, M, &P, &A);
        double l1 = 0.0, l2 = 0.0;
        for (int k = 1; k < M; k++) {
            const int s = lab[k] > 0.5f;
            const double2 r = rec[(size_t)b * M + k];
            // dtypes of the reference's graph: the GWRP path is float64 (float64 weights), log(1 - max) and its
            // product with the int8 mask are float32, the division by the integer counts is float64
            l1 += (double)s * log(r.x) / (double)P;
            l2 += (double)((float)(1 - s) * logf(1.0f - (float)r.y)) / (double)A;
        }
        img[(size_t)b * 3 + 0] = l1;
        img[(size_t)b * 3 + 1] = l2;
        img[(size_t)b * 3 + 2] = log(rec[(size_t)b * M].x);
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        double t = 0.0;
        for (int b = 0; b < B; b++) t += img[(size_t)b * 3 + threadIdx.x];
        terms[threadIdx.x] = (float)t;
    }
}

// grid (M, B).  Re-sorts (the reference recomputes from the bottoms), then writes, for the element of rank i,
//   cs * w_i / Z + [x == max] * cm
// with cs = dloss/dG and cm = dloss/dmax of the plane; the values are staged in shared memory by pixel index
// so that the global stores are coalesced.
__global__ void __launch_bounds__(kSortThreads)
k_gwrp_bwd(GwrpArgs a, double inv_n, float *grad) {
    extern __shared__ unsigned long long sh_keys[];
    __shared__ double scratch[33];
    float *sh_grad = reinterpret_cast<float *>(sh_keys + a.n2);
    const int k = blockIdx.x, b = blockIdx.y;
    const size_t base = ((size_t)b * a.M + k) * a.n;
    sort_plane(a.probs + base, a.n, a.n2, sh_keys);
    const double *w = k == 0 ? a.w_bg : a.w_fg;
    const double Z = k == 0 ? a.z_bg : a.z_fg;
    const double G = gwrp_sum(sh_keys, a.n, w, Z, scratch);
    const float mx = key_float((uint32_t)(sh_keys[a.n - 1] >> 32));
    double cs, cm;
    if (k == 0) {
        cs = -inv_n / G;  // d(-mean log G_bg)/dG
        cm = 0.0;
    } else {
        const float *lab = a.labels + (size_t)b * a.M;
        int P, A;
        image_counts(lab, a.M, &P, &A);
        const int s = lab[k] > 0.5f;
        cs = -inv_n * ((double)s / (double)P) / G;                                  // 0/0 = NaN when P = 0
        cm = inv_n * ((double)(1 - s) / (double)A) / (double)(1.0f - mx);          // 0/0 = NaN when A = 0
    }
    for (int i = threadIdx.x; i < a.n; i += blockDim.x) {
        const unsigned long long e = sh_keys[i];
        const float x = key_float((uint32_t)(e >> 32));
        // eq(xmax, x) * g_max: 0 * NaN stays NaN, so a NaN max gradient reaches every element of the plane
        const double g = cs * (w[i] / Z) + (x == mx ? cm : cm * 0.0);
        sh_grad[(uint32_t)e & 0xFFFFu] = (float)g;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < a.n; i += blockDim.x) grad[base + i] = sh_grad[i];
}

// ---- SeedLossLayer ----
// grid (kPlainChunks, B): part[b][chunk] = (sum lab * log p, sum lab) over a fixed slice of image b
template <bool kLog>
__global__ void __launch_bounds__(kThreads)
k_plainseed_partial(const float *probs, const float *seeds, double2 *part, int MN) {
    __shared__ double scratch[33];
    const int b = blockIdx.y;
    const size_t base = (size_t)b * MN;
    double s = 0.0, c = 0.0;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < MN; t += gridDim.x * blockDim.x) {
        const float lab = seeds[base + t];
        if (kLog) s += (double)lab * (double)logf(probs[base + t]);  // no skip of lab == 0: 0 * log(0) is NaN there too
        c += lab;
    }
    if (kLog) s = block_sum_d(s, scratch);
    c = block_sum_d(c, scratch);
    if (threadIdx.x == 0) part[(size_t)b * gridDim.x + blockIdx.x] = make_double2(s, c);
}

// img[b] = (S_b, cnt_b) in chunk order; terms[0] = sum_b S_b / cnt_b in image order (NaN for cnt_b = 0)
__global__ void k_plainseed_final(const double2 *part, double2 *img, float *terms, int B) {
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        double s = 0.0, c = 0.0;
        for (int j = 0; j < kPlainChunks; j++) {
            s += part[(size_t)b * kPlainChunks + j].x;
            c += part[(size_t)b * kPlainChunks + j].y;
        }
        img[b] = make_double2(s, c);
    }
    __syncthreads();
    if (terms && threadIdx.x == 0) {
        double t = 0.0;
        for (int b = 0; b < B; b++) t += img[b].x / img[b].y;
        terms[0] = (float)t;
    }
}

// grad = lab * (-1 / (N * cnt)) / p; an image without seeds (cnt = 0) gets 0 * -inf = NaN, as Theano's graph does
__global__ void __launch_bounds__(kThreads)
k_plainseed_grad(const float *probs, const float *seeds, const double2 *img, double n_global, float *grad, int MN) {
    const int b = blockIdx.y;
    const size_t base = (size_t)b * MN;
    const float inv = (float)(-1.0 / (n_global * img[b].y));
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < MN; t += gridDim.x * blockDim.x)
        grad[base + t] = seeds[base + t] * inv / probs[base + t];
}

int next_pow2(int n) {
    int p = 1;
    while (p < n) p <<= 1;
    return p;
}

// the q^i table of one (q, n), built on the host with libm pow like the reference's `q ** i` (:202, :209)
int gwrp_weights(Engine *e, int which, double q, cudaStream_t s) {
    const int n = e->N;
    if (e->sec_n[which] == n && e->sec_q[which] == q) return DSRG_OK;
    std::vector<double> &w = e->sec_w_host[which];
    w.resize(n);
    for (int i = 0; i < n; i++) w[i] = pow(q, (double)(n - 1 - i));
    double z = 0.0;
    for (int i = 0; i < n; i++) z += w[i];
    // w lives in the engine: the copy may still be reading it after this call returns
    DSRG_CUDA_TRY(cudaMemcpyAsync(e->sec_w + (size_t)which * e->sec_wcap, w.data(), n * sizeof(double),
                                  cudaMemcpyHostToDevice, s));
    e->sec_q[which] = q;
    e->sec_n[which] = n;
    e->sec_z[which] = z;
    return DSRG_OK;
}

int gwrp_setup(Engine *e, const float *probs, const float *labels, double q_fg, double q_bg, GwrpArgs *a,
               size_t *smem_fwd, size_t *smem_bwd, cudaStream_t s) {
    if (e->N > DSRG_GWRP_MAX_PLANE) {
        set_error("ExpandLoss: a %dx%d plane has %d pixels; the GWRP kernels sort at most %d", e->H, e->W, e->N,
                  DSRG_GWRP_MAX_PLANE);
        return DSRG_E_INVALID;
    }
    if (e->M < 2) {
        set_error("ExpandLoss needs a background and at least one foreground class (engine has M=%d)", e->M);
        return DSRG_E_INVALID;
    }
    if (!(q_fg > 0.0) || !(q_bg > 0.0)) {
        set_error("ExpandLoss: q_fg and q_bg must be positive (got %g, %g)", q_fg, q_bg);
        return DSRG_E_INVALID;
    }
    int rc;
    if ((rc = gwrp_weights(e, 0, q_fg, s)) || (rc = gwrp_weights(e, 1, q_bg, s))) return rc;
    a->probs = probs;
    a->labels = labels;
    a->w_fg = e->sec_w;
    a->w_bg = e->sec_w + e->sec_wcap;
    a->z_fg = e->sec_z[0];
    a->z_bg = e->sec_z[1];
    a->M = e->M;
    a->n = e->N;
    a->n2 = next_pow2(e->N);
    *smem_fwd = (size_t)a->n2 * sizeof(unsigned long long);
    *smem_bwd = *smem_fwd + (size_t)a->n2 * sizeof(float);
    DSRG_CUDA_TRY(cudaFuncSetAttribute(k_gwrp_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem_fwd));
    DSRG_CUDA_TRY(cudaFuncSetAttribute(k_gwrp_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem_bwd));
    return DSRG_OK;
}

}  // namespace

int expandloss_forward(Engine *e, int B, const float *probs, const float *labels, double q_fg, double q_bg,
                       float *terms_out, cudaStream_t s) {
    GwrpArgs a;
    size_t sf, sb;
    int rc = gwrp_setup(e, probs, labels, q_fg, q_bg, &a, &sf, &sb, s);
    if (rc) return rc;
    DSRG_LAUNCH(e, T_LOSS, s, k_gwrp_fwd<<<dim3(e->M, B), kSortThreads, sf, s>>>(a, e->sec_rec));
    DSRG_LAUNCH(e, T_LOSS, s, k_gwrp_final<<<1, 128, 0, s>>>(e->sec_rec, labels, e->sec_img, terms_out, B, e->M));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int expandloss_backward(Engine *e, int B, int n_global, const float *probs, const float *labels, double q_fg,
                        double q_bg, float *grad, cudaStream_t s) {
    GwrpArgs a;
    size_t sf, sb;
    int rc = gwrp_setup(e, probs, labels, q_fg, q_bg, &a, &sf, &sb, s);
    if (rc) return rc;
    DSRG_LAUNCH(e, T_LOSS, s, k_gwrp_bwd<<<dim3(e->M, B), kSortThreads, sb, s>>>(a, 1.0 / n_global, grad));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int plainseed_forward(Engine *e, int B, const float *probs, const float *seeds, float *terms_out, cudaStream_t s) {
    const int MN = e->M * e->N;
    double2 *img = reinterpret_cast<double2 *>(e->sec_img);
    DSRG_LAUNCH(e, T_LOSS, s,
                k_plainseed_partial<true><<<dim3(kPlainChunks, B), kThreads, 0, s>>>(probs, seeds, e->sec_part, MN));
    DSRG_LAUNCH(e, T_LOSS, s, k_plainseed_final<<<1, 128, 0, s>>>(e->sec_part, img, terms_out, B));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int plainseed_backward(Engine *e, int B, int n_global, const float *probs, const float *seeds, float *grad,
                       cudaStream_t s) {
    const int MN = e->M * e->N;
    double2 *img = reinterpret_cast<double2 *>(e->sec_img);
    DSRG_LAUNCH(e, T_LOSS, s,
                k_plainseed_partial<false><<<dim3(kPlainChunks, B), kThreads, 0, s>>>(probs, seeds, e->sec_part, MN));
    DSRG_LAUNCH(e, T_LOSS, s, k_plainseed_final<<<1, 128, 0, s>>>(e->sec_part, img, nullptr, B));
    DSRG_LAUNCH(e, T_LOSS, s,
                k_plainseed_grad<<<dim3(cdiv(MN, kThreads * 8), B), kThreads, 0, s>>>(probs, seeds, img,
                                                                                      (double)n_global, grad, MN));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

}  // namespace dsrg

using namespace dsrg;

// the *_host twins stage probs in st_unary and the labels or seeds in st_cues; the terms come back through
// st_labels, the gradient through st_out
extern "C" {
int dsrg_expandloss_forward_dev(dsrg_engine *h, int B, const float *probs, const float *labels, double q_fg,
                                double q_bg, float *terms_out, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, probs && labels && terms_out,
                    [&](Engine *e) { return expandloss_forward(e, B, probs, labels, q_fg, q_bg, terms_out, s); });
}
int dsrg_expandloss_backward_dev(dsrg_engine *h, int B, int n_global, const float *probs, const float *labels,
                                 double q_fg, double q_bg, float *grad_out, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, probs && labels && grad_out && n_global >= 1, [&](Engine *e) {
        return expandloss_backward(e, B, n_global, probs, labels, q_fg, q_bg, grad_out, s);
    });
}
int dsrg_expandloss_forward_host(dsrg_engine *h, int B, const float *probs, const float *labels, double q_fg,
                                 double q_bg, float *terms_out) {
    return host_call(h, B, probs && labels && terms_out, false, [&](Engine *e, cudaStream_t s) {
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, probs, (size_t)B * e->M * e->N * sizeof(float), cudaMemcpyHostToDevice, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_cues, labels, (size_t)B * e->M * sizeof(float), cudaMemcpyHostToDevice, s));
        if (int rc = expandloss_forward(e, B, e->st_unary, e->st_cues, q_fg, q_bg, e->st_labels, s)) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(terms_out, e->st_labels, 3 * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}
int dsrg_expandloss_backward_host(dsrg_engine *h, int B, int n_global, const float *probs, const float *labels,
                                  double q_fg, double q_bg, float *grad_out) {
    return host_call(h, B, probs && labels && grad_out && n_global >= 1, false, [&](Engine *e, cudaStream_t s) {
        const size_t n = (size_t)B * e->M * e->N;
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, probs, n * sizeof(float), cudaMemcpyHostToDevice, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_cues, labels, (size_t)B * e->M * sizeof(float), cudaMemcpyHostToDevice, s));
        if (int rc = expandloss_backward(e, B, n_global, e->st_unary, e->st_cues, q_fg, q_bg, e->st_out, s)) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(grad_out, e->st_out, n * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}
int dsrg_seedloss_plain_forward_dev(dsrg_engine *h, int B, const float *probs, const float *seeds, float *terms_out,
                                    void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, probs && seeds && terms_out,
                    [&](Engine *e) { return plainseed_forward(e, B, probs, seeds, terms_out, s); });
}
int dsrg_seedloss_plain_backward_dev(dsrg_engine *h, int B, int n_global, const float *probs, const float *seeds,
                                     float *grad_out, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, probs && seeds && grad_out && n_global >= 1,
                    [&](Engine *e) { return plainseed_backward(e, B, n_global, probs, seeds, grad_out, s); });
}
int dsrg_seedloss_plain_forward_host(dsrg_engine *h, int B, const float *probs, const float *seeds, float *terms_out) {
    return host_call(h, B, probs && seeds && terms_out, false, [&](Engine *e, cudaStream_t s) {
        const size_t n = (size_t)B * e->M * e->N;
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, probs, n * sizeof(float), cudaMemcpyHostToDevice, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_cues, seeds, n * sizeof(float), cudaMemcpyHostToDevice, s));
        if (int rc = plainseed_forward(e, B, e->st_unary, e->st_cues, e->st_labels, s)) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(terms_out, e->st_labels, sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}
int dsrg_seedloss_plain_backward_host(dsrg_engine *h, int B, int n_global, const float *probs, const float *seeds,
                                      float *grad_out) {
    return host_call(h, B, probs && seeds && grad_out && n_global >= 1, false, [&](Engine *e, cudaStream_t s) {
        const size_t n = (size_t)B * e->M * e->N;
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, probs, n * sizeof(float), cudaMemcpyHostToDevice, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_cues, seeds, n * sizeof(float), cudaMemcpyHostToDevice, s));
        if (int rc = plainseed_backward(e, B, n_global, e->st_unary, e->st_cues, e->st_out, s)) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(grad_out, e->st_out, n * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}
}
