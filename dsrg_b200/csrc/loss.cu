// Balanced seeding loss (sm_90a); replaces BalancedSeedLossLayer's Theano graphs
// (pylayers/pylayers/pylayers.py:126-152).
//   S_bg(n) = sum lab_bg log p_bg, cnt_bg(n) = sum lab_bg   (channel 0)
//   S_fg(n), cnt_fg(n) likewise over channels 1..M-1
//   loss = -mean_n S_bg/max(cnt_bg,1e-4) - mean_n S_fg/max(cnt_fg,1e-4)
// Per-image sums are accumulated in float64 (Theano's float32 reduction order is unspecified).
#include "common.cuh"

namespace dsrg {

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// grid (chunks, B); acc[b][0..3] = S_bg, cnt_bg, S_fg, cnt_fg
__global__ void __launch_bounds__(kThreads)
k_seedloss_partial(const float *probs, const float *seeds, double *acc, int M, int N) {
    const int b = blockIdx.y;
    double s_bg = 0, c_bg = 0, s_fg = 0, c_fg = 0;
    const size_t base = (size_t)b * M * N;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < (long long)M * N;
         t += (long long)gridDim.x * blockDim.x) {
        const float lab = seeds[base + t];
        if (lab != 0.0f) {
            const double term = (double)lab * (double)logf(probs[base + t]);
            if (t < N) {
                s_bg += term;
                c_bg += lab;
            } else {
                s_fg += term;
                c_fg += lab;
            }
        }
    }
    __shared__ double sh[4][kThreads / 32];
    s_bg = warp_sum(s_bg);
    c_bg = warp_sum(c_bg);
    s_fg = warp_sum(s_fg);
    c_fg = warp_sum(c_fg);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) {
        sh[0][w] = s_bg;
        sh[1][w] = c_bg;
        sh[2][w] = s_fg;
        sh[3][w] = c_fg;
    }
    __syncthreads();
    if (threadIdx.x < 4) {
        double v = 0;
        for (int k = 0; k < kThreads / 32; k++) v += sh[threadIdx.x][k];
        if (v != 0.0) atomicAdd(acc + (size_t)b * 4 + threadIdx.x, v);
    }
}

__global__ void k_seedloss_final(const double *acc, float *terms, int B) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        double t0 = 0, t1 = 0;
        for (int b = 0; b < B; b++) {
            t0 += acc[b * 4 + 0] / fmax(acc[b * 4 + 1], (double)kMinProb);
            t1 += acc[b * 4 + 2] / fmax(acc[b * 4 + 3], (double)kMinProb);
        }
        terms[0] = (float)t0;
        terms[1] = (float)t1;
    }
}

// counts only (for backward)
__global__ void __launch_bounds__(kThreads)
k_seedloss_counts(const float *seeds, double *acc, int M, int N) {
    const int b = blockIdx.y;
    double c_bg = 0, c_fg = 0;
    const size_t base = (size_t)b * M * N;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < (long long)M * N;
         t += (long long)gridDim.x * blockDim.x) {
        const float lab = seeds[base + t];
        if (t < N) c_bg += lab; else c_fg += lab;
    }
    c_bg = warp_sum(c_bg);
    c_fg = warp_sum(c_fg);
    if ((threadIdx.x & 31) == 0) {
        if (c_bg != 0.0) atomicAdd(acc + (size_t)b * 4 + 1, c_bg);
        if (c_fg != 0.0) atomicAdd(acc + (size_t)b * 4 + 3, c_fg);
    }
}

__global__ void __launch_bounds__(kThreads)
k_seedloss_grad(const float *probs, const float *seeds, const double *acc, float scale, float *grad,
                int M, int N) {
    const int b = blockIdx.y;
    const size_t base = (size_t)b * M * N;
    const float cnt_bg = fmaxf((float)acc[b * 4 + 1], kMinProb);
    const float cnt_fg = fmaxf((float)acc[b * 4 + 3], kMinProb);
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < (long long)M * N;
         t += (long long)gridDim.x * blockDim.x) {
        const float lab = seeds[base + t];
        const float cnt = t < N ? cnt_bg : cnt_fg;
        grad[base + t] = (lab != 0.0f) ? -scale * lab / (probs[base + t] * cnt) : 0.0f;
    }
}

int seedloss_forward(Engine *e, int B, const float *probs, const float *seeds, float *terms_out,
                     cudaStream_t s) {
    DSRG_CUDA_TRY(cudaMemsetAsync(e->loss_acc, 0, sizeof(double) * 4 * B, s));
    dim3 g(cdiv((long long)e->M * e->N, kThreads * 8), B);
    DSRG_LAUNCH(e, T_LOSS, s, k_seedloss_partial<<<g, kThreads, 0, s>>>(probs, seeds, e->loss_acc, e->M, e->N));
    DSRG_LAUNCH(e, T_LOSS, s, k_seedloss_final<<<1, 32, 0, s>>>(e->loss_acc, terms_out, B));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int seedloss_backward(Engine *e, int B, int n_global, const float *probs, const float *seeds,
                      float top_diff, float *grad, cudaStream_t s) {
    DSRG_CUDA_TRY(cudaMemsetAsync(e->loss_acc, 0, sizeof(double) * 4 * B, s));
    dim3 g(cdiv((long long)e->M * e->N, kThreads * 8), B);
    DSRG_LAUNCH(e, T_LOSS, s, k_seedloss_counts<<<g, kThreads, 0, s>>>(seeds, e->loss_acc, e->M, e->N));
    DSRG_LAUNCH(e, T_LOSS, s,
                k_seedloss_grad<<<g, kThreads, 0, s>>>(probs, seeds, e->loss_acc, top_diff / (float)n_global, grad,
                                                       e->M, e->N));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

}  // namespace dsrg

// =================================================================================================
// SURVEY.md 8f rank 1: the producer of `probs` and the other consumer of the CRF result, on device.
// SoftmaxLayer (pylayers/pylayers/pylayers.py:23-51):  probs = (softmax(x) + 1e-4) / sum(softmax(x) + 1e-4)
// ConstrainLossLayer (pylayers.py:154-180): loss = mean_{n,h,w} sum_c ps log(clip(ps/p, 0.05, 20)), ps = exp(l)
// Backward passes are the analytic gradients of those expressions (what T.grad builds).
// =================================================================================================
namespace dsrg {

template <int MAXM>
__global__ void __launch_bounds__(kThreads)
k_softmax_fwd(const float *x, float *probs, int M, int N) {
    const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const float *xb = x + (size_t)b * M * N + i;
    float v[MAXM], mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < MAXM; k++)
        if (k < M) {
            v[k] = xb[(size_t)k * N];
            mx = fmaxf(mx, v[k]);
        }
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < MAXM; k++)
        if (k < M) {
            v[k] = expf(v[k] - mx);
            s += v[k];
        }
    float z = 0.0f;
#pragma unroll
    for (int k = 0; k < MAXM; k++)
        if (k < M) {
            v[k] = v[k] / s + kMinProb;
            z += v[k];
        }
    float *pb = probs + (size_t)b * M * N + i;
#pragma unroll
    for (int k = 0; k < MAXM; k++)
        if (k < M) pb[(size_t)k * N] = v[k] / z;
}

template <int MAXM>
__global__ void __launch_bounds__(kThreads)
k_softmax_bwd(const float *x, const float *top, float *grad, int M, int N) {
    const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const size_t o = (size_t)b * M * N + i;
    float s[MAXM], mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < MAXM; k++)
        if (k < M) {
            s[k] = x[o + (size_t)k * N];
            mx = fmaxf(mx, s[k]);
        }
    float sum = 0.0f;
#pragma unroll
    for (int k = 0; k < MAXM; k++)
        if (k < M) {
            s[k] = expf(s[k] - mx);
            sum += s[k];
        }
    float z = 0.0f, dot = 0.0f;  // z = sum(s + m), dot = sum top * (s + m)
#pragma unroll
    for (int k = 0; k < MAXM; k++)
        if (k < M) {
            s[k] /= sum;
            z += s[k] + kMinProb;
            dot += top[o + (size_t)k * N] * (s[k] + kMinProb);
        }
    float gs_dot_s = 0.0f;
#pragma unroll
    for (int k = 0; k < MAXM; k++)
        if (k < M) gs_dot_s += (top[o + (size_t)k * N] / z - dot / (z * z)) * s[k];
#pragma unroll
    for (int k = 0; k < MAXM; k++)
        if (k < M) grad[o + (size_t)k * N] = s[k] * ((top[o + (size_t)k * N] / z - dot / (z * z)) - gs_dot_s);
}

__global__ void __launch_bounds__(kThreads)
k_constrain_fwd(const float *probs, const float *logs, double *acc, long long total) {
    double a = 0.0;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const float ps = expf(logs[t]);
        const float r = fminf(fmaxf(ps / probs[t], 0.05f), 20.0f);
        a += (double)(ps * logf(r));
    }
    a = warp_sum(a);
    __shared__ double sh[kThreads / 32];
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = a;
    __syncthreads();
    if (threadIdx.x == 0) {
        double v = 0;
        for (int k = 0; k < kThreads / 32; k++) v += sh[k];
        atomicAdd(acc, v);
    }
}

__global__ void k_constrain_final(const double *acc, float *loss, double cnt) {
    if (threadIdx.x == 0 && blockIdx.x == 0) loss[0] = (float)(acc[0] / cnt);
}

__global__ void __launch_bounds__(kThreads)
k_constrain_bwd(const float *probs, const float *logs, float *gp, float *gl, long long total, float inv_cnt) {
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const float p = probs[t], ps = expf(logs[t]);
        const float ratio = ps / p;
        const float inside = (ratio >= 0.05f && ratio <= 20.0f) ? 1.0f : 0.0f;  // gradient of clip
        gp[t] = -(ps / p) * inside * inv_cnt;
        gl[t] = ps * (logf(fminf(fmaxf(ratio, 0.05f), 20.0f)) + inside) * inv_cnt;
    }
}

// CRFLayer.backward (pylayers.py:90-92): grad = (1 - result) * top_diff.  numpy evaluates it in float32, one rounding
// per operation; the explicit _rn intrinsics keep nvcc from contracting the pair into an FMA.
__global__ void __launch_bounds__(kThreads)
k_crflayer_bwd(const float *result, const float *top, float *grad, long long total) {
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x)
        grad[t] = __fmul_rn(__fsub_rn(1.0f, result[t]), top[t]);
}

int crflayer_backward(Engine *e, int B, const float *result, const float *top, float *grad, cudaStream_t s) {
    const long long total = (long long)B * e->M * e->N;
    const int grid = (int)(cdiv(total, kThreads) < 8 * e->sm_count ? cdiv(total, kThreads) : 8 * e->sm_count);
    DSRG_LAUNCH(e, T_LOSS, s, k_crflayer_bwd<<<grid, kThreads, 0, s>>>(result, top, grad, total));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

static int narrow_only(const Engine *e, const char *what) {
    if (e->M <= DSRG_MAX_LABELS) return DSRG_OK;
    set_error("%s supports at most %d labels (engine has %d)", what, DSRG_MAX_LABELS, e->M);
    return DSRG_E_INVALID;
}

int softmax_forward(Engine *e, int B, const float *x, float *probs, cudaStream_t s) {
    if (int rc = narrow_only(e, "SoftmaxLayer")) return rc;
    dim3 g(cdiv(e->N, kThreads), B);
    DSRG_LAUNCH(e, T_LOSS, s, k_softmax_fwd<DSRG_MAX_LABELS><<<g, kThreads, 0, s>>>(x, probs, e->M, e->N));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int softmax_backward(Engine *e, int B, const float *x, const float *top, float *grad, cudaStream_t s) {
    if (int rc = narrow_only(e, "SoftmaxLayer")) return rc;
    dim3 g(cdiv(e->N, kThreads), B);
    DSRG_LAUNCH(e, T_LOSS, s, k_softmax_bwd<DSRG_MAX_LABELS><<<g, kThreads, 0, s>>>(x, top, grad, e->M, e->N));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int constrain_forward(Engine *e, int B, const float *probs, const float *logs, float *loss, cudaStream_t s) {
    const long long total = (long long)B * e->M * e->N;
    DSRG_CUDA_TRY(cudaMemsetAsync(e->loss_acc, 0, sizeof(double), s));
    DSRG_LAUNCH(e, T_LOSS, s, k_constrain_fwd<<<4 * e->sm_count, kThreads, 0, s>>>(probs, logs, e->loss_acc, total));
    DSRG_LAUNCH(e, T_LOSS, s, k_constrain_final<<<1, 32, 0, s>>>(e->loss_acc, loss, (double)B * e->N));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int constrain_backward(Engine *e, int B, const float *probs, const float *logs, float *gp, float *gl,
                       cudaStream_t s) {
    const long long total = (long long)B * e->M * e->N;
    DSRG_LAUNCH(e, T_LOSS, s,
                k_constrain_bwd<<<4 * e->sm_count, kThreads, 0, s>>>(probs, logs, gp, gl, total,
                                                                     1.0f / ((float)B * (float)e->N)));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

}  // namespace dsrg

using namespace dsrg;

extern "C" {
int dsrg_seedloss_forward_dev(dsrg_engine *h, int B, const float *probs, const float *seeds, float *terms_out,
                              void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, probs && seeds && terms_out,
                    [&](Engine *e) { return seedloss_forward(e, B, probs, seeds, terms_out, s); });
}
int dsrg_seedloss_backward_dev(dsrg_engine *h, int B, int n_global, const float *probs, const float *seeds,
                               float top_diff, float *grad, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, probs && seeds && grad && n_global >= 1, [&](Engine *e) {
        return seedloss_backward(e, B, n_global, probs, seeds, top_diff, grad, s);
    });
}
int dsrg_seedloss_forward_host(dsrg_engine *h, int B, const float *probs, const float *seeds, float *terms_out) {
    return host_call(h, B, probs && seeds && terms_out, false, [&](Engine *e, cudaStream_t s) {
        const size_t n = (size_t)B * e->M * e->N;
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, probs, n * sizeof(float), cudaMemcpyHostToDevice, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_cues, seeds, n * sizeof(float), cudaMemcpyHostToDevice, s));
        if (int rc = seedloss_forward(e, B, e->st_unary, e->st_cues, e->st_labels, s)) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(terms_out, e->st_labels, 2 * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}
int dsrg_seedloss_backward_host(dsrg_engine *h, int B, int n_global, const float *probs, const float *seeds,
                                float top_diff, float *grad) {
    return host_call(h, B, probs && seeds && grad && n_global >= 1, false, [&](Engine *e, cudaStream_t s) {
        const size_t n = (size_t)B * e->M * e->N;
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, probs, n * sizeof(float), cudaMemcpyHostToDevice, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_cues, seeds, n * sizeof(float), cudaMemcpyHostToDevice, s));
        if (int rc = seedloss_backward(e, B, n_global, e->st_unary, e->st_cues, top_diff, e->st_out, s)) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(grad, e->st_out, n * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}

int dsrg_softmax_forward_dev(dsrg_engine *h, int B, const float *preds, float *probs_out, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, preds && probs_out, [&](Engine *e) { return softmax_forward(e, B, preds, probs_out, s); });
}
int dsrg_softmax_backward_dev(dsrg_engine *h, int B, const float *preds, const float *top_diff, float *grad_out,
                              void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, preds && top_diff && grad_out,
                    [&](Engine *e) { return softmax_backward(e, B, preds, top_diff, grad_out, s); });
}
int dsrg_constrainloss_forward_dev(dsrg_engine *h, int B, const float *probs, const float *log_smooth,
                                   float *loss_out, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, probs && log_smooth && loss_out,
                    [&](Engine *e) { return constrain_forward(e, B, probs, log_smooth, loss_out, s); });
}
int dsrg_constrainloss_backward_dev(dsrg_engine *h, int B, const float *probs, const float *log_smooth,
                                    float *grad_probs, float *grad_log, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, probs && log_smooth && grad_probs && grad_log,
                    [&](Engine *e) { return constrain_backward(e, B, probs, log_smooth, grad_probs, grad_log, s); });
}
int dsrg_crflayer_backward_dev(dsrg_engine *h, const float *result, const float *top_diff, int B, float *grad_out,
                               void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, result && top_diff && grad_out,
                    [&](Engine *e) { return crflayer_backward(e, B, result, top_diff, grad_out, s); });
}
int dsrg_softmax_forward_host(dsrg_engine *h, int B, const float *preds, float *probs_out) {
    return host_call(h, B, preds && probs_out, false, [&](Engine *e, cudaStream_t s) {
        const size_t n = (size_t)B * e->M * e->N;
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, preds, n * sizeof(float), cudaMemcpyHostToDevice, s));
        if (int rc = softmax_forward(e, B, e->st_unary, e->st_out, s)) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(probs_out, e->st_out, n * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}
int dsrg_softmax_backward_host(dsrg_engine *h, int B, const float *preds, const float *top_diff, float *grad_out) {
    return host_call(h, B, preds && top_diff && grad_out, false, [&](Engine *e, cudaStream_t s) {
        const size_t n = (size_t)B * e->M * e->N;
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, preds, n * sizeof(float), cudaMemcpyHostToDevice, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_cues, top_diff, n * sizeof(float), cudaMemcpyHostToDevice, s));
        if (int rc = softmax_backward(e, B, e->st_unary, e->st_cues, e->st_out, s)) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(grad_out, e->st_out, n * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}
int dsrg_constrainloss_forward_host(dsrg_engine *h, int B, const float *probs, const float *log_smooth,
                                    float *loss_out) {
    return host_call(h, B, probs && log_smooth && loss_out, false, [&](Engine *e, cudaStream_t s) {
        const size_t n = (size_t)B * e->M * e->N;
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, probs, n * sizeof(float), cudaMemcpyHostToDevice, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_cues, log_smooth, n * sizeof(float), cudaMemcpyHostToDevice, s));
        if (int rc = constrain_forward(e, B, e->st_unary, e->st_cues, e->st_labels, s)) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(loss_out, e->st_labels, sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}
int dsrg_constrainloss_backward_host(dsrg_engine *h, int B, const float *probs, const float *log_smooth,
                                     float *grad_probs, float *grad_log) {
    return host_call(h, B, probs && log_smooth && grad_probs && grad_log, false, [&](Engine *e, cudaStream_t s) {
        const size_t n = (size_t)B * e->M * e->N;
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, probs, n * sizeof(float), cudaMemcpyHostToDevice, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_cues, log_smooth, n * sizeof(float), cudaMemcpyHostToDevice, s));
        // the second gradient is staged through U: every st_* buffer of this size already holds an input or output
        if (int rc = constrain_backward(e, B, e->st_unary, e->st_cues, e->st_out, e->U, s)) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(grad_probs, e->st_out, n * sizeof(float), cudaMemcpyDeviceToHost, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(grad_log, e->U, n * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}
}
