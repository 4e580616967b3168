// Full-resolution inference post-processing on the device (SURVEY.md 8f rank 3): the tail of
// predict_mask() in the reference's evaluation / ground-truth tools, i.e. everything between the
// network's fc8 score blob and the label map that is written as a PNG:
//
//   DSRG_POST_SUM_SCORES  training/tools/test-ms.py:84-111
//       scores_all = sum_k zoom(scores_k (h_k,w_k,M) -> (d1,d2,M), order=1)        :91-98
//       probs = softmax(scores_all, axis=2); probs[probs < eps] = eps               :100-104
//       result = argmax(CRF(im, log(probs), scale_factor=1.0), axis=2)              :106-109
//   DSRG_POST_ZOOM_PROBS  training/tools/generate_train_gt.py:76-104
//       probs = softmax(scores (h,w,M)); probs = zoom(probs -> (d1,d2,M), order=1)  :86-88
//       probs[probs < eps] = eps; probs = CRF(im, log(probs), scale_factor=1.0)     :90-94
//       result = labels[argmax(probs[:, :, labels])],  labels = [0] + image tags    :96-100
//
// The zoom keeps scipy's arithmetic exactly (float64, scipy's tap order, float32 result; see zoom.cuh),
// so with identical scores the unary handed to the CRF differs from the reference's only by the ulps of
// expf/logf; the label map then follows the CRF's 1e-4 parity bound (ties within it may flip).
#include "common.cuh"
#include "zoom.cuh"

namespace dsrg {

// in [M][h][w] float32 (the blob the reference transposes to (h,w,M) before zooming) -> out [H][W][M]
template <bool ACC>
__global__ void __launch_bounds__(kThreads)
k_zoom_scores(const float *__restrict__ in, float *out, int M, int hi, int wi, int Ho, int Wo) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)Ho * Wo * M) return;
    const int c = (int)(idx % M);
    const int pix = (int)(idx / M);
    const int oy = pix / Wo, ox = pix - oy * Wo;
    const float z = zoom_apply(in + (size_t)c * hi * wi, wi, zoom_tap(oy, ox, hi, wi, Ho, Wo));
    out[idx] = ACC ? __fadd_rn(out[idx], z) : z;  // scores_all += scores (float32)
}

// softmax over the labels of every pixel, strides in elements: label stride ls, pixel stride ps
// (CHW blob: ls = npix, ps = 1; HWC map: ls = 1, ps = M).  Mirrors
//   e = np.exp(s - np.max(s)); p = e / np.sum(e)            (float32)
// and, when CLAMPLOG, the clamp at eps followed by np.log; `probs` (optional) receives the clamped p.
template <bool CLAMPLOG>
__global__ void __launch_bounds__(kThreads)
k_post_softmax(const float *in, float *out, float *probs, int npix, int M, long long ls, long long ps,
               float eps) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    const float *s = in + (size_t)i * ps;
    float v[DSRG_MAX_LABELS];
    float m = -INFINITY;
#pragma unroll
    for (int l = 0; l < DSRG_MAX_LABELS; l++)
        if (l < M) {
            v[l] = s[(size_t)l * ls];
            m = fmaxf(m, v[l]);
        }
    float sum = 0.f;
#pragma unroll
    for (int l = 0; l < DSRG_MAX_LABELS; l++)
        if (l < M) {
            v[l] = expf(__fsub_rn(v[l], m));
            sum = __fadd_rn(sum, v[l]);
        }
#pragma unroll
    for (int l = 0; l < DSRG_MAX_LABELS; l++)
        if (l < M) {
            float p = __fdiv_rn(v[l], sum);
            if (CLAMPLOG) {
                if (p < eps) p = eps;
                if (probs) probs[(size_t)i * ps + (size_t)l * ls] = p;
                p = logf(p);
            }
            out[(size_t)i * ps + (size_t)l * ls] = p;
        }
}

// The same for M > DSRG_MAX_LABELS (the COCO tools' 81 labels): the label vector does not fit in registers, so
// exp(s - max) is parked in `out` (in may alias out: each thread owns its pixel) and read back for the division.
// Same float32 operations in the same order as k_post_softmax.
template <bool CLAMPLOG>
__global__ void __launch_bounds__(kThreads)
k_post_softmax_wide(const float *in, float *out, float *probs, int npix, int M, long long ls, long long ps,
                    float eps) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    const float *s = in + (size_t)i * ps;
    float *o = out + (size_t)i * ps;
    float m = -INFINITY;
    for (int l = 0; l < M; l++) m = fmaxf(m, s[(size_t)l * ls]);
    float sum = 0.f;
    for (int l = 0; l < M; l++) {
        const float v = expf(__fsub_rn(s[(size_t)l * ls], m));
        o[(size_t)l * ls] = v;
        sum = __fadd_rn(sum, v);
    }
    for (int l = 0; l < M; l++) {
        float p = __fdiv_rn(o[(size_t)l * ls], sum);
        if (CLAMPLOG) {
            if (p < eps) p = eps;
            if (probs) probs[(size_t)i * ps + (size_t)l * ls] = p;
            p = logf(p);
        }
        o[(size_t)l * ls] = p;
    }
}

template <bool CLAMPLOG>
static void post_softmax(Engine *e, const float *in, float *out, float *probs, int npix, long long ls, long long ps,
                         float eps, cudaStream_t s) {
    const int g = cdiv(npix, kThreads), M = e->M;
    if (M > DSRG_MAX_LABELS)
        DSRG_LAUNCH(e, T_POST, s, k_post_softmax_wide<CLAMPLOG><<<g, kThreads, 0, s>>>(in, out, probs, npix, M, ls, ps, eps));
    else
        DSRG_LAUNCH(e, T_POST, s, k_post_softmax<CLAMPLOG><<<g, kThreads, 0, s>>>(in, out, probs, npix, M, ls, ps, eps));
}

// probs[probs < eps] = eps; unary = np.log(probs)   (generate_train_gt.py:90-94), element-wise
__global__ void __launch_bounds__(kThreads)
k_post_clamp_log(const float *in, float *out, float *probs, long long n, float eps) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float p = in[i];
    if (p < eps) p = eps;
    if (probs) probs[i] = p;
    out[i] = logf(p);
}

struct LabelSel {   // 1 KB of kernel parameters
    int n;
    int id[DSRG_MAX_LABELS_WIDE];
};

// np.argmax (first maximum) over the selected labels, result = the selected label's id
__global__ void __launch_bounds__(kThreads)
k_post_argmax(const float *q, int32_t *out, int npix, long long ls, long long ps, LabelSel sel) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    const float *s = q + (size_t)i * ps;
    float best = s[(size_t)sel.id[0] * ls];
    int arg = sel.id[0];
    for (int k = 1; k < sel.n; k++) {
        const float v = s[(size_t)sel.id[k] * ls];
        if (v > best) {
            best = v;
            arg = sel.id[k];
        }
    }
    out[i] = arg;
}

int zoom_scores(Engine *e, const float *in, int hi, int wi, float *out, int accumulate, cudaStream_t s) {
    const long long n = (long long)e->N * e->M;
    const int g = cdiv(n, kThreads);
    if (accumulate)
        DSRG_LAUNCH(e, T_POST, s, k_zoom_scores<true><<<g, kThreads, 0, s>>>(in, out, e->M, hi, wi, e->H, e->W));
    else
        DSRG_LAUNCH(e, T_POST, s, k_zoom_scores<false><<<g, kThreads, 0, s>>>(in, out, e->M, hi, wi, e->H, e->W));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int crf_core_for_post(Engine *e, const float *unary_hwc, const uint8_t *image, const dsrg_crf_params *p,
                      cudaStream_t s);  // api.cu

static int predict_mask_body(Engine *e, int mode, int n_scales, const float *const *scores, const int *hs, const int *ws,
                             const uint8_t *image, float eps, int smooth, const dsrg_crf_params *p, const LabelSel &sel,
                             int32_t *result, float *probs_out, cudaStream_t s) {
    int rc;
    const int N = e->N, M = e->M;
    float *unary = e->st_unary;                       // [H][W][M]
    float *clamped = smooth ? nullptr : (probs_out ? probs_out : e->st_out);
    if (mode == DSRG_POST_SUM_SCORES) {
        for (int k = 0; k < n_scales; k++)
            if ((rc = zoom_scores(e, scores[k], hs[k], ws[k], unary, k > 0, s))) return rc;
        post_softmax<true>(e, unary, unary, clamped, N, 1, M, eps, s);
    } else {
        const int np = hs[0] * ws[0];
        float *small = e->st_cues;                    // [M][h][w] probabilities at network resolution
        post_softmax<false>(e, scores[0], small, nullptr, np, np, 1, eps, s);
        if ((rc = zoom_scores(e, small, hs[0], ws[0], unary, 0, s))) return rc;
        const long long n = (long long)N * M;
        DSRG_LAUNCH(e, T_POST, s, k_post_clamp_log<<<cdiv(n, kThreads), kThreads, 0, s>>>(unary, unary, clamped, n, eps));
    }
    DSRG_CUDA_TRY(cudaGetLastError());
    if (smooth) {
        if ((rc = crf_core_for_post(e, unary, image, p, s))) return rc;
        if (probs_out && (rc = meanfield_export(e, 1, probs_out, DSRG_LAYOUT_NHWC, s))) return rc;
        DSRG_LAUNCH(e, T_POST, s, k_post_argmax<<<cdiv(N, kThreads), kThreads, 0, s>>>(e->Qcur, result, N, N, 1, sel));
    } else {
        DSRG_LAUNCH(e, T_POST, s, k_post_argmax<<<cdiv(N, kThreads), kThreads, 0, s>>>(clamped, result, N, 1, M, sel));
    }
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

static int predict_mask(Engine *e, int mode, int n_scales, const float *const *scores, const int *hs,
                        const int *ws, const uint8_t *image, float eps, int smooth, const dsrg_crf_params *p,
                        const int32_t *labels_sel, int n_sel, int32_t *result, float *probs_out,
                        cudaStream_t s) {
    if (mode != DSRG_POST_SUM_SCORES && mode != DSRG_POST_ZOOM_PROBS) {
        set_error("bad mode %d", mode);
        return DSRG_E_INVALID;
    }
    if (n_scales < 1 || (mode == DSRG_POST_ZOOM_PROBS && n_scales != 1) || !scores || !hs || !ws || !result ||
        (smooth && (!image || !p)) || n_sel < 0 || n_sel > DSRG_MAX_LABELS_WIDE || (n_sel > 0 && !labels_sel)) {
        set_error("bad argument");
        return DSRG_E_INVALID;
    }
    LabelSel sel;
    sel.n = n_sel ? n_sel : e->M;
    for (int k = 0; k < sel.n; k++) {
        sel.id[k] = n_sel ? labels_sel[k] : k;
        if (sel.id[k] < 0 || sel.id[k] >= e->M) {
            set_error("selected label %d outside [0, %d)", sel.id[k], e->M);
            return DSRG_E_INVALID;
        }
    }
    for (int k = 0; k < n_scales; k++)
        if (!scores[k] || hs[k] < 1 || ws[k] < 1 || (long long)hs[k] * ws[k] > e->Ncap) {
            set_error("score map %d: bad pointer or size %dx%d (capacity %d pixels)", k, hs[k], ws[k], e->Ncap);
            return DSRG_E_INVALID;
        }
    int rc = ensure_staging(e);
    if (rc) return rc;
    // the whole post-processing of one image as one graph per (shape, score sizes, options): the evaluation tools
    // meet the same few dozen image sizes over and over (api.cu:post_pass_needs_spatial)
    const bool rebuild = smooth && post_pass_needs_spatial(e, p);
    GraphKey key;
    key.add(6).add(e->H).add(e->W).add(mode).add(n_scales).add(image).add(eps).add(smooth).add(result).add(probs_out).add(rebuild);
    for (int k = 0; k < n_scales; k++) key.add(scores[k]).add(hs[k]).add(ws[k]);
    if (smooth) key.add(*p);
    for (int k = 0; k < sel.n; k++) key.add(sel.id[k]);
    if (rebuild) e->sp_valid = false;
    rc = run_pass(e, s, key, true, [&]() { return predict_mask_body(e, mode, n_scales, scores, hs, ws, image, eps, smooth, p, sel, result, probs_out, s); });
    if (smooth) post_pass_done(e, p, 1, rc);
    return rc;
}

static int grow_raw(Engine *e, size_t need) {
    if (need <= e->st_raw_cap) return DSRG_OK;
    cudaFree(e->st_raw);  // synchronises with anything still reading it
    e->st_raw = nullptr;
    e->st_raw_cap = 0;
    int rc = dalloc(e, &e->st_raw, need);
    if (rc) return rc;
    e->st_raw_cap = need;
    return DSRG_OK;
}

}  // namespace dsrg

using namespace dsrg;

extern "C" int dsrg_zoom_scores_dev(dsrg_engine *h, const float *scores_dev, int hi, int wi, float *out_dev,
                                    int accumulate, void *stream) {
    Engine *e = (Engine *)h;
    DeviceScope dev_scope(e);
    int rc = check_batch(e, 1);
    if (rc) return rc;
    StreamScope stream_scope(e, (cudaStream_t)stream);
    if (!scores_dev || !out_dev || hi < 1 || wi < 1) {
        set_error("bad argument");
        return DSRG_E_INVALID;
    }
    return zoom_scores(e, scores_dev, hi, wi, out_dev, accumulate, (cudaStream_t)stream);
}

extern "C" int dsrg_zoom_scores_host(dsrg_engine *h, const float *scores, int hi, int wi, float *out,
                                     int accumulate) {
    Engine *e = (Engine *)h;
    DeviceScope dev_scope(e);
    int rc = check_batch(e, 1);
    if (rc) return rc;
    if (!scores || !out || hi < 1 || wi < 1) {
        set_error("bad argument");
        return DSRG_E_INVALID;
    }
    if ((rc = ensure_staging(e))) return rc;
    const size_t nin = (size_t)e->M * hi * wi, nout = (size_t)e->N * e->M;
    if ((rc = grow_raw(e, nin))) return rc;
    cudaStream_t s = e->own_stream;
    StreamScope stream_scope(e, s);
    DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_raw, scores, nin * sizeof(float), cudaMemcpyHostToDevice, s));
    if (accumulate)
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, out, nout * sizeof(float), cudaMemcpyHostToDevice, s));
    if ((rc = zoom_scores(e, e->st_raw, hi, wi, e->st_unary, accumulate, s))) return rc;
    DSRG_CUDA_TRY(cudaMemcpyAsync(out, e->st_unary, nout * sizeof(float), cudaMemcpyDeviceToHost, s));
    DSRG_CUDA_TRY(cudaStreamSynchronize(s));
    return DSRG_OK;
}

extern "C" int dsrg_predict_mask_dev(dsrg_engine *h, int mode, int n_scales, const float *const *scores_dev,
                                     const int *hs, const int *ws, const uint8_t *image_dev, float eps,
                                     int smooth, const dsrg_crf_params *params, const int32_t *labels_sel,
                                     int n_sel, int32_t *result_out_dev, float *probs_out_dev, void *stream) {
    Engine *e = (Engine *)h;
    DeviceScope dev_scope(e);
    int rc = check_batch(e, 1);
    if (rc) return rc;
    StreamScope stream_scope(e, (cudaStream_t)stream);
    return predict_mask(e, mode, n_scales, scores_dev, hs, ws, image_dev, eps, smooth, params, labels_sel, n_sel,
                        result_out_dev, probs_out_dev, (cudaStream_t)stream);
}

extern "C" int dsrg_predict_mask_host(dsrg_engine *h, int mode, int n_scales, const float *const *scores,
                                      const int *hs, const int *ws, const uint8_t *image, float eps, int smooth,
                                      const dsrg_crf_params *params, const int32_t *labels_sel, int n_sel,
                                      int32_t *result_out, float *probs_out) {
    Engine *e = (Engine *)h;
    DeviceScope dev_scope(e);
    int rc = check_batch(e, 1);
    if (rc) return rc;
    if (n_scales < 1 || n_scales > 16 || !scores || !hs || !ws || !result_out || (smooth && !image)) {
        set_error("bad argument");
        return DSRG_E_INVALID;
    }
    if ((rc = ensure_staging(e))) return rc;
    size_t total = 0;
    for (int k = 0; k < n_scales; k++) {
        if (!scores[k] || hs[k] < 1 || ws[k] < 1) {
            set_error("score map %d: bad pointer or size", k);
            return DSRG_E_INVALID;
        }
        total += (size_t)e->M * hs[k] * ws[k];
    }
    if ((rc = grow_raw(e, total))) return rc;
    cudaStream_t s = e->own_stream;
    StreamScope stream_scope(e, s);
    const float *dptr[16];
    size_t at = 0;
    for (int k = 0; k < n_scales; k++) {
        const size_t n = (size_t)e->M * hs[k] * ws[k];
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_raw + at, scores[k], n * sizeof(float), cudaMemcpyHostToDevice, s));
        dptr[k] = e->st_raw + at;
        at += n;
    }
    if (smooth)
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_image, image, (size_t)e->N * 3, cudaMemcpyHostToDevice, s));
    if ((rc = predict_mask(e, mode, n_scales, dptr, hs, ws, e->st_image, eps, smooth, params, labels_sel, n_sel,
                           e->st_lmap, probs_out ? e->st_out : nullptr, s)))
        return rc;
    DSRG_CUDA_TRY(cudaMemcpyAsync(result_out, e->st_lmap, (size_t)e->N * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (probs_out)
        DSRG_CUDA_TRY(cudaMemcpyAsync(probs_out, e->st_out, (size_t)e->N * e->M * sizeof(float),
                                      cudaMemcpyDeviceToHost, s));
    DSRG_CUDA_TRY(cudaStreamSynchronize(s));
    return DSRG_OK;
}
