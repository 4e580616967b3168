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
//
// One pass serves every entry point: B images of one size (every scale's zoom and the sum in one launch, the batched
// CRF, a per-image label selection read from device memory).  dsrg_predict_mask_{dev,host} are that pass at B = 1,
// their selection written into the engine by the pass; dsrg_zoom_scores_* is its zoom kernel on one scale.
#include "common.cuh"
#include "zoom.cuh"

namespace dsrg {

constexpr int kPostMaxScales = 16;

// one batched network forward per scale: scale k is [B][M][h[k]][w[k]] float32 at p[k]
struct ZoomScales {  // 264 bytes of kernel parameters
    const float *p[kPostMaxScales];
    int h[kPostMaxScales], w[kPostMaxScales];
    int n;
};

// out [B][H][W][M] = sum_k zoom(scores_k[b]), one thread per output element, image b = blockIdx.y.  The float32 sum
// is formed in the order of test-ms.py:97: scale 0 stored, then += each further scale; with `accumulate` every scale
// is added to what out holds (`scores_all += scores`).  Capped at 40 registers, so that 6 CTAs fit on an SM: the
// float64 tap arithmetic is latency-bound (one 81-label scale of a COCO-sized image: 248 us against 256 at 46
// registers, H100 SXM at 700 W).
__global__ void __launch_bounds__(kThreads, 6)
k_zoom_sum_batch(ZoomScales sc, float *__restrict__ out, int M, int Ho, int Wo, int accumulate) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long NM = (long long)Ho * Wo * M;
    if (idx >= NM) return;
    const int b = blockIdx.y, c = (int)(idx % M), pix = (int)(idx / M);
    const int oy = pix / Wo, ox = pix - oy * Wo;
    out += b * NM;
    float acc = accumulate ? out[idx] : 0.f;
#pragma unroll
    for (int k = 0; k < kPostMaxScales; k++) {
        if (k >= sc.n) break;
        const int hi = sc.h[k], wi = sc.w[k];
        const float z = zoom_apply(sc.p[k] + ((size_t)b * M + c) * hi * wi, wi, zoom_tap(oy, ox, hi, wi, Ho, Wo));
        acc = k || accumulate ? __fadd_rn(acc, z) : z;
    }
    out[idx] = acc;
}

static void zoom_sum(Engine *e, int B, const ZoomScales &sc, float *out, int accumulate, cudaStream_t s) {
    const dim3 g(cdiv((long long)e->N * e->M, kThreads), B);
    DSRG_LAUNCH(e, T_POST, s, k_zoom_sum_batch<<<g, kThreads, 0, s>>>(sc, out, e->M, e->H, e->W, accumulate));
}

// softmax over the labels of every pixel of B images of npix pixels: pixel i of image b = blockIdx.y starts at
// b * M * npix + i * ps and its labels are ls apart ([B][M][npix] blob: ls = npix, ps = 1; [B][npix][M] map: ls = 1,
// ps = M).  Mirrors
//   e = np.exp(s - np.max(s)); p = e / np.sum(e)            (float32)
// and, when CLAMPLOG, the clamp at eps followed by np.log; `probs` (optional) receives the clamped p.
template <bool CLAMPLOG>
__global__ void __launch_bounds__(kThreads)
k_post_softmax(const float *in, float *out, float *probs, int npix, int M, long long ls, long long ps,
               float eps) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    const size_t base = (size_t)blockIdx.y * M * npix + (size_t)i * ps;
    const float *s = in + base;
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
                if (probs) probs[base + (size_t)l * ls] = p;
                p = logf(p);
            }
            out[base + (size_t)l * ls] = p;
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
    const size_t base = (size_t)blockIdx.y * M * npix + (size_t)i * ps;
    const float *s = in + base;
    float *o = out + base;
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
            if (probs) probs[base + (size_t)l * ls] = p;
            p = logf(p);
        }
        o[(size_t)l * ls] = p;
    }
}

template <bool CLAMPLOG>
static void post_softmax(Engine *e, const float *in, float *out, float *probs, int B, int npix, long long ls,
                         long long ps, float eps, cudaStream_t s) {
    const dim3 g(cdiv(npix, kThreads), B);
    const int M = e->M;
    if (M > DSRG_MAX_LABELS)
        DSRG_LAUNCH(e, T_POST, s,
                    k_post_softmax_wide<CLAMPLOG><<<g, kThreads, 0, s>>>(in, out, probs, npix, M, ls, ps, eps));
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

// One selection row of k_post_argmax_batch, by value: the per-image entry points take their selection from host
// memory the caller may reuse at once, and a replayed graph or a caller's capture has to write the same ids again.
struct LabelRow {  // 1 KB of kernel parameters
    int32_t id[DSRG_MAX_LABELS_WIDE];
};

__global__ void __launch_bounds__(kThreads) k_post_sel_row(LabelRow row, int32_t *sel, int M) {
    for (int k = threadIdx.x; k < M; k += blockDim.x) sel[k] = row.id[k];
}

// Per (pixel, image b = blockIdx.y): np.argmax (first maximum) over image b's selected labels, result = the label's
// id.  q holds image b at b * M * N: [M][N] (ls = N, ps = 1, the CRF marginals) or [N][M] (ls = 1, ps = M).
// sel: [B][M] label ids, each row ending at its first -1; NULL or an empty row selects every label.  A row with
// an entry outside [0, M) before its -1 is not read past: every pixel of that image gets -1.
__global__ void __launch_bounds__(kThreads)
k_post_argmax_batch(const float *q, int32_t *out, int N, int M, long long ls, long long ps, const int32_t *sel) {
    __shared__ int s_id[DSRG_MAX_LABELS_WIDE];
    __shared__ int s_n;
    const int b = blockIdx.y;
    for (int k = threadIdx.x; k < M; k += blockDim.x) s_id[k] = sel ? sel[(size_t)b * M + k] : k;
    __syncthreads();
    if (threadIdx.x == 0) {
        int n = sel ? 0 : M;  // without a selection there is no row to scan
        while (n < M && s_id[n] != -1) {
            if (s_id[n] < 0 || s_id[n] >= M) {
                n = -1;
                break;
            }
            n++;
        }
        if (n == 0)
            for (int k = 0; k < M; k++) s_id[k] = k;
        s_n = n == 0 ? M : n;
    }
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int n = s_n;
    if (n < 0) {
        out[(size_t)b * N + i] = -1;
        return;
    }
    const float *s = q + (size_t)b * M * N + (size_t)i * ps;
    int arg = s_id[0];
    float best = s[(size_t)arg * ls];
    for (int k = 1; k < n; k++) {
        const int id = s_id[k];
        const float v = s[(size_t)id * ls];
        if (v > best) {
            best = v;
            arg = id;
        }
    }
    out[(size_t)b * N + i] = arg;
}

int crf_core_batch_for_post(Engine *e, int B, const float *unary_hwc, const uint8_t *images,
                            const dsrg_crf_params *p, cudaStream_t s);  // api.cu

// sel: device rows as k_post_argmax_batch reads them, or NULL; row (B = 1): a selection written to st_sel by the pass
static int predict_mask_batch_body(Engine *e, int B, int mode, const ZoomScales &sc, const uint8_t *images, float eps,
                                   int smooth, const dsrg_crf_params *p, const int32_t *sel, const LabelRow *row,
                                   int32_t *result, float *probs_out, cudaStream_t s) {
    const int N = e->N, M = e->M;
    const long long n = (long long)B * N * M;
    float *unary = e->st_unary;                       // [B][H][W][M]
    float *clamped = smooth ? nullptr : (probs_out ? probs_out : e->st_out);
    if (mode == DSRG_POST_SUM_SCORES) {
        zoom_sum(e, B, sc, unary, 0, s);
        post_softmax<true>(e, unary, unary, clamped, B, N, 1, M, eps, s);
    } else {
        const int np = sc.h[0] * sc.w[0];
        float *small = e->st_cues;                    // [B][M][h][w] probabilities at network resolution
        post_softmax<false>(e, sc.p[0], small, nullptr, B, np, np, 1, eps, s);
        ZoomScales zs = sc;
        zs.p[0] = small;
        zoom_sum(e, B, zs, unary, 0, s);
        DSRG_LAUNCH(e, T_POST, s, k_post_clamp_log<<<cdiv(n, kThreads), kThreads, 0, s>>>(unary, unary, clamped, n, eps));
    }
    if (row) {
        DSRG_LAUNCH(e, T_POST, s, k_post_sel_row<<<1, kThreads, 0, s>>>(*row, e->st_sel, M));
        sel = e->st_sel;
    }
    DSRG_CUDA_TRY(cudaGetLastError());
    const dim3 ga(cdiv(N, kThreads), B);
    if (smooth) {
        if (int rc = crf_core_batch_for_post(e, B, unary, images, p, s)) return rc;
        if (probs_out)
            if (int rc = meanfield_export(e, B, probs_out, DSRG_LAYOUT_NHWC, s)) return rc;
        DSRG_LAUNCH(e, T_POST, s, k_post_argmax_batch<<<ga, kThreads, 0, s>>>(e->Qcur, result, N, M, N, 1, sel));
    } else {
        DSRG_LAUNCH(e, T_POST, s, k_post_argmax_batch<<<ga, kThreads, 0, s>>>(clamped, result, N, M, 1, M, sel));
    }
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

// what the batched pass checks before anything is staged or launched (B and the NULL pointers: the prologue)
static int post_batch_check(const Engine *e, int mode, int n_scales, const float *const *scores, const int *hs,
                            const int *ws) {
    if (mode != DSRG_POST_SUM_SCORES && mode != DSRG_POST_ZOOM_PROBS) {
        set_error("bad mode %d", mode);
        return DSRG_E_INVALID;
    }
    if (mode == DSRG_POST_ZOOM_PROBS && n_scales != 1) {
        set_error("DSRG_POST_ZOOM_PROBS takes one score map per image, not %d", n_scales);
        return DSRG_E_INVALID;
    }
    for (int k = 0; k < n_scales; k++)
        if (!scores[k] || hs[k] < 1 || ws[k] < 1 || (long long)hs[k] * ws[k] > e->Ncap) {
            set_error("score map %d: bad pointer or size %dx%d (capacity %d pixels)", k, hs[k], ws[k], e->Ncap);
            return DSRG_E_INVALID;
        }
    return DSRG_OK;
}

static int predict_mask_batch(Engine *e, int B, int mode, int n_scales, const float *const *scores, const int *hs,
                              const int *ws, const uint8_t *images, float eps, int smooth, const dsrg_crf_params *p,
                              const int32_t *sel, const LabelRow *row, int32_t *result, float *probs_out,
                              cudaStream_t s) {
    int rc = post_batch_check(e, mode, n_scales, scores, hs, ws);
    if (rc || (rc = ensure_staging(e))) return rc;
    ZoomScales sc = {};
    sc.n = n_scales;
    for (int k = 0; k < n_scales; k++) {
        sc.p[k] = scores[k];
        sc.h[k] = hs[k];
        sc.w[k] = ws[k];
    }
    // the pass reads sel, so its content is not part of the key: a replay follows what sel holds.  A row is a kernel
    // parameter of the pass, so a replay writes the ids it was captured with: they are part of the key.
    const bool rebuild = smooth && post_pass_needs_spatial(e, p);
    GraphKey key;
    key.add(7).add(B).add(e->H).add(e->W).add(mode).add(n_scales).add(images).add(eps).add(smooth).add(sel)
        .add(result).add(probs_out).add(rebuild).add(row != nullptr);
    for (int k = 0; k < n_scales; k++) key.add(scores[k]).add(hs[k]).add(ws[k]);
    if (smooth) key.add(*p);
    if (row) key.add(*row);
    if (rebuild) e->sp_valid = false;
    rc = run_pass(e, s, key, true, [&]() {
        return predict_mask_batch_body(e, B, mode, sc, images, eps, smooth, p, sel, row, result, probs_out, s);
    });
    if (smooth) post_pass_done(e, p, B, rc);
    return rc;
}

// The *_host entry points: the score maps, the images (when smoothing) and the selection rows in through the
// engine's staging, the pass, the label maps (and probabilities) back.  sel: host [B][M] rows, or NULL.
static int predict_mask_staged(Engine *e, int B, int mode, int n_scales, const float *const *scores, const int *hs,
                               const int *ws, const uint8_t *images, float eps, int smooth, const dsrg_crf_params *p,
                               const int32_t *sel, const LabelRow *row, int32_t *result_out, float *probs_out,
                               cudaStream_t s) {
    const int M = e->M;
    if (int rc = post_batch_check(e, mode, n_scales, scores, hs, ws)) return rc;
    for (int b = 0; sel && b < B; b++)
        for (int k = 0; k < M && sel[(size_t)b * M + k] != -1; k++) {
            const int v = sel[(size_t)b * M + k];
            if (v < 0 || v >= M) {
                set_error("image %d: selected label %d outside [0, %d)", b, v, M);
                return DSRG_E_INVALID;
            }
        }
    size_t total = 0;
    for (int k = 0; k < n_scales; k++) total += (size_t)B * M * hs[k] * ws[k];
    if (int rc = grow_staging(e, (void **)&e->st_raw, &e->st_raw_cap, total * sizeof(float))) return rc;
    if (sel)
        if (int rc = grow_staging(e, (void **)&e->st_idx, &e->st_idx_cap, (size_t)B * M * sizeof(int32_t)))
            return rc;
    const float *dptr[kPostMaxScales];
    size_t at = 0;
    for (int k = 0; k < n_scales; k++) {
        const size_t n = (size_t)B * M * hs[k] * ws[k];
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_raw + at, scores[k], n * sizeof(float), cudaMemcpyHostToDevice, s));
        dptr[k] = e->st_raw + at;
        at += n;
    }
    if (smooth)
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_image, images, (size_t)B * e->N * 3, cudaMemcpyHostToDevice, s));
    if (sel)
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_idx, sel, (size_t)B * M * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    if (int rc = predict_mask_batch(e, B, mode, n_scales, dptr, hs, ws, e->st_image, eps, smooth, p,
                                    sel ? e->st_idx : nullptr, row, e->st_lmap, probs_out ? e->st_out : nullptr, s))
        return rc;
    DSRG_CUDA_TRY(cudaMemcpyAsync(result_out, e->st_lmap, (size_t)B * e->N * sizeof(int32_t),
                                  cudaMemcpyDeviceToHost, s));
    if (probs_out)
        DSRG_CUDA_TRY(cudaMemcpyAsync(probs_out, e->st_out, (size_t)B * e->N * M * sizeof(float),
                                      cudaMemcpyDeviceToHost, s));
    return DSRG_OK;
}

// labels_sel / n_sel of the per-image entry points as one selection row: each id's first occurrence, in the caller's
// order (the arg-max keeps the first strict maximum, so a repeated id never wins again), then -1
static int label_row(const Engine *e, const int32_t *labels_sel, int n_sel, LabelRow *row) {
    bool seen[DSRG_MAX_LABELS_WIDE] = {};
    int n = 0;
    for (int k = 0; k < n_sel; k++) {
        const int v = labels_sel[k];
        if (v < 0 || v >= e->M) {
            set_error("selected label %d outside [0, %d)", v, e->M);
            return DSRG_E_INVALID;
        }
        if (!seen[v]) {
            seen[v] = true;
            row->id[n++] = v;
        }
    }
    for (int k = n; k < DSRG_MAX_LABELS_WIDE; k++) row->id[k] = -1;
    return DSRG_OK;
}

}  // namespace dsrg

using namespace dsrg;

// a predict_mask call's arguments: 1 to kPostMaxScales score maps, their pointers, hs / ws and the result always;
// the image and the CRF parameters when it smooths; the label selection when it has one
static bool post_args_ok(int n_scales, const float *const *scores, const int *hs, const int *ws, const uint8_t *image,
                         int smooth, const dsrg_crf_params *params, const int32_t *labels_sel, int n_sel,
                         const int32_t *result) {
    return n_scales >= 1 && n_scales <= kPostMaxScales && scores && hs && ws && result &&
           (!smooth || (image && params)) && n_sel >= 0 && n_sel <= DSRG_MAX_LABELS_WIDE && (n_sel == 0 || labels_sel);
}

extern "C" int dsrg_zoom_scores_dev(dsrg_engine *h, const float *scores_dev, int hi, int wi, float *out_dev,
                                    int accumulate, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, 1, s, scores_dev && out_dev && hi >= 1 && wi >= 1, [&](Engine *e) {
        zoom_sum(e, 1, {{scores_dev}, {hi}, {wi}, 1}, out_dev, accumulate, s);
        DSRG_CUDA_TRY(cudaGetLastError());
        return DSRG_OK;
    });
}

extern "C" int dsrg_zoom_scores_host(dsrg_engine *h, const float *scores, int hi, int wi, float *out,
                                     int accumulate) {
    return host_call(h, 1, scores && out && hi >= 1 && wi >= 1, false, [&](Engine *e, cudaStream_t s) {
        const size_t nin = (size_t)e->M * hi * wi, nout = (size_t)e->N * e->M;
        if (int rc = grow_staging(e, (void **)&e->st_raw, &e->st_raw_cap, nin * sizeof(float))) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_raw, scores, nin * sizeof(float), cudaMemcpyHostToDevice, s));
        if (accumulate)
            DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, out, nout * sizeof(float), cudaMemcpyHostToDevice, s));
        zoom_sum(e, 1, {{e->st_raw}, {hi}, {wi}, 1}, e->st_unary, accumulate, s);
        DSRG_CUDA_TRY(cudaGetLastError());
        DSRG_CUDA_TRY(cudaMemcpyAsync(out, e->st_unary, nout * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}

extern "C" int dsrg_predict_mask_dev(dsrg_engine *h, int mode, int n_scales, const float *const *scores_dev,
                                     const int *hs, const int *ws, const uint8_t *image_dev, float eps,
                                     int smooth, const dsrg_crf_params *params, const int32_t *labels_sel,
                                     int n_sel, int32_t *result_out_dev, float *probs_out_dev, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    const bool ok = post_args_ok(n_scales, scores_dev, hs, ws, image_dev, smooth, params, labels_sel, n_sel,
                                 result_out_dev);
    return dev_call(h, 1, s, ok, [&](Engine *e) {
        LabelRow row;
        if (int rc = label_row(e, labels_sel, n_sel, &row)) return rc;
        return predict_mask_batch(e, 1, mode, n_scales, scores_dev, hs, ws, image_dev, eps, smooth, params, nullptr,
                                  n_sel ? &row : nullptr, result_out_dev, probs_out_dev, s);
    });
}

extern "C" int dsrg_predict_mask_host(dsrg_engine *h, int mode, int n_scales, const float *const *scores,
                                      const int *hs, const int *ws, const uint8_t *image, float eps, int smooth,
                                      const dsrg_crf_params *params, const int32_t *labels_sel, int n_sel,
                                      int32_t *result_out, float *probs_out) {
    const bool ok = post_args_ok(n_scales, scores, hs, ws, image, smooth, params, labels_sel, n_sel, result_out);
    return host_call(h, 1, ok, false, [&](Engine *e, cudaStream_t s) {
        LabelRow row;
        if (int rc = label_row(e, labels_sel, n_sel, &row)) return rc;
        return predict_mask_staged(e, 1, mode, n_scales, scores, hs, ws, image, eps, smooth, params, nullptr,
                                   n_sel ? &row : nullptr, result_out, probs_out, s);
    });
}

extern "C" int dsrg_predict_mask_batch_dev(dsrg_engine *h, const float *const *scores_dev, const int *hs,
                                           const int *ws, int n_scales, int B, int mode, const uint8_t *images_dev,
                                           float eps, int smooth, const dsrg_crf_params *params,
                                           const int32_t *sel_dev, int32_t *result_out_dev, float *probs_out_dev,
                                           void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    const bool ok = post_args_ok(n_scales, scores_dev, hs, ws, images_dev, smooth, params, nullptr, 0, result_out_dev);
    return dev_call(h, B, s, ok, [&](Engine *e) {
        return predict_mask_batch(e, B, mode, n_scales, scores_dev, hs, ws, images_dev, eps, smooth, params, sel_dev,
                                  nullptr, result_out_dev, probs_out_dev, s);
    });
}

extern "C" int dsrg_predict_mask_batch_host(dsrg_engine *h, const float *const *scores, const int *hs, const int *ws,
                                            int n_scales, int B, int mode, const uint8_t *images, float eps,
                                            int smooth, const dsrg_crf_params *params, const int32_t *sel,
                                            int32_t *result_out, float *probs_out) {
    const bool ok = post_args_ok(n_scales, scores, hs, ws, images, smooth, params, nullptr, 0, result_out);
    return host_call(h, B, ok, false, [&](Engine *e, cudaStream_t s) {
        return predict_mask_staged(e, B, mode, n_scales, scores, hs, ws, images, eps, smooth, params, sel, nullptr,
                                   result_out, probs_out, s);
    });
}
