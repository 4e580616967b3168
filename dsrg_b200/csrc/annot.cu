// AnnotationLayer.forward on the device (SURVEY.md 8f rank 4): the step that feeds the path,
// pylayers/pylayers/pylayers.py:369-387:
//   top[0].data[...] = 0; top[1].data[...] = 0; top[2].data[...] = bottom[1].data        :371-373
//   top[0].data[i,0,0,0] = 1; top[0].data[i,0,0,labels_i] = 1                               :377-379
//   top[1].data[i, cues_i[0], cues_i[1], cues_i[2]] = 1                                      :381-382
//   if mirror: flip = choice(2)*2-1; top[1].data[i] = top[1].data[i,:,:,::flip]; same for top[2]   :384-387
// The pickle and the random draw stay on the host (the caller passes the index lists and the flip
// flags); the dense planes are produced in HBM, where dsrg_dsrg_forward_dev reads them.
//
// AnnotationLayerCOCO.forward (pylayers.py:432-512) below: decoded images and label maps in, the three tops out.
#include <climits>
#include <vector>

#include "common.cuh"
#include "zoom.cuh"

namespace dsrg {

__global__ void __launch_bounds__(kThreads)
k_annot_tags(const int32_t *tag_off, const int32_t *tags, float *labels, int M) {
    const int b = blockIdx.x;
    float *row = labels + (size_t)b * M;
    for (int l = threadIdx.x; l < M; l += blockDim.x) row[l] = l == 0 ? 1.0f : 0.0f;
    __syncthreads();
    for (int k = tag_off[b] + threadIdx.x; k < tag_off[b + 1]; k += blockDim.x) {
        int t = tags[k];
        if (t < 0) t += M;
        row[t] = 1.0f;
    }
}

// one thread per cue entry; `img` = image of the entry (entries are grouped by image)
__global__ void __launch_bounds__(kThreads)
k_annot_scatter(const int32_t *cue_off, const int32_t *idx, long long ktot, const int32_t *flip, float *cues,
                int B, int M, int H, int W) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= ktot) return;
    int lo = 0, hi = B;  // largest b with cue_off[b] <= k
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (cue_off[mid] <= k) lo = mid; else hi = mid;
    }
    int c = idx[k], y = idx[ktot + k], x = idx[2 * ktot + k];
    if (c < 0) c += M;
    if (y < 0) y += H;
    if (x < 0) x += W;
    if (flip && flip[lo]) x = W - 1 - x;
    cues[(((size_t)lo * M + c) * H + y) * W + x] = 1.0f;
}

__global__ void __launch_bounds__(kThreads)
k_annot_images(const float *in, float *out, const int32_t *flip, long long per_image, int Wi, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int b = (int)(i / per_image);
    const int x = (int)(i % Wi);
    const long long src = (flip && flip[b]) ? i - x + (Wi - 1 - x) : i;
    out[i] = in[src];
}

// host-side validation with numpy's rules: -dim <= index < dim, else IndexError
static int check_indices(const int32_t *v, long long n, int dim, const char *what) {
    for (long long k = 0; k < n; k++)
        if (v[k] < -dim || v[k] >= dim) {
            set_error("index %d is out of bounds for %s with size %d", v[k], what, dim);
            return DSRG_E_INVALID;
        }
    return DSRG_OK;
}

static int annotation_forward(Engine *e, int B, const int32_t *tag_off, const int32_t *tags,
                              const int32_t *cue_off, const int32_t *cue_idx, const int32_t *flip,
                              const float *images_in, int Hi, int Wi, float *labels_out, float *cues_out,
                              float *images_out, cudaStream_t s) {
    const long long nt = tag_off[B], nk = cue_off[B];
    if (tag_off[0] != 0 || cue_off[0] != 0 || nt < 0 || nk < 0 || (nt && !tags) || (nk && !cue_idx)) {
        set_error("bad offsets");
        return DSRG_E_INVALID;
    }
    for (int b = 0; b < B; b++)
        if (tag_off[b + 1] < tag_off[b] || cue_off[b + 1] < cue_off[b]) {
            set_error("offsets must be non-decreasing");
            return DSRG_E_INVALID;
        }
    int rc;
    if ((rc = check_indices(tags, nt, e->M, "the label axis"))) return rc;
    if ((rc = check_indices(cue_idx, nk, e->M, "axis 1 (class)"))) return rc;
    if ((rc = check_indices(cue_idx + nk, nk, e->H, "axis 2 (row)"))) return rc;
    if ((rc = check_indices(cue_idx + 2 * nk, nk, e->W, "axis 3 (column)"))) return rc;
    // device copy of the index lists: [tag_off B+1][cue_off B+1][flip B][tags nt][cue_idx 3*nk]
    const size_t n_ints = (size_t)(2 * (B + 1) + B) + nt + 3 * nk;
    if ((rc = grow_staging(e, (void **)&e->st_idx, &e->st_idx_cap, n_ints * sizeof(int32_t)))) return rc;
    std::vector<int32_t> pack(n_ints);
    int32_t *p = pack.data();
    memcpy(p, tag_off, sizeof(int32_t) * (B + 1));
    memcpy(p + (B + 1), cue_off, sizeof(int32_t) * (B + 1));
    for (int b = 0; b < B; b++) p[2 * (B + 1) + b] = flip ? (flip[b] != 0) : 0;
    if (nt) memcpy(p + 2 * (B + 1) + B, tags, sizeof(int32_t) * nt);
    if (nk) memcpy(p + 2 * (B + 1) + B + nt, cue_idx, sizeof(int32_t) * 3 * nk);
    // pageable source: the copy is staged before the call returns, `pack` may die afterwards
    DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_idx, p, sizeof(int32_t) * n_ints, cudaMemcpyHostToDevice, s));
    const int32_t *d_tag_off = e->st_idx, *d_cue_off = e->st_idx + (B + 1), *d_flip = e->st_idx + 2 * (B + 1);
    const int32_t *d_tags = d_flip + B, *d_idx = d_tags + nt;
    DSRG_CUDA_TRY(cudaMemsetAsync(cues_out, 0, sizeof(float) * (size_t)B * e->M * e->N, s));
    DSRG_LAUNCH(e, T_ANNOT, s, k_annot_tags<<<B, 32, 0, s>>>(d_tag_off, d_tags, labels_out, e->M));
    if (nk)
        DSRG_LAUNCH(e, T_ANNOT, s,
                    k_annot_scatter<<<cdiv(nk, kThreads), kThreads, 0, s>>>(d_cue_off, d_idx, nk, flip ? d_flip : nullptr,
                                                                          cues_out, B, e->M, e->H, e->W));
    if (images_out) {
        const long long per = 3ll * Hi * Wi, n = per * B;
        DSRG_LAUNCH(e, T_ANNOT, s,
                    k_annot_images<<<cdiv(n, kThreads), kThreads, 0, s>>>(images_in, images_out, flip ? d_flip : nullptr,
                                                                        per, Wi, n));
    }
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

// ---- AnnotationLayerCOCO (pylayers.py:477-512), per image of the batch ----
//   image = zoom(image.astype('float32'), (new_h/H, new_w/W, 1.0), order=1)[:, :, [2, 1, 0]] - mean; CHW
//   cues[v, y, x] = 1 for every label pixel with v != ignore_label                           (:494-498)
//   if mirror: image, cues = image[:, :, ::-1], cues[:, :, ::-1]                              (:500-503)
//   image_label[v] = 1 for every value of np.unique(label) other than ignore_label            (:505-510)
// One entry of this table per image, in the staging buffer st_idx: B is bounded by the engine, not by the size
// of a kernel parameter.
struct CocoImage {
    const uint8_t *im;  // [H][W][3] uint8, as cv2.imread(..., IMREAD_COLOR) returns it (BGR)
    int H, W;
    int flip;           // 1: mirror along the width
};

// one thread per output pixel; blocks [b * per_image, (b + 1) * per_image) belong to image b
__global__ void __launch_bounds__(kThreads)
k_coco_images(const CocoImage *__restrict__ src, int per_image, int h, int w, double m0, double m1, double m2,
              float *out) {
    const int b = blockIdx.x / per_image;
    const int pix = (blockIdx.x - b * per_image) * blockDim.x + threadIdx.x;
    if (pix >= h * w) return;
    const CocoImage s = src[b];
    const int oy = pix / w, ox = pix - oy * w;
    const ZoomTap tap = zoom_tap(oy, s.flip ? w - 1 - ox : ox, s.H, s.W, h, w);  // the mirror reads column w-1-ox
    const double mean[3] = {m0, m1, m2};
    net_input_pixel(s.im, s.W, tap, mean, out + (size_t)b * 3 * h * w, h, w, pix);
}

// one thread per cue element [b][k][pixel]: 1 where the (mirrored) label map holds k and k is not ignored.  A value
// >= K matches no plane, so it is never written anywhere.
__global__ void __launch_bounds__(kThreads)
k_coco_cues(const uint8_t *__restrict__ lab, const CocoImage *__restrict__ src, int K, int H, int W, int ignore,
            float *cues, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int N = H * W;
    const long long bk = i / N;
    const int pix = (int)(i - bk * N);
    const int b = (int)(bk / K), k = (int)(bk - (long long)b * K);
    const int y = pix / W;
    int x = pix - y * W;
    if (src[b].flip) x = W - 1 - x;
    const int v = lab[(size_t)b * N + (size_t)y * W + x];
    cues[i] = (v == k && v != ignore) ? 1.0f : 0.0f;
}

// one CTA per image: the presence row [b][K], and in bad[b] the raster index of the first pixel whose value is
// neither ignore_label nor below K (-1: none)
__global__ void __launch_bounds__(kThreads)
k_coco_tags(const uint8_t *__restrict__ lab, int N, int K, int ignore, float *labels, int32_t *bad) {
    __shared__ int seen[256];
    __shared__ unsigned first_bad;
    const int b = blockIdx.x;
    for (int v = threadIdx.x; v < 256; v += blockDim.x) seen[v] = 0;
    if (threadIdx.x == 0) first_bad = 0xFFFFFFFFu;
    __syncthreads();
    const uint8_t *l = lab + (size_t)b * N;
    for (int p = threadIdx.x; p < N; p += blockDim.x) {
        const int v = l[p];
        if (v == ignore) continue;
        if (v < K)
            seen[v] = 1;
        else
            atomicMin(&first_bad, (unsigned)p);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < K; k += blockDim.x) labels[(size_t)b * K + k] = seen[k] ? 1.0f : 0.0f;
    if (bad && threadIdx.x == 0) bad[b] = (int32_t)first_bad;
}

// Per-image arguments, read once the batch size is known to be in range.  Every size >= 1, every plane below 2^31
// pixels, and every image pointer non-NULL.
static bool coco_images_ok(int B, const uint8_t *const *images, const int *Hs, const int *Ws) {
    for (int b = 0; b < B; b++)
        if (!images[b] || Hs[b] < 1 || Ws[b] < 1 || (long long)Hs[b] * Ws[b] > INT_MAX) {
            set_error("bad argument: image %d (NULL pointer or size out of range)", b);
            return false;
        }
    return true;
}

static int annotation_coco(Engine *e, int B, const std::vector<CocoImage> &table, const uint8_t *label_maps,
                           int new_h, int new_w, const double *mean, int ignore, float *labels_out, float *cues_out,
                           float *images_out, int32_t *bad_out, cudaStream_t s) {
    const int per_image = cdiv((long long)new_h * new_w, kThreads);
    if ((long long)per_image * B > INT_MAX) {
        set_error("bad argument: %d images of %d x %d pixels", B, new_h, new_w);
        return DSRG_E_INVALID;
    }
    if (int rc = grow_staging(e, (void **)&e->st_idx, &e->st_idx_cap, sizeof(CocoImage) * B)) return rc;
    const CocoImage *d_table = (const CocoImage *)e->st_idx;
    // pageable source: the copy is staged before the call returns, `table` may die afterwards
    DSRG_CUDA_TRY(cudaMemcpyAsync((void *)d_table, table.data(), sizeof(CocoImage) * B, cudaMemcpyHostToDevice, s));
    const long long ncue = (long long)B * e->M * e->N;
    DSRG_LAUNCH(e, T_ANNOT, s,
                k_coco_images<<<per_image * B, kThreads, 0, s>>>(d_table, per_image, new_h, new_w, mean[0], mean[1],
                                                                 mean[2], images_out));
    DSRG_LAUNCH(e, T_ANNOT, s,
                k_coco_cues<<<cdiv(ncue, kThreads), kThreads, 0, s>>>(label_maps, d_table, e->M, e->H, e->W, ignore,
                                                                     cues_out, ncue));
    DSRG_LAUNCH(e, T_ANNOT, s, k_coco_tags<<<B, kThreads, 0, s>>>(label_maps, e->N, e->M, ignore, labels_out, bad_out));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

}  // namespace dsrg

using namespace dsrg;

// the pointers every call needs, and the image pair when the images are copied
static bool annot_args_ok(const int32_t *tag_off, const int32_t *cue_off, const float *images_in, int Hi, int Wi,
                          const float *labels_out, const float *cues_out, const float *images_out) {
    return tag_off && cue_off && labels_out && cues_out && (!images_out || (images_in && Hi >= 1 && Wi >= 1));
}

extern "C" int dsrg_annotation_forward_dev(dsrg_engine *h, int B, const int32_t *tag_offsets, const int32_t *tags,
                                           const int32_t *cue_offsets, const int32_t *cue_idx, const int32_t *flip,
                                           const float *images_in_dev, int Hi, int Wi, float *labels_out_dev,
                                           float *cues_out_dev, float *images_out_dev, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    // the mirror reads and writes whole rows: the two image buffers must be distinct
    const bool ok = annot_args_ok(tag_offsets, cue_offsets, images_in_dev, Hi, Wi, labels_out_dev, cues_out_dev,
                                  images_out_dev) && (!images_out_dev || images_in_dev != images_out_dev);
    return dev_call(h, B, s, ok, [&](Engine *e) {
        return annotation_forward(e, B, tag_offsets, tags, cue_offsets, cue_idx, flip, images_in_dev, Hi, Wi,
                                  labels_out_dev, cues_out_dev, images_out_dev, s);
    });
}

extern "C" int dsrg_annotation_forward_host(dsrg_engine *h, int B, const int32_t *tag_offsets, const int32_t *tags,
                                            const int32_t *cue_offsets, const int32_t *cue_idx, const int32_t *flip,
                                            const float *images_in, int Hi, int Wi, float *labels_out,
                                            float *cues_out, float *images_out) {
    const bool ok = annot_args_ok(tag_offsets, cue_offsets, images_in, Hi, Wi, labels_out, cues_out, images_out);
    return host_call(h, B, ok, false, [&](Engine *e, cudaStream_t s) {
        float *d_in = nullptr, *d_out = nullptr;
        const size_t nimg = images_out ? (size_t)B * 3 * Hi * Wi : 0;
        if (images_out) {
            if (int rc = grow_staging(e, (void **)&e->st_raw, &e->st_raw_cap, 2 * nimg * sizeof(float))) return rc;
            d_in = e->st_raw;
            d_out = e->st_raw + nimg;
            DSRG_CUDA_TRY(cudaMemcpyAsync(d_in, images_in, nimg * sizeof(float), cudaMemcpyHostToDevice, s));
        }
        if (int rc = annotation_forward(e, B, tag_offsets, tags, cue_offsets, cue_idx, flip, d_in, Hi, Wi,
                                        e->st_labels, e->st_cues, d_out, s))
            return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(labels_out, e->st_labels, sizeof(float) * (size_t)B * e->M, cudaMemcpyDeviceToHost, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(cues_out, e->st_cues, sizeof(float) * (size_t)B * e->M * e->N, cudaMemcpyDeviceToHost, s));
        if (images_out)
            DSRG_CUDA_TRY(cudaMemcpyAsync(images_out, d_out, nimg * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}

// pointers and sizes that do not depend on the batch; the per-image ones are read in the body (coco_images_ok),
// once check_batch has bounded B
static bool coco_args_ok(const void *images, const int *Hs, const int *Ws, const void *label_maps, int new_h,
                         int new_w, const double *mean, const float *labels_out, const float *cues_out,
                         const float *images_out) {
    return images && Hs && Ws && label_maps && mean && labels_out && cues_out && images_out && new_h >= 1 &&
           new_w >= 1 && (long long)new_h * new_w <= INT_MAX;
}

static std::vector<CocoImage> coco_table(int B, const uint8_t *const *images, const int *Hs, const int *Ws,
                                         const int32_t *flip) {
    std::vector<CocoImage> t(B);
    for (int b = 0; b < B; b++) t[b] = {images[b], Hs[b], Ws[b], flip ? (flip[b] != 0) : 0};
    return t;
}

extern "C" int dsrg_annotation_coco_forward_dev(dsrg_engine *h, const uint8_t *const *images_dev, const int *Hs,
                                                const int *Ws, int B, const uint8_t *label_maps_dev,
                                                const int32_t *flip, int new_h, int new_w, const double *mean_pixel,
                                                int ignore_label, float *labels_out_dev, float *cues_out_dev,
                                                float *images_out_dev, int32_t *bad_out_dev, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    const bool ok = coco_args_ok(images_dev, Hs, Ws, label_maps_dev, new_h, new_w, mean_pixel, labels_out_dev,
                                 cues_out_dev, images_out_dev);
    return dev_call(h, B, s, ok, [&](Engine *e) {
        if (!coco_images_ok(B, images_dev, Hs, Ws)) return DSRG_E_INVALID;
        return annotation_coco(e, B, coco_table(B, images_dev, Hs, Ws, flip), label_maps_dev, new_h, new_w,
                               mean_pixel, ignore_label, labels_out_dev, cues_out_dev, images_out_dev, bad_out_dev, s);
    });
}

extern "C" int dsrg_annotation_coco_forward_host(dsrg_engine *h, const uint8_t *const *images, const int *Hs,
                                                 const int *Ws, int B, const uint8_t *label_maps,
                                                 const int32_t *flip, int new_h, int new_w,
                                                 const double *mean_pixel, int ignore_label, float *labels_out,
                                                 float *cues_out, float *images_out) {
    const bool ok = coco_args_ok(images, Hs, Ws, label_maps, new_h, new_w, mean_pixel, labels_out, cues_out,
                                 images_out);
    return host_call(h, B, ok, false, [&](Engine *e, cudaStream_t s) {
        if (!coco_images_ok(B, images, Hs, Ws)) return DSRG_E_INVALID;
        // numpy's IndexError of cues[v, x, y] = 1 (pylayers.py:498), raised at the first such pixel in the
        // reference's order (image by image, row-major), before anything is copied or launched
        const size_t N = (size_t)e->N;
        for (int b = 0; b < B; b++)
            for (size_t p = 0; p < N; p++) {
                const int v = label_maps[b * N + p];
                if (v != ignore_label && v >= e->M) {
                    set_error("index %d is out of bounds for axis 0 with size %d", v, e->M);
                    return DSRG_E_INVALID;
                }
            }
        // st_prep: [network input B x 3 x new_h x new_w float32][label maps, padded to 256 bytes][image 0, padded]...
        // A buffer of its own: dsrg_predict_mask_host's graph keys hold the address of st_raw, and growing st_raw
        // here would move it
        const size_t out_bytes = ((size_t)B * 3 * new_h * new_w * sizeof(float) + 255) / 256 * 256;
        const size_t lab_bytes = (B * N + 255) / 256 * 256;
        size_t total = out_bytes + lab_bytes;
        for (int b = 0; b < B; b++) total += ((size_t)Hs[b] * Ws[b] * 3 + 255) / 256 * 256;
        if (int rc = grow_staging(e, (void **)&e->st_prep, &e->st_prep_cap, total)) return rc;
        float *d_out = (float *)e->st_prep;
        uint8_t *d_lab = e->st_prep + out_bytes;
        std::vector<const uint8_t *> d_im(B);
        uint8_t *at = d_lab + lab_bytes;
        DSRG_CUDA_TRY(cudaMemcpyAsync(d_lab, label_maps, B * N, cudaMemcpyHostToDevice, s));
        for (int b = 0; b < B; b++) {
            const size_t bytes = (size_t)Hs[b] * Ws[b] * 3;
            DSRG_CUDA_TRY(cudaMemcpyAsync(at, images[b], bytes, cudaMemcpyHostToDevice, s));
            d_im[b] = at;
            at += (bytes + 255) / 256 * 256;
        }
        if (int rc = annotation_coco(e, B, coco_table(B, d_im.data(), Hs, Ws, flip), d_lab, new_h, new_w, mean_pixel,
                                     ignore_label, e->st_labels, e->st_cues, d_out, nullptr, s))
            return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(labels_out, e->st_labels, sizeof(float) * B * e->M, cudaMemcpyDeviceToHost, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(cues_out, e->st_cues, sizeof(float) * B * e->M * N, cudaMemcpyDeviceToHost, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(images_out, d_out, sizeof(float) * B * 3 * new_h * new_w,
                                      cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}
