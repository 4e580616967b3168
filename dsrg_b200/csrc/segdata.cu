// ImageSegDataLayer.forward on the device (pylayers/pylayers/layer.py:51-61), the stage-2 training input of
// training/experiment/seed_mc/train-f.prototxt: per image, SimpleTransformer.preprocess(image, label) (:169-236)
//   image = float32(image); image -= mean; image *= scale                 float64 subtract, float32 multiply
//   pad_h, pad_w = max(crop - label.shape, 0)                              bottom and right, from the label's shape
//   img_pad = copyMakeBorder(image, 0.0); label_pad = copyMakeBorder(label, saturate_cast<uchar>(ignore_label))
//   image, label = img_pad[h_off:+crop_h, w_off:+crop_w], label_pad[...]  CHW float32, label float32
//   if mirror and flip == -1: image, label = image[:, :, ::-1], label[:, ::-1]
// and the two other paths of SimpleTransformer with the same arithmetic: preprocess(image) without a label (padding
// from the image's shape, :179-199) and pre_test_image (channels swapped before the mean, no scale, :147-167).
// Decoding and the random draws (shuffle, the two randints, the mirror) stay on the host, in the reference's order;
// the caller passes the offsets and flips.
#include <algorithm>
#include <climits>
#include <vector>

#include "common.cuh"

namespace dsrg {

// One entry per image, in the staging buffer st_idx, so B is bounded by the engine only.
struct SegImage {
    const uint8_t *im;   // [Hi][Wi][3] uint8, as cv2.imread(..., IMREAD_COLOR) returns it (BGR)
    const uint8_t *lab;  // [Hl][Wl] uint8, as cv2.imread(..., IMREAD_GRAYSCALE) returns it; NULL without labels
    int Hi, Wi, Hl, Wl;
    int h_off, w_off;    // top-left corner of the crop window in the padded arrays
    int flip;            // 1: the window is read right to left (the mirror)
};

// one thread per output pixel (b, y, x): the three channels of the image top and, when labels_out is given, the
// label.  Blocks [b * per_image, (b + 1) * per_image) belong to image b.  Outside the unpadded arrays the image
// reads 0.0 (padding after the mean and the scale) and the label the pad byte.
__global__ void __launch_bounds__(kThreads)
k_seg_data(const SegImage *__restrict__ src, int per_image, int h, int w, double m0, double m1, double m2,
           float scale, int swap_rb, float pad, float *__restrict__ images_out, float *__restrict__ labels_out) {
    const int b = blockIdx.x / per_image;
    const int pix = (blockIdx.x - b * per_image) * blockDim.x + threadIdx.x;
    if (pix >= h * w) return;
    const SegImage s = src[b];
    const int y = pix / w, x = pix - y * w;
    const int r = s.h_off + y, c = s.w_off + (s.flip ? w - 1 - x : x);
    const size_t plane = (size_t)h * w;
    float *o = images_out + (size_t)b * 3 * plane + pix;
    float v0 = 0.0f, v1 = 0.0f, v2 = 0.0f;
    if (r < s.Hi && c < s.Wi) {
        const uint8_t *p = s.im + ((size_t)r * s.Wi + c) * 3;
        const int c0 = swap_rb ? 2 : 0;  // pre_test_image: image[:, :, [2, 1, 0]] before the mean
        v0 = __fmul_rn((float)((double)p[c0] - m0), scale);
        v1 = __fmul_rn((float)((double)p[1] - m1), scale);
        v2 = __fmul_rn((float)((double)p[2 - c0] - m2), scale);
    }
    o[0] = v0;
    o[plane] = v1;
    o[2 * plane] = v2;
    if (labels_out)
        labels_out[(size_t)b * plane + pix] =
            (r < s.Hl && c < s.Wl) ? (float)s.lab[(size_t)r * s.Wl + c] : pad;
}

// Per-image arguments, read once check_batch has bounded B: pointers non-NULL, sizes >= 1, offsets >= 0, and the
// window inside the padded image and the padded label.  The padding is crop - size at the bottom and right, from the
// label's size (from the image's without labels); the same rows and columns are added to the image.  A window that
// leaves the padded image is where the reference's slice comes back short and numpy refuses to store it.
static bool seg_images_ok(int B, const uint8_t *const *images, const int *Hs, const int *Ws,
                          const uint8_t *const *labels, const int *Hl, const int *Wl, const int *h_off,
                          const int *w_off, int crop_h, int crop_w) {
    for (int b = 0; b < B; b++) {
        if (!images[b] || Hs[b] < 1 || Ws[b] < 1 || (labels && (!labels[b] || Hl[b] < 1 || Wl[b] < 1))) {
            set_error("bad argument: image %d (NULL pointer or size out of range)", b);
            return false;
        }
        const long long ph = std::max(0, crop_h - (labels ? Hl[b] : Hs[b]));
        const long long pw = std::max(0, crop_w - (labels ? Wl[b] : Ws[b]));
        long long rows = Hs[b] + ph, cols = Ws[b] + pw;
        if (labels) {
            rows = std::min(rows, Hl[b] + ph);
            cols = std::min(cols, Wl[b] + pw);
        }
        if (h_off[b] < 0 || w_off[b] < 0 || h_off[b] + (long long)crop_h > rows ||
            w_off[b] + (long long)crop_w > cols) {
            set_error("bad argument: image %d: the %d x %d window at (%d, %d) leaves the padded %lld x %lld arrays",
                      b, crop_h, crop_w, h_off[b], w_off[b], rows, cols);
            return false;
        }
    }
    return true;
}

static std::vector<SegImage> seg_table(int B, const uint8_t *const *images, const int *Hs, const int *Ws,
                                       const uint8_t *const *labels, const int *Hl, const int *Wl,
                                       const int *h_off, const int *w_off, const int32_t *flip) {
    std::vector<SegImage> t(B);
    for (int b = 0; b < B; b++)
        t[b] = {images[b], labels ? labels[b] : nullptr, Hs[b], Ws[b], labels ? Hl[b] : 0, labels ? Wl[b] : 0,
                h_off[b], w_off[b], flip ? (flip[b] != 0) : 0};
    return t;
}

static int seg_data(Engine *e, int B, const std::vector<SegImage> &table, int crop_h, int crop_w, const double *mean,
                    float scale, int swap_rb, int pad, float *images_out, float *labels_out, cudaStream_t s) {
    const int per_image = cdiv((long long)crop_h * crop_w, kThreads);
    if ((long long)per_image * B > INT_MAX) {
        set_error("bad argument: %d images of %d x %d pixels", B, crop_h, crop_w);
        return DSRG_E_INVALID;
    }
    if (int rc = grow_staging(e, (void **)&e->st_idx, &e->st_idx_cap, sizeof(SegImage) * B)) return rc;
    const SegImage *d_table = (const SegImage *)e->st_idx;
    // pageable source: the copy is staged before the call returns, `table` may die afterwards
    DSRG_CUDA_TRY(cudaMemcpyAsync((void *)d_table, table.data(), sizeof(SegImage) * B, cudaMemcpyHostToDevice, s));
    DSRG_LAUNCH(e, T_ANNOT, s,
                k_seg_data<<<per_image * B, kThreads, 0, s>>>(d_table, per_image, crop_h, crop_w, mean[0], mean[1],
                                                             mean[2], scale, swap_rb != 0, (float)pad, images_out,
                                                             labels_out));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

}  // namespace dsrg

using namespace dsrg;

// pointers and sizes that do not depend on the batch; the per-image ones are read in the body (seg_images_ok), once
// check_batch has bounded B.  With labels, Hl, Wl and labels_out are required; without, they are not read.
static bool seg_args_ok(const void *images, const int *Hs, const int *Ws, const void *labels, const int *Hl,
                        const int *Wl, const int *h_off, const int *w_off, int crop_h, int crop_w, const double *mean,
                        int pad, const float *images_out, const float *labels_out) {
    return images && Hs && Ws && h_off && w_off && mean && images_out && (!labels || (Hl && Wl && labels_out)) &&
           crop_h >= 1 && crop_w >= 1 && (long long)crop_h * crop_w <= INT_MAX && pad >= 0 && pad <= 255;
}

extern "C" int dsrg_seg_data_forward_dev(dsrg_engine *h, const uint8_t *const *images_dev, const int *Hs,
                                         const int *Ws, const uint8_t *const *labels_dev, const int *Hl,
                                         const int *Wl, int B, const int *h_off, const int *w_off,
                                         const int32_t *flip, int crop_h, int crop_w, const double *mean,
                                         float scale, int swap_rb, int pad_label, float *images_out_dev,
                                         float *labels_out_dev, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    const bool ok = seg_args_ok(images_dev, Hs, Ws, labels_dev, Hl, Wl, h_off, w_off, crop_h, crop_w, mean,
                                pad_label, images_out_dev, labels_out_dev);
    return dev_call(h, B, s, ok, [&](Engine *e) {
        if (!seg_images_ok(B, images_dev, Hs, Ws, labels_dev, Hl, Wl, h_off, w_off, crop_h, crop_w))
            return DSRG_E_INVALID;
        return seg_data(e, B, seg_table(B, images_dev, Hs, Ws, labels_dev, Hl, Wl, h_off, w_off, flip), crop_h,
                        crop_w, mean, scale, swap_rb, pad_label, images_out_dev,
                        labels_dev ? labels_out_dev : nullptr, s);
    });
}

extern "C" int dsrg_seg_data_forward_host(dsrg_engine *h, const uint8_t *const *images, const int *Hs,
                                          const int *Ws, const uint8_t *const *labels, const int *Hl, const int *Wl,
                                          int B, const int *h_off, const int *w_off, const int32_t *flip,
                                          int crop_h, int crop_w, const double *mean, float scale, int swap_rb,
                                          int pad_label, float *images_out, float *labels_out) {
    const bool ok = seg_args_ok(images, Hs, Ws, labels, Hl, Wl, h_off, w_off, crop_h, crop_w, mean, pad_label,
                                images_out, labels_out);
    return host_call(h, B, ok, false, [&](Engine *e, cudaStream_t s) {
        if (!seg_images_ok(B, images, Hs, Ws, labels, Hl, Wl, h_off, w_off, crop_h, crop_w)) return DSRG_E_INVALID;
        // st_prep: [image top B x 3 x crop float32][label top B x crop float32][image 0][label 0][image 1]..., each
        // part padded to 256 bytes.  A buffer of its own: dsrg_predict_mask_host's graph keys hold the address of
        // st_raw, and growing st_raw here would move it
        auto padded = [](size_t n) { return (n + 255) / 256 * 256; };
        const size_t plane = (size_t)crop_h * crop_w;
        const size_t im_out = padded((size_t)B * 3 * plane * sizeof(float));
        const size_t lab_out = labels ? padded((size_t)B * plane * sizeof(float)) : 0;
        size_t total = im_out + lab_out;
        for (int b = 0; b < B; b++)
            total += padded((size_t)Hs[b] * Ws[b] * 3) + (labels ? padded((size_t)Hl[b] * Wl[b]) : 0);
        if (int rc = grow_staging(e, (void **)&e->st_prep, &e->st_prep_cap, total)) return rc;
        float *d_im_out = (float *)e->st_prep;
        float *d_lab_out = labels ? (float *)(e->st_prep + im_out) : nullptr;
        std::vector<const uint8_t *> d_im(B), d_lab(labels ? B : 0);
        uint8_t *at = e->st_prep + im_out + lab_out;
        for (int b = 0; b < B; b++) {
            const size_t bytes = (size_t)Hs[b] * Ws[b] * 3;
            DSRG_CUDA_TRY(cudaMemcpyAsync(at, images[b], bytes, cudaMemcpyHostToDevice, s));
            d_im[b] = at;
            at += padded(bytes);
            if (labels) {
                const size_t lbytes = (size_t)Hl[b] * Wl[b];
                DSRG_CUDA_TRY(cudaMemcpyAsync(at, labels[b], lbytes, cudaMemcpyHostToDevice, s));
                d_lab[b] = at;
                at += padded(lbytes);
            }
        }
        if (int rc = seg_data(e, B, seg_table(B, d_im.data(), Hs, Ws, labels ? d_lab.data() : nullptr, Hl, Wl,
                                              h_off, w_off, flip),
                              crop_h, crop_w, mean, scale, swap_rb, pad_label, d_im_out, d_lab_out, s))
            return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(images_out, d_im_out, (size_t)B * 3 * plane * sizeof(float),
                                      cudaMemcpyDeviceToHost, s));
        if (labels)
            DSRG_CUDA_TRY(cudaMemcpyAsync(labels_out, d_lab_out, (size_t)B * plane * sizeof(float),
                                          cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}
