// Image preprocessing of the Python layers on the device (SURVEY.md 8f rank 2):
//   im = zoom(im, (1, 1, h/H, w/W), order=1); im = im.transpose(0,2,3,1) + mean_pixel; np.round(im)
// (pylayers/pylayers/pylayers.py:70-75, :315-319), followed by the ubyte cast CRF() applies
// (CRF/krahenbuhl2013/CRF.py:32).  At the training shape scipy's zoom alone costs ~13 ms per batch on
// the host, an order of magnitude more than the whole GPU pass.
//
// The zoom follows scipy.ndimage.zoom(order=1) operation by operation (zoom.cuh); the result is cast to
// float32 (the blob dtype), + mean in float64, round half to even, C cast to unsigned char.
#include <algorithm>
#include <climits>
#include <vector>

#include "common.cuh"
#include "zoom.cuh"

namespace dsrg {

__global__ void __launch_bounds__(kThreads)
k_prepare_image(const float *in, uint8_t *out, int Hi, int Wi, int Ho, int Wo, double m0, double m1,
                double m2) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Ho * Wo) return;
    const int oy = i / Wo, ox = i - oy * Wo;
    const ZoomTap tap = zoom_tap(oy, ox, Hi, Wi, Ho, Wo);
    const double mean[3] = {m0, m1, m2};
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float z = zoom_apply(in + ((size_t)b * 3 + c) * Hi * Wi, Wi, tap);  // float32 like the blob
        const double r = rint(__dadd_rn((double)z, mean[c]));  // + mean_pixel (float64), np.round
        out[((size_t)b * Ho * Wo + i) * 3 + c] = (uint8_t)(long long)r;  // .astype('ubyte')
    }
}

int prepare_image(Engine *e, int B, int Hi, int Wi, const float *in, const double *mean, uint8_t *out,
                  cudaStream_t s) {
    dim3 g(cdiv((long long)e->H * e->W, kThreads), B);
    DSRG_LAUNCH(e, T_PREP, s,
                k_prepare_image<<<g, kThreads, 0, s>>>(in, out, Hi, Wi, e->H, e->W, mean[0], mean[1], mean[2]));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

// The network input of the evaluation tools, every scale of one image (test-ms.py:68-81, test.py:60-73,
// test-coco.py:92-105, generate_train_gt.py:62-75, show-result.py:64-77; test-ms-f.py:100-112 and
// test-coco-f.py:124-136 with zoom factors):
//   image = nd.zoom(image.astype('float32'), (h/H, w/W, 1.0), order=1); image = image[:, :, [2, 1, 0]]
//   image = image - mean_pixel; image = image.transpose([2, 0, 1])    -> stored into the float32 blob
// The zoom is scipy's (zoom.cuh) on channel 2 - c, cast to float32; the mean is subtracted in float64 (numpy
// promotes the float32 image against the float64 mean_pixel) and the blob's store casts back to float32.
//
// B images of any sizes go to every scale's shared (h_k, w_k), so one network batch per scale follows.  Both tables
// travel as kernel parameters, never through a host-to-device copy, so a *_dev call can be captured in a CUDA graph.
// A batch larger than kNetInputImages is cut into launches of kNetInputImages images each.
constexpr int kNetInputImages = DSRG_PREP_IMAGES_PER_LAUNCH;

struct NetInputImage {
    const uint8_t *im;   // [H][W][3] uint8
    int H, W;
};

struct NetInputBatch {           // kernel parameters (about 1.5 KB)
    int n;
    int h[DSRG_PREP_MAX_SCALES], w[DSRG_PREP_MAX_SCALES];
    long long first[DSRG_PREP_MAX_SCALES + 1];   // first output pixel of scale k in an image's flat index
    float *out[DSRG_PREP_MAX_SCALES];           // [B][3][h][w] each, at this launch's first image
    double mean[3];
    NetInputImage img[kNetInputImages];
};

// one thread per output pixel of any scale of image blockIdx.y, all three channels (they share the tap)
__global__ void __launch_bounds__(kThreads)
k_prepare_net_input_batch(const __grid_constant__ NetInputBatch sc) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sc.first[sc.n]) return;
    int k = 0;
    while (i >= sc.first[k + 1]) k++;
    const int h = sc.h[k], w = sc.w[k];
    const int pix = (int)(i - sc.first[k]);
    const int oy = pix / w, ox = pix - oy * w;
    const NetInputImage m = sc.img[blockIdx.y];
    const ZoomTap tap = zoom_tap(oy, ox, m.H, m.W, h, w);
    float *o = sc.out[k] + (size_t)blockIdx.y * 3 * h * w;
    net_input_pixel(m.im, m.W, tap, sc.mean, o, h, w, pix);
}

// images[b] of Hs[b] x Ws[b]; the arguments were checked (net_input_args_ok, net_input_images_ok)
static int prepare_net_input(Engine *e, int B, const uint8_t *const *images, const int *Hs, const int *Ws, int n,
                             const int *hs, const int *ws, const double *mean, float *const *out, cudaStream_t s) {
    NetInputBatch sc;
    sc.n = n;
    sc.first[0] = 0;
    for (int k = 0; k < n; k++) {
        sc.h[k] = hs[k];
        sc.w[k] = ws[k];
        sc.first[k + 1] = sc.first[k] + (long long)hs[k] * ws[k];
    }
    for (int c = 0; c < 3; c++) sc.mean[c] = mean[c];
    for (int b0 = 0; b0 < B; b0 += kNetInputImages) {
        const int nb = std::min(kNetInputImages, B - b0);
        for (int k = 0; k < n; k++) sc.out[k] = out[k] + (size_t)b0 * 3 * hs[k] * ws[k];
        for (int j = 0; j < nb; j++) sc.img[j] = {images[b0 + j], Hs[b0 + j], Ws[b0 + j]};
        const dim3 g((unsigned)cdiv(sc.first[n], kThreads), (unsigned)nb);
        DSRG_LAUNCH(e, T_PREP, s, k_prepare_net_input_batch<<<g, kThreads, 0, s>>>(sc));
        DSRG_CUDA_TRY(cudaGetLastError());
    }
    return DSRG_OK;
}

}  // namespace dsrg

using namespace dsrg;

extern "C" int dsrg_prepare_image_dev(dsrg_engine *h, int B, int Hi, int Wi, const float *images_dev,
                                      const double *mean_pixel, uint8_t *image_out_dev, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, images_dev && mean_pixel && image_out_dev && Hi >= 1 && Wi >= 1, [&](Engine *e) {
        return prepare_image(e, B, Hi, Wi, images_dev, mean_pixel, image_out_dev, s);
    });
}

extern "C" int dsrg_prepare_image_host(dsrg_engine *h, int B, int Hi, int Wi, const float *images,
                                       const double *mean_pixel, uint8_t *image_out) {
    const bool ok = images && mean_pixel && image_out && Hi >= 1 && Wi >= 1;
    return host_call(h, B, ok, false, [&](Engine *e, cudaStream_t s) {
        const size_t need = (size_t)B * 3 * Hi * Wi;  // raw images come in any size
        if (int rc = grow_staging(e, (void **)&e->st_raw, &e->st_raw_cap, need * sizeof(float))) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_raw, images, need * sizeof(float), cudaMemcpyHostToDevice, s));
        if (int rc = prepare_image(e, B, Hi, Wi, e->st_raw, mean_pixel, e->st_image, s)) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(image_out, e->st_image, (size_t)B * e->N * 3, cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}

// The scale table: pointers non-NULL, 1 <= n_scales <= DSRG_PREP_MAX_SCALES, every size >= 1 and every plane below
// 2^31 pixels.  Read before the engine is looked at; the engine's own size plays no part.
static bool net_input_scales_ok(int n, const int *hs, const int *ws, const double *mean, float *const *out) {
    if (!hs || !ws || !mean || !out || n < 1 || n > DSRG_PREP_MAX_SCALES) return false;
    for (int k = 0; k < n; k++)
        if (!out[k] || hs[k] < 1 || ws[k] < 1 || (long long)hs[k] * ws[k] > INT_MAX) return false;
    return true;
}

// the scale table and one image of H x W
static bool net_input_args_ok(const void *image, int H, int W, int n, const int *hs, const int *ws,
                              const double *mean, float *const *out) {
    return image && H >= 1 && W >= 1 && (long long)H * W <= INT_MAX && net_input_scales_ok(n, hs, ws, mean, out);
}

// The per-image sizes of a batch, read once check_batch has bounded B: every image pointer non-NULL, every size >= 1
// and every plane below 2^31 pixels.
static bool net_input_images_ok(int B, const uint8_t *const *images, const int *Hs, const int *Ws) {
    for (int b = 0; b < B; b++)
        if (!images[b] || Hs[b] < 1 || Ws[b] < 1 || (long long)Hs[b] * Ws[b] > INT_MAX) {
            set_error("bad argument: image %d (NULL pointer or size out of range)", b);
            return false;
        }
    return true;
}

// B images staged through st_prep and every scale of them copied back.  st_prep: [scale 0 B x 3 x h x w float32]
// [scale 1]...[image 0][image 1]..., each part padded to 256 bytes.  A buffer of its own: the score maps that
// dsrg_predict_mask_host stages through st_raw are part of its graph keys, and growing st_raw here would move them.
static int prepare_net_input_staged(Engine *e, int B, const uint8_t *const *images, const int *Hs, const int *Ws,
                                    int n, const int *hs, const int *ws, const double *mean, float *const *out,
                                    cudaStream_t s) {
    auto padded = [](size_t bytes) { return (bytes + 255) / 256 * 256; };
    size_t total = 0;
    for (int k = 0; k < n; k++) total += padded((size_t)B * 3 * hs[k] * ws[k] * sizeof(float));
    for (int b = 0; b < B; b++) total += padded((size_t)Hs[b] * Ws[b] * 3);
    if (int rc = grow_staging(e, (void **)&e->st_prep, &e->st_prep_cap, total)) return rc;
    float *d_out[DSRG_PREP_MAX_SCALES];
    std::vector<const uint8_t *> d_im(B);
    uint8_t *at = e->st_prep;
    for (int k = 0; k < n; k++) {
        d_out[k] = (float *)at;
        at += padded((size_t)B * 3 * hs[k] * ws[k] * sizeof(float));
    }
    for (int b = 0; b < B; b++) {
        const size_t bytes = (size_t)Hs[b] * Ws[b] * 3;
        DSRG_CUDA_TRY(cudaMemcpyAsync(at, images[b], bytes, cudaMemcpyHostToDevice, s));
        d_im[b] = at;
        at += padded(bytes);
    }
    if (int rc = prepare_net_input(e, B, d_im.data(), Hs, Ws, n, hs, ws, mean, d_out, s)) return rc;
    for (int k = 0; k < n; k++)
        DSRG_CUDA_TRY(cudaMemcpyAsync(out[k], d_out[k], (size_t)B * 3 * hs[k] * ws[k] * sizeof(float),
                                      cudaMemcpyDeviceToHost, s));
    return DSRG_OK;
}

extern "C" int dsrg_prepare_net_input_dev(dsrg_engine *h, const uint8_t *image_dev, int H, int W, int n_scales,
                                          const int *hs, const int *ws, const double *mean_pixel,
                                          float *const *out_dev, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    const bool ok = net_input_args_ok(image_dev, H, W, n_scales, hs, ws, mean_pixel, out_dev);
    return dev_call(h, 1, s, ok, [&](Engine *e) {
        return prepare_net_input(e, 1, &image_dev, &H, &W, n_scales, hs, ws, mean_pixel, out_dev, s);
    });
}

extern "C" int dsrg_prepare_net_input_host(dsrg_engine *h, const uint8_t *image, int H, int W, int n_scales,
                                           const int *hs, const int *ws, const double *mean_pixel,
                                           float *const *out) {
    const bool ok = net_input_args_ok(image, H, W, n_scales, hs, ws, mean_pixel, out);
    return host_call(h, 1, ok, false, [&](Engine *e, cudaStream_t s) {
        return prepare_net_input_staged(e, 1, &image, &H, &W, n_scales, hs, ws, mean_pixel, out, s);
    });
}

extern "C" int dsrg_prepare_net_input_batch_dev(dsrg_engine *h, const uint8_t *const *images_dev, const int *Hs,
                                                const int *Ws, int B, int n_scales, const int *hs, const int *ws,
                                                const double *mean_pixel, float *const *out_dev, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    // the per-image entries are read in the body (net_input_images_ok), once check_batch has bounded B
    const bool ok = images_dev && Hs && Ws && net_input_scales_ok(n_scales, hs, ws, mean_pixel, out_dev);
    return dev_call(h, B, s, ok, [&](Engine *e) {
        if (!net_input_images_ok(B, images_dev, Hs, Ws)) return DSRG_E_INVALID;
        return prepare_net_input(e, B, images_dev, Hs, Ws, n_scales, hs, ws, mean_pixel, out_dev, s);
    });
}

extern "C" int dsrg_prepare_net_input_batch_host(dsrg_engine *h, const uint8_t *const *images, const int *Hs,
                                                 const int *Ws, int B, int n_scales, const int *hs, const int *ws,
                                                 const double *mean_pixel, float *const *out) {
    const bool ok = images && Hs && Ws && net_input_scales_ok(n_scales, hs, ws, mean_pixel, out);
    return host_call(h, B, ok, false, [&](Engine *e, cudaStream_t s) {
        if (!net_input_images_ok(B, images, Hs, Ws)) return DSRG_E_INVALID;
        return prepare_net_input_staged(e, B, images, Hs, Ws, n_scales, hs, ws, mean_pixel, out, s);
    });
}
