// Image preprocessing of the Python layers on the device (SURVEY.md 8f rank 2):
//   im = zoom(im, (1, 1, h/H, w/W), order=1); im = im.transpose(0,2,3,1) + mean_pixel; np.round(im)
// (pylayers/pylayers/pylayers.py:70-75, :315-319), followed by the ubyte cast CRF() applies
// (CRF/krahenbuhl2013/CRF.py:32).  At the training shape scipy's zoom alone costs ~13 ms per batch on
// the host, an order of magnitude more than the whole GPU pass.
//
// The zoom follows scipy.ndimage.zoom(order=1) operation by operation (zoom.cuh); the result is cast to
// float32 (the blob dtype), + mean in float64, round half to even, C cast to unsigned char.
#include <climits>

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
struct NetInputScales {           // kernel parameters
    int n;
    int h[DSRG_PREP_MAX_SCALES], w[DSRG_PREP_MAX_SCALES];
    long long first[DSRG_PREP_MAX_SCALES + 1];   // first output pixel of scale k in the flat index; first[n] = total
    float *out[DSRG_PREP_MAX_SCALES];           // [3][h][w] each
    double mean[3];
};

// one thread per output pixel of any scale, all three channels (they share the tap)
__global__ void __launch_bounds__(kThreads)
k_prepare_net_input(const uint8_t *__restrict__ im, int H, int W, NetInputScales sc) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sc.first[sc.n]) return;
    int k = 0;
    while (i >= sc.first[k + 1]) k++;
    const int h = sc.h[k], w = sc.w[k];
    const int pix = (int)(i - sc.first[k]);
    const int oy = pix / w, ox = pix - oy * w;
    const ZoomTap tap = zoom_tap(oy, ox, H, W, h, w);
    float *o = sc.out[k];
    net_input_pixel(im, W, tap, sc.mean, o, h, w, pix);
}

static int prepare_net_input(Engine *e, int H, int W, const uint8_t *image, int n, const int *hs, const int *ws,
                             const double *mean, float *const *out, cudaStream_t s) {
    NetInputScales sc;
    sc.n = n;
    sc.first[0] = 0;
    for (int k = 0; k < n; k++) {
        sc.h[k] = hs[k];
        sc.w[k] = ws[k];
        sc.out[k] = out[k];
        sc.first[k + 1] = sc.first[k] + (long long)hs[k] * ws[k];
    }
    for (int c = 0; c < 3; c++) sc.mean[c] = mean[c];
    DSRG_LAUNCH(e, T_PREP, s, k_prepare_net_input<<<cdiv(sc.first[n], kThreads), kThreads, 0, s>>>(image, H, W, sc));
    DSRG_CUDA_TRY(cudaGetLastError());
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

// Pointers non-NULL, 1 <= n_scales <= DSRG_PREP_MAX_SCALES, every size >= 1 and every plane below 2^31 pixels.
// Read before the engine is looked at; the engine's own size plays no part.
static bool net_input_args_ok(const void *image, int H, int W, int n, const int *hs, const int *ws,
                              const double *mean, float *const *out) {
    if (!image || !hs || !ws || !mean || !out || H < 1 || W < 1 || (long long)H * W > INT_MAX || n < 1 ||
        n > DSRG_PREP_MAX_SCALES)
        return false;
    for (int k = 0; k < n; k++)
        if (!out[k] || hs[k] < 1 || ws[k] < 1 || (long long)hs[k] * ws[k] > INT_MAX) return false;
    return true;
}

extern "C" int dsrg_prepare_net_input_dev(dsrg_engine *h, const uint8_t *image_dev, int H, int W, int n_scales,
                                          const int *hs, const int *ws, const double *mean_pixel,
                                          float *const *out_dev, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    const bool ok = net_input_args_ok(image_dev, H, W, n_scales, hs, ws, mean_pixel, out_dev);
    return dev_call(h, 1, s, ok, [&](Engine *e) {
        return prepare_net_input(e, H, W, image_dev, n_scales, hs, ws, mean_pixel, out_dev, s);
    });
}

extern "C" int dsrg_prepare_net_input_host(dsrg_engine *h, const uint8_t *image, int H, int W, int n_scales,
                                           const int *hs, const int *ws, const double *mean_pixel,
                                           float *const *out) {
    const bool ok = net_input_args_ok(image, H, W, n_scales, hs, ws, mean_pixel, out);
    return host_call(h, 1, ok, false, [&](Engine *e, cudaStream_t s) {
        // st_prep: [image, padded to 256 bytes][scale 0][scale 1]...  A buffer of its own: the score maps that
        // dsrg_predict_mask_host stages through st_raw are part of its graph keys, and growing st_raw here would
        // move them
        const size_t in_bytes = ((size_t)H * W * 3 + 255) / 256 * 256;
        size_t total = 0;
        for (int k = 0; k < n_scales; k++) total += (size_t)3 * hs[k] * ws[k];
        if (int rc = grow_staging(e, (void **)&e->st_prep, &e->st_prep_cap, in_bytes + total * sizeof(float)))
            return rc;
        uint8_t *d_im = (uint8_t *)e->st_prep;
        float *d_out[DSRG_PREP_MAX_SCALES];
        float *at = (float *)(e->st_prep + in_bytes);
        for (int k = 0; k < n_scales; k++) {
            d_out[k] = at;
            at += (size_t)3 * hs[k] * ws[k];
        }
        DSRG_CUDA_TRY(cudaMemcpyAsync(d_im, image, (size_t)H * W * 3, cudaMemcpyHostToDevice, s));
        if (int rc = prepare_net_input(e, H, W, d_im, n_scales, hs, ws, mean_pixel, d_out, s)) return rc;
        for (int k = 0; k < n_scales; k++)
            DSRG_CUDA_TRY(cudaMemcpyAsync(out[k], d_out[k], (size_t)3 * hs[k] * ws[k] * sizeof(float),
                                          cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}
