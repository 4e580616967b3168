// Image preprocessing of the Python layers on the device (SURVEY.md 8f rank 2):
//   im = zoom(im, (1, 1, h/H, w/W), order=1); im = im.transpose(0,2,3,1) + mean_pixel; np.round(im)
// (pylayers/pylayers/pylayers.py:70-75, :315-319), followed by the ubyte cast CRF() applies
// (CRF/krahenbuhl2013/CRF.py:32).  At the training shape scipy's zoom alone costs ~13 ms per batch on
// the host, an order of magnitude more than the whole GPU pass.
//
// The zoom follows scipy.ndimage.zoom(order=1) operation by operation (zoom.cuh); the result is cast to
// float32 (the blob dtype), + mean in float64, round half to even, C cast to unsigned char.
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
