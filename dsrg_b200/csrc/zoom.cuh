// scipy.ndimage.zoom(order=1, mode='constant', grid_mode=False) for one output pixel, operation by
// operation (scipy ni_interpolation.c NI_ZoomShift + ni_splines.c; oracle/crf_oracle.py
// zoom_order1_restated is the numpy twin, checked bit-for-bit against scipy in tests/):
//   * output index o -> input coordinate c = o * ((in-1)/(out-1)), float64
//   * c > in-1 (one rounding error at the last row / column of some size pairs) is out of bounds and the
//     output pixel is cval = 0
//   * weights w0 = 1 - (c - floor(c)), w1 = 1 - w0
//   * value = ((v00*wy0)*wx0 + (v01*wy0)*wx1) + (v10*wy1)*wx0 + (v11*wy1)*wx1, summed left to right in
//     float64 without contraction, then cast to float32 (the array dtype)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dsrg {

struct ZoomTap {
    int y0, y1, x0, x1;
    double wy0, wy1, wx0, wx1;
    bool oob;
};

__device__ __forceinline__ ZoomTap zoom_tap(int oy, int ox, int Hi, int Wi, int Ho, int Wo) {
    ZoomTap z;
    const double zy = Ho > 1 ? (double)(Hi - 1) / (double)(Ho - 1) : 0.0;
    const double zx = Wo > 1 ? (double)(Wi - 1) / (double)(Wo - 1) : 0.0;
    const double ys = __dmul_rn((double)oy, zy), xs = __dmul_rn((double)ox, zx);
    z.oob = ys > (double)(Hi - 1) || xs > (double)(Wi - 1);
    z.y0 = min((int)floor(ys), Hi - 1);
    z.x0 = min((int)floor(xs), Wi - 1);
    z.y1 = min(z.y0 + 1, Hi - 1);
    z.x1 = min(z.x0 + 1, Wi - 1);
    z.wy0 = __dsub_rn(1.0, __dsub_rn(ys, (double)z.y0));
    z.wx0 = __dsub_rn(1.0, __dsub_rn(xs, (double)z.x0));
    z.wy1 = __dsub_rn(1.0, z.wy0);
    z.wx1 = __dsub_rn(1.0, z.wx0);
    return z;
}

// the four taps of z, `at(y, x)` giving the input value at (y, x) as float64
template <typename At>
__device__ __forceinline__ float zoom_taps(const ZoomTap &z, At at) {
    if (z.oob) return 0.0f;
    double t = __dmul_rn(__dmul_rn(at(z.y0, z.x0), z.wy0), z.wx0);
    t = __dadd_rn(t, __dmul_rn(__dmul_rn(at(z.y0, z.x1), z.wy0), z.wx1));
    t = __dadd_rn(t, __dmul_rn(__dmul_rn(at(z.y1, z.x0), z.wy1), z.wx0));
    t = __dadd_rn(t, __dmul_rn(__dmul_rn(at(z.y1, z.x1), z.wy1), z.wx1));
    return (float)t;
}

// p: one [Hi][Wi] float32 plane
__device__ __forceinline__ float zoom_apply(const float *__restrict__ p, int Wi, const ZoomTap &z) {
    return zoom_taps(z, [&](int y, int x) { return (double)p[(size_t)y * Wi + x]; });
}

// p: an interleaved [Hi][Wi][3] uint8 image, channel c.  Its values are what image.astype('float32') hands to
// scipy: the float32 cast of a uint8 is exact, and so is the float64 one.
__device__ __forceinline__ float zoom_apply(const uint8_t *__restrict__ p, int Wi, int c, const ZoomTap &z) {
    return zoom_taps(z, [&](int y, int x) { return (double)p[((size_t)y * Wi + x) * 3 + c]; });
}

// One pixel of a network input built the way the evaluation tools' preprocess() and AnnotationLayerCOCO build it:
//   nd.zoom(image.astype('float32'), (h/H, w/W, 1.0), order=1)[:, :, [2, 1, 0]] - mean, transposed to CHW
// The zoom of channel 2 - c of the interleaved [H][W][3] image at `tap` (zoom_tap of the pixel in an h x w output),
// minus mean[c] in float64 (numpy promotes against the float64 mean), stored as float32 at o[c * h * w + pix].
__device__ __forceinline__ void net_input_pixel(const uint8_t *__restrict__ im, int W, const ZoomTap &tap,
                                                const double *mean, float *o, int h, int w, int pix) {
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float z = zoom_apply(im, W, 2 - c, tap);                     // float32, like nd.zoom's result
        o[(size_t)c * h * w + pix] = (float)__dsub_rn((double)z, mean[c]);  // - mean_pixel (float64)
    }
}

}  // namespace dsrg
