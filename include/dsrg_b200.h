/*
 * dsrg_b200.h -- C ABI of the H100-native DSRG pixel-labelling hot path.
 *
 * Plain C, no torch / C++ types.  All `*_dev` pointers are CUDA device pointers on the
 * engine's device (e.g. torch.Tensor.data_ptr()); all `*_host` pointers are host memory
 * (pinned memory from dsrg_host_alloc() makes the copies asynchronous).  `stream` is a
 * cudaStream_t passed as void* (NULL = legacy default stream).  Every function returning int
 * returns 0 on success and a negative DSRG_E_* code on failure; dsrg_last_error() then holds a
 * human-readable message (thread-local).  Nothing in this library falls back to a CPU path:
 * without a usable sm_90 device every call fails with DSRG_E_CUDA.
 *
 * Each entry point names the reference interface (speedinghzl/DSRG, path:line) it replaces.
 * Layout names: NHWC = [B][H][W][M] (pixel-major, what krahenbuhl2013.CRF and DenseCRFWrapper
 * use), NCHW = [B][M][H][W] (Caffe blobs, what pylayers.py passes around).
 */
#ifndef DSRG_B200_H
#define DSRG_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DSRG_OK 0
#define DSRG_E_INVALID (-1)   /* bad argument (shape, layout, NULL pointer, batch > max_batch) */
#define DSRG_E_CUDA (-2)      /* CUDA runtime error, or no sm_90 device                         */
#define DSRG_E_KEYRANGE (-3)  /* lattice coordinates exceed the packed-key range (see DESIGN.md) */
#define DSRG_E_STATE (-4)     /* call order violated (e.g. inference before add_pairwise)       */
#define DSRG_E_NOMEM (-5)

#define DSRG_LAYOUT_NHWC 0
#define DSRG_LAYOUT_NCHW 1

#define DSRG_MAX_LABELS 32 /* labels per pixel of the fused, register-tiled kernels (the 21-class hot path) */
/* CRF (batch, layer and DenseCRF-object entry points), SRG, the predict_mask post-processing and the confusion
 * matrix accept up to this many labels: above DSRG_MAX_LABELS the mean field runs on a generic label-chunked path
 * (csrc/meanfield_wide.cu) -- the reference's COCO tool uses DenseCRF(W, H, 81), training/tools/test-coco.py.
 * Of the layers, only Softmax is limited to DSRG_MAX_LABELS; ConstrainLoss, BalancedSeedLoss, the SEC losses and
 * the COCO annotation layer have no label limit of their own. */
#define DSRG_MAX_LABELS_WIDE 255
/* pixels per class plane the GWRP kernels of dsrg_expandloss_* sort in shared memory (41x41 and the 65x65 maps
 * of a 513 crop fit; larger planes return DSRG_E_INVALID) */
#define DSRG_GWRP_MAX_PLANE 8192

int dsrg_version(void);               /* 10000*major + 100*minor + patch */
const char *dsrg_last_error(void);    /* message of the last failing call on this thread */
int dsrg_device_count(void);          /* number of visible CUDA devices (0 if none / no driver) */
/* The device an engine is created on when `device` is -1, and the one the drop-ins (pylayers, krahenbuhl2013,
 * the DenseCRF objects) use: DSRG_B200_DEVICE if set, else the calling thread's current CUDA device -- what
 * caffe.set_device(N) (training/tools/train.py:77-79) or torch.cuda.set_device selected.  -1 if there is none.
 * Every entry point restores the caller's current device before it returns. */
int dsrg_current_device(void);

/* Pinned host memory so the *_host entry points overlap their copies (cudaHostAlloc). */
void *dsrg_host_alloc(size_t bytes);
void dsrg_host_free(void *p);
/* Page-lock memory the caller already owns (a Caffe blob's CPU buffer in CPU mode, a numpy array) so that the
 * *_host entry points copy from / to it asynchronously at full PCIe rate (cudaHostRegister / Unregister). */
int dsrg_host_register(void *p, size_t bytes);
int dsrg_host_unregister(void *p);

/* ------------------------------------------------------------------------------------------
 * Pairwise parameters of krahenbuhl2013.CRF -- CRF/krahenbuhl2013/CRF.py:31-32 passes
 * (w1=10, 80/s, 80/s, 13, 13, 13, w2=3, 3/s, 3/s); argument order and meaning are those of
 * DenseCRFWrapper::add_pairwise_energy, CRF/src/densecrf_wrapper.cpp:18-30
 * (Gaussian/spatial kernel w2 is applied BEFORE the bilateral kernel w1).
 * ------------------------------------------------------------------------------------------ */
typedef struct dsrg_crf_params {
    float w1;            /* bilateral Potts weight                     */
    float theta_alpha_x; /* bilateral spatial sigma (x)                */
    float theta_alpha_y; /* bilateral spatial sigma (y)                */
    float theta_beta_r;  /* bilateral colour sigmas, channel 0 / 1 / 2 */
    float theta_beta_g;
    float theta_beta_b;
    float w2;            /* spatial Potts weight                       */
    float theta_gamma_x; /* spatial sigma (x)                          */
    float theta_gamma_y; /* spatial sigma (y)                          */
    int n_iters;         /* mean-field iterations (CRF.py:4 maxiter=10) */
} dsrg_crf_params;

/* Fill `p` exactly as CRF.py:31-32 does for a given scale_factor / color_factor / maxiter. */
void dsrg_crf_params_default(dsrg_crf_params *p, float scale_factor, float color_factor, int maxiter);

/* ------------------------------------------------------------------------------------------
 * Engine: owns every device buffer the batched kernels need for up to max_batch images of
 * H x W pixels and M labels on `device` (-1: dsrg_current_device()).  No allocation happens on the hot calls.
 * ------------------------------------------------------------------------------------------ */
typedef struct dsrg_engine dsrg_engine;

dsrg_engine *dsrg_engine_create(int device, int max_batch, int H, int W, int M);
void dsrg_engine_destroy(dsrg_engine *e);
size_t dsrg_engine_device_bytes(const dsrg_engine *e); /* bytes of HBM held by the engine */
/* The H x W given to dsrg_engine_create is a capacity: any H' <= H, W' <= W can be selected afterwards
 * without reallocating (the evaluation tools run one image at a time, each of its own size --
 * training/tools/test-ms.py:86-87).  Waits for queued work; the cached spatial lattice is rebuilt. */
int dsrg_engine_set_size(dsrg_engine *e, int H, int W);
/* The same re-shape without the wait, for a caller that drives the engine only through its entry points: each of
 * them orders its pass after the engine's previous one (same stream, or a wait for its order event), and queued
 * passes keep their own strides.  A replay of the caller's own CUDA graph of this engine's launches is not ordered
 * that way: replays and later calls go on one stream, or the caller orders them. */
int dsrg_engine_set_size_ordered(dsrg_engine *e, int H, int W);
int dsrg_engine_get_size(const dsrg_engine *e, int *H, int *W, int *H_capacity, int *W_capacity);
/* The *_host full-pass entry points pipeline the batch in chunks (default B/8, 3B/8, B/2 images) through
 * H2D | kernels | D2H streams; `images` > 0 caps the chunk size, 0 restores the default. */
int dsrg_engine_set_host_chunk(dsrg_engine *e, int images);
/* Device passes (*_dev entry points, and through them the chunks of the *_host ones) are captured into CUDA
 * graphs the second time a pass is issued with the same arguments and replayed afterwards -- one launch instead
 * of 40-130 dependent ones.  Needs a real stream (not the legacy default stream); enable = 0 turns it off and
 * drops the cached graphs (also: environment DSRG_B200_GRAPHS=0).  graph_replays counts the passes replayed. */
int dsrg_engine_set_graphs(dsrg_engine *e, int enable);
long long dsrg_engine_graph_replays(const dsrg_engine *e);
/* Kernel launches issued by this engine since the last call (bench.py's gpu_launches); the kernels inside a
 * replayed graph are counted. */
long long dsrg_engine_take_launch_count(dsrg_engine *e);
/* Diagnostic: how many tiles of the last mean-field pass took the hybrid path (the shared-memory list of the tile's
 * most-touched bilateral vertices plus direct global slices / reductions for the rest -- textured images; see
 * csrc/tiles.cu).  Synchronises the device; < 0 on error.  No reference analogue (permutohedral.cpp:545-584 visits
 * every (pixel, vertex) incidence the same way). */
long long dsrg_engine_hybrid_tiles(dsrg_engine *e);

/*
 * Batched dense-CRF mean-field inference; replaces the per-image loop
 *   for i in range(N): result[i] = CRF(im[i], unary[i], scale_factor)
 * of pylayers/pylayers/pylayers.py:81-82 / :325-326, i.e. B x { CRF.py:4-37 ->
 * wrapper.pyx:23-60 -> densecrf_wrapper.cpp:5-50 -> DenseCRF::inference, densecrf.cpp:115-131 }.
 *   unary : B x (H,W,M) values as passed to CRF(image, unary): energy = -unary (CRF.py:28)
 *   image : B x (H,W,3) uint8 (CRF.py:32 casts to ubyte)
 *   out   : B x marginals Q, float32
 * Results are within 1e-4 (max abs) of the reference; see DESIGN.md for why not bit-exact.
 */
int dsrg_crf_batch_dev(dsrg_engine *e, int B, const float *unary_dev, int unary_layout,
                       const uint8_t *image_dev, const dsrg_crf_params *params, float *out_dev,
                       int out_layout, void *stream);
int dsrg_crf_batch_host(dsrg_engine *e, int B, const float *unary_host, int unary_layout,
                        const uint8_t *image_host, const dsrg_crf_params *params, float *out_host,
                        int out_layout);
/* arg-max labelling after inference: DenseCRFWrapper::map, densecrf_wrapper.cpp:39-43 */
int dsrg_crf_map_batch_dev(dsrg_engine *e, int B, const float *unary_dev, int unary_layout,
                           const uint8_t *image_dev, const dsrg_crf_params *params,
                           int32_t *labels_out_dev, void *stream);

/*
 * Batched seeded region growing; replaces
 *   self.pool.map(generate_seed_step, items)     pylayers/pylayers/pylayers.py:341-342
 * = B x generate_seed_step (pylayers.py:237-275) incl. CC_labeling_8.CC_lab
 * (pylayers/pylayers/CC_labeling_8.py:103-282).
 *   labels : [B][M]       image-level tags, class c present iff labels[c] == 1
 *   probs  : [B][M][H][W] float32 (compared in float64 like the reference's data)
 *   cues   : [B][M][H][W] float32 0/1 seeds
 *   th1,th2: background / foreground thresholds as float64 (the reference compares Python
 *            floats 0.99 / 0.85 against float64 data with strict >)
 *   renorm : 1 = first apply the post-CRF clamp(1e-4) + float64 renormalisation of
 *            pylayers.py:328-330 to `probs` (the DSRGLayer path); 0 = use probs as given
 *   seeds_out     : [B][M][H][W] float32 0/1 (old seeds are kept, pylayers.py:275)
 *   label_map_out : optional [B][H][W] int32 (0 = none, c+1 = class c), may be NULL
 * Bit-exact against the reference for identical inputs.
 */
int dsrg_srg_batch_dev(dsrg_engine *e, int B, const float *labels_dev, const float *probs_dev,
                       const float *cues_dev, double th1, double th2, int renorm,
                       float *seeds_out_dev, int32_t *label_map_out_dev, void *stream);
int dsrg_srg_batch_host(dsrg_engine *e, int B, const float *labels_host, const float *probs_host,
                        const float *cues_host, double th1, double th2, int renorm,
                        float *seeds_out_host, int32_t *label_map_out_host);

/*
 * The whole DSRGLayer.forward body (pylayers.py:297-304, :333-344): refinement
 * (pylayers.py:310-331: in-place clamp of probs at 1e-4, CRF with unary = probs, clamp +
 * float64 renormalise) followed by SRG.  `image` is the already zoomed / mean-added / rounded
 * uint8 image at the probs resolution (the host shim does pylayers.py:315-319).
 *   probs_dev     : [B][M][H][W], CLAMPED IN PLACE like the reference's bottom blob (:312)
 *   crf_out_dev   : optional [B][M][H][W] float32 RAW CRF marginals of this very call, i.e. before
 *                   the clamp + float64 renormalisation of :328-330 (NULL to skip)
 */
int dsrg_dsrg_forward_dev(dsrg_engine *e, int B, const float *labels_dev, float *probs_dev,
                          const float *cues_dev, const uint8_t *image_dev,
                          const dsrg_crf_params *params, double th1, double th2,
                          float *seeds_out_dev, float *crf_out_dev, void *stream);
int dsrg_dsrg_forward_host(dsrg_engine *e, int B, const float *labels_host, float *probs_host,
                           const float *cues_host, const uint8_t *image_host,
                           const dsrg_crf_params *params, double th1, double th2,
                           float *seeds_out_host, float *crf_out_host);

/*
 * SURVEY 8f rank 1 -- the producer of `probs` and the other consumer of the CRF result:
 * SoftmaxLayer (pylayers.py:23-51): probs = (softmax(preds) + 1e-4) / sum(...); backward = d sum(probs*top_diff)/d preds.
 * ConstrainLossLayer (pylayers.py:154-180): loss = mean_{n,h,w} sum_c ps log(clip(ps/probs, 0.05, 20)), ps = exp(log_smooth);
 * backward writes both gradients (pylayers.py:176-180).  All arrays [B][M][H][W] float32.
 */
int dsrg_softmax_forward_dev(dsrg_engine *e, int B, const float *preds_dev, float *probs_out_dev, void *stream);
int dsrg_softmax_backward_dev(dsrg_engine *e, int B, const float *preds_dev, const float *top_diff_dev,
                              float *grad_out_dev, void *stream);
int dsrg_constrainloss_forward_dev(dsrg_engine *e, int B, const float *probs_dev, const float *log_smooth_dev,
                                   float *loss_out_dev /* 1 float */, void *stream);
int dsrg_constrainloss_backward_dev(dsrg_engine *e, int B, const float *probs_dev, const float *log_smooth_dev,
                                    float *grad_probs_dev, float *grad_log_dev, void *stream);
int dsrg_softmax_forward_host(dsrg_engine *e, int B, const float *preds_host, float *probs_out_host);
int dsrg_softmax_backward_host(dsrg_engine *e, int B, const float *preds_host, const float *top_diff_host,
                               float *grad_out_host);
int dsrg_constrainloss_forward_host(dsrg_engine *e, int B, const float *probs_host, const float *log_smooth_host,
                                    float *loss_out_host /* 1 float */);
int dsrg_constrainloss_backward_host(dsrg_engine *e, int B, const float *probs_host, const float *log_smooth_host,
                                     float *grad_probs_host, float *grad_log_host);

/*
 * Image preprocessing of CRFLayer / DSRGLayer (pylayers.py:70-75, :315-319) + the ubyte cast of
 * CRF.py:32: bilinear zoom (scipy.ndimage.zoom order=1 semantics, float64 arithmetic, bit-exact) of the
 * [B][3][Hi][Wi] float32 network input to the engine's H x W, + mean_pixel[3], round half to even, ->
 * [B][H][W][3] uint8, the `image` argument of the entry points above.
 */
int dsrg_prepare_image_dev(dsrg_engine *e, int B, int Hi, int Wi, const float *images_dev,
                           const double *mean_pixel /* host, 3 */, uint8_t *image_out_dev, void *stream);
int dsrg_prepare_image_host(dsrg_engine *e, int B, int Hi, int Wi, const float *images_host,
                            const double *mean_pixel /* host, 3 */, uint8_t *image_out_host);

/*
 * The network input of the evaluation tools: preprocess(image, size) of training/tools/test-ms.py:68-81,
 * test.py:60-73, test-coco.py:92-105, generate_train_gt.py:62-75, show-result.py:64-77 (absolute sizes) and
 * test-ms-f.py:100-112, test-coco-f.py:124-136 (zoom factors), for every scale of one image in one launch:
 *   image = nd.zoom(image.astype('float32'), (h/H, w/W, 1.0), order=1)   scipy.ndimage.zoom order=1 semantics,
 *                                                                         float64 arithmetic, float32 result
 *   image = image[:, :, [2, 1, 0]]; image = image - mean_pixel            float64, like numpy with the tools'
 *   image = image.transpose([2, 0, 1])                                    np.array([104.0, 117.0, 123.0])
 * stored into the float32 `images` blob; bit-exact.
 *   image   : [H][W][3] uint8, interleaved, as pylab.imread / cv2.imread return it
 *   hs, ws  : n_scales output sizes, host memory in both variants (1 <= n_scales <= DSRG_PREP_MAX_SCALES); the
 *             tools' sizes are int(round(H * f)), int(round(W * f)) -- scipy's output shape
 *   out     : host array of n_scales pointers to [3][hs[k]][ws[k]] float32
 * H and W are the image's: the call neither reads nor changes the engine's size (dsrg_engine_set_size).
 */
#define DSRG_PREP_MAX_SCALES 16
int dsrg_prepare_net_input_dev(dsrg_engine *e, const uint8_t *image_dev, int H, int W, int n_scales,
                               const int *hs, const int *ws, const double *mean_pixel /* host, 3 */,
                               float *const *out_dev, void *stream);
int dsrg_prepare_net_input_host(dsrg_engine *e, const uint8_t *image_host, int H, int W, int n_scales,
                                const int *hs, const int *ws, const double *mean_pixel /* host, 3 */,
                                float *const *out_host);
/*
 * The same network input for B images of any sizes (1 <= B <= the engine's max_batch): one network batch per scale.
 * The evaluation tools pass absolute sizes, so every image of a list goes to the same (h_k, w_k) whatever its own size.
 *   images  : host array of B pointers to [Hs[b]][Ws[b]][3] uint8 images (device memory in _dev)
 *   Hs, Ws  : host arrays of the B image sizes
 *   hs, ws  : as above; every image of the call is zoomed to (hs[k], ws[k])
 *   out     : host array of n_scales pointers to [B][3][hs[k]][ws[k]] float32
 * Image b of out[k] is bit-identical to dsrg_prepare_net_input_* of that image alone.  The image and scale tables are
 * kernel parameters: _dev copies nothing from the host and can be captured in a CUDA graph.  One launch covers up to
 * DSRG_PREP_IMAGES_PER_LAUNCH images.  Like the per-image call, it neither reads nor changes the engine's size.
 */
#define DSRG_PREP_IMAGES_PER_LAUNCH 64
int dsrg_prepare_net_input_batch_dev(dsrg_engine *e, const uint8_t *const *images_dev, const int *Hs, const int *Ws,
                                     int B, int n_scales, const int *hs, const int *ws,
                                     const double *mean_pixel /* host, 3 */, float *const *out_dev, void *stream);
int dsrg_prepare_net_input_batch_host(dsrg_engine *e, const uint8_t *const *images_host, const int *Hs,
                                      const int *Ws, int B, int n_scales, const int *hs, const int *ws,
                                      const double *mean_pixel /* host, 3 */, float *const *out_host);

/*
 * Full-resolution inference post-processing: what predict_mask() of the evaluation / ground-truth tools
 * does between the network's score blob and the label map (engine batch 1, size = the image's):
 *   DSRG_POST_SUM_SCORES  training/tools/test-ms.py:84-111: scores_all = sum_k zoom(scores_k, order=1);
 *                         softmax over labels; clamp at eps; CRF(im, log(probs)); argmax
 *   DSRG_POST_ZOOM_PROBS  training/tools/generate_train_gt.py:76-104: softmax at network resolution;
 *                         zoom(probs, order=1); clamp at eps; CRF(im, log(probs)); argmax over `labels_sel`
 * These two are dsrg_predict_mask_batch_* below at B = 1, with the selection taken from host memory.
 *   scores     : n_scales pointers (1 <= n_scales <= 16) to [M][h_k][w_k] float32 (net.blobs['fc8-SEC'].data[0]);
 *                the array of pointers and hs / ws live on the host in both variants
 *   image      : [H][W][3] uint8 as handed to krahenbuhl2013.CRF (may be NULL when smooth == 0)
 *   smooth     : 0 skips the CRF (the tools' `smooth=False`)
 *   labels_sel : n_sel (<= 255) label ids in [0, M), on the host in both variants ([0] + image tags in
 *                generate_train_gt.py:96-97); n_sel == 0 = all labels.  Read during the call only
 *   result_out : [H][W] int32 label map;  probs_out : optional [H][W][M] float32 (CRF marginals, or the
 *                clamped probabilities when smooth == 0)
 * dsrg_zoom_scores_* is the zoom step alone ([M][h][w] -> [H][W][M], scipy.ndimage.zoom order=1 semantics,
 * bit-exact; accumulate != 0 adds to `out` in float32 like `scores_all += scores`).
 */
#define DSRG_POST_SUM_SCORES 0
#define DSRG_POST_ZOOM_PROBS 1
int dsrg_zoom_scores_dev(dsrg_engine *e, const float *scores_dev, int h, int w, float *out_dev, int accumulate,
                         void *stream);
int dsrg_zoom_scores_host(dsrg_engine *e, const float *scores_host, int h, int w, float *out_host,
                          int accumulate);
int dsrg_predict_mask_dev(dsrg_engine *e, int mode, int n_scales, const float *const *scores_dev, const int *hs,
                          const int *ws, const uint8_t *image_dev, float eps, int smooth,
                          const dsrg_crf_params *params, const int32_t *labels_sel, int n_sel,
                          int32_t *result_out_dev, float *probs_out_dev, void *stream);
int dsrg_predict_mask_host(dsrg_engine *e, int mode, int n_scales, const float *const *scores_host,
                           const int *hs, const int *ws, const uint8_t *image_host, float eps, int smooth,
                           const dsrg_crf_params *params, const int32_t *labels_sel, int n_sel,
                           int32_t *result_out_host, float *probs_out_host);
/*
 * The same post-processing for B images of the engine's current size in one pass (1 <= B <= max_batch): the
 * pseudo-label run of test-ms.py / generate_train_gt.py over a dataset, or an evaluation loop that keeps fc8 on the
 * device.  One batched pass replaces B per-image ones of ~90 dependent launches each.
 *   scores    : n_scales pointers (1 <= n_scales <= 16) to [B][M][h_k][w_k] float32, one batched forward per
 *               scale; the array of pointers and hs / ws live on the host in both variants
 *   images    : [B][H][W][3] uint8 (may be NULL when smooth == 0)
 *   mode, eps, smooth, params : as for dsrg_predict_mask_*; DSRG_POST_ZOOM_PROBS takes n_scales == 1
 *   sel       : optional [B][M] int32; row b lists image b's label ids in the order the arg-max visits them (the
 *               first maximum wins, generate_train_gt.py:96-100) and ends at its first -1.  NULL or an empty row
 *               selects every label.  In _dev it is device memory read when the pass runs (its content is not
 *               part of a cached graph's key)
 *   result_out: [B][H][W] int32;  probs_out : optional [B][H][W][M] float32
 * dsrg_predict_mask_* runs this pass at B = 1, so with smooth == 0 every image's result and probs_out are
 * bit-identical to dsrg_predict_mask_* on that image alone: the same kernels compute every image the same way.
 * With smooth == 1 the CRF marginals follow the batched CRF's 1e-4 bound.
 * A sel entry outside [0, M) before the row's -1:
 *   _host: DSRG_E_INVALID before any copy or launch.
 *   _dev : the row is not read past it, and every pixel of that image's result is -1 (a prediction that
 *          dsrg_confusion_add_dev counts in invalid[1]); the caller checks it once the stream has run.
 */
int dsrg_predict_mask_batch_dev(dsrg_engine *e, const float *const *scores_dev, const int *hs, const int *ws,
                                int n_scales, int B, int mode, const uint8_t *images_dev, float eps, int smooth,
                                const dsrg_crf_params *params, const int32_t *sel_dev, int32_t *result_out_dev,
                                float *probs_out_dev, void *stream);
int dsrg_predict_mask_batch_host(dsrg_engine *e, const float *const *scores_host, const int *hs, const int *ws,
                                 int n_scales, int B, int mode, const uint8_t *images_host, float eps, int smooth,
                                 const dsrg_crf_params *params, const int32_t *sel_host, int32_t *result_out_host,
                                 float *probs_out_host);

/*
 * AnnotationLayer.forward (pylayers/pylayers/pylayers.py:369-387): image tags + sparse localisation cues
 * -> the dense `labels` [B][1][1][M] and `cues` [B][M][H][W] blobs (H x W = the engine's size), and the
 * optionally mirrored copy of the images.  Reading the pickle and drawing `flip` stay with the caller:
 *   tag_offsets [B+1], tags       : CSR of data_file['%i_labels'] per image (class ids; label 0 is always set)
 *   cue_offsets [B+1], cue_idx    : CSR of data_file['%i_cues']; cue_idx is [3][K] (class, row, column rows,
 *                                   K = cue_offsets[B]); negative indices wrap like numpy's, others are errors
 *   flip [B] or NULL              : 1 = mirror this image's cues and pixels along the width (flip == -1, :385)
 *   images_in / images_out        : [B][3][Hi][Wi] float32, distinct buffers; both NULL = skip the copy
 * All index arrays live on the host in both variants.
 */
int dsrg_annotation_forward_dev(dsrg_engine *e, int B, const int32_t *tag_offsets, const int32_t *tags,
                                const int32_t *cue_offsets, const int32_t *cue_idx, const int32_t *flip,
                                const float *images_in_dev, int Hi, int Wi, float *labels_out_dev,
                                float *cues_out_dev, float *images_out_dev, void *stream);
int dsrg_annotation_forward_host(dsrg_engine *e, int B, const int32_t *tag_offsets, const int32_t *tags,
                                 const int32_t *cue_offsets, const int32_t *cue_idx, const int32_t *flip,
                                 const float *images_in_host, int Hi, int Wi, float *labels_out_host,
                                 float *cues_out_host, float *images_out_host);

/*
 * AnnotationLayerCOCO.forward (pylayers/pylayers/pylayers.py:432-512), the COCO training input, after the caller
 * has decoded the files and drawn the random numbers (the shuffle and `flip`) in the reference's order.  Per image b:
 *   images[b]  : [Hs[b]][Ws[b]][3] uint8 BGR, as cv2.imread(..., IMREAD_COLOR) returns it; each image has its own size
 *   label_maps : [B][H][W] uint8 (H x W = the engine's size), as cv2.imread(..., IMREAD_GRAYSCALE) returns them
 *   flip [B] or NULL : 1 = mirror this image's pixels and cues along the width (flip == -1, :500-503)
 * ->
 *   images_out : [B][3][new_h][new_w] float32: zoom(image.astype('float32'), (new_h/H, new_w/W, 1.0), order=1),
 *                channels reversed, - mean_pixel in float64 (scipy.ndimage.zoom order=1 semantics, bit-exact; the
 *                arithmetic of dsrg_prepare_net_input_*)
 *   cues_out   : [B][K][H][W] float32 0/1, cues[v, y, x] = 1 for every pixel with value v != ignore_label
 *   labels_out : [B][1][1][K] float32 0/1, 1 for every value present other than ignore_label (label 0 is not forced)
 * K is the engine's M (81 for COCO).  The arrays of image pointers, Hs, Ws, flip and mean_pixel live on the host in
 * both variants.  The images are staged through a table in device memory, so B is bounded by the engine only.
 * A label value v >= K other than ignore_label is what numpy refuses with IndexError:
 *   _host: DSRG_E_INVALID before any copy or launch, with numpy's message ("index 90 is out of bounds for axis 0
 *          with size 81") for the first such pixel, image by image in raster order.
 *   _dev : such pixels are skipped (no cue plane, no tag; nothing is written out of bounds).  bad_out_dev [B] int32
 *          (may be NULL) receives per image the raster index, in the label map as given (before the mirror), of the
 *          first such pixel, or -1 if there is none; the caller checks it once the stream has run.
 */
int dsrg_annotation_coco_forward_dev(dsrg_engine *e, const uint8_t *const *images_dev, const int *Hs, const int *Ws,
                                     int B, const uint8_t *label_maps_dev, const int32_t *flip, int new_h, int new_w,
                                     const double *mean_pixel /* host, 3 */, int ignore_label, float *labels_out_dev,
                                     float *cues_out_dev, float *images_out_dev, int32_t *bad_out_dev, void *stream);
int dsrg_annotation_coco_forward_host(dsrg_engine *e, const uint8_t *const *images_host, const int *Hs,
                                      const int *Ws, int B, const uint8_t *label_maps_host, const int32_t *flip,
                                      int new_h, int new_w, const double *mean_pixel /* host, 3 */, int ignore_label,
                                      float *labels_out_host, float *cues_out_host, float *images_out_host);

/*
 * ImageSegDataLayer.forward (pylayers/pylayers/layer.py:51-61, SimpleTransformer.preprocess :169-236), the stage-2
 * training input of training/experiment/seed_mc/train-f.prototxt, after the caller has decoded the files and drawn
 * the random numbers (the shuffle, the two randints and the mirror) in the reference's order.  Per image b:
 *   images[b] : [Hs[b]][Ws[b]][3] uint8 BGR, as cv2.imread(..., IMREAD_COLOR) returns it; each image has its own size
 *   labels[b] : [Hl[b]][Wl[b]] uint8, as cv2.imread(..., IMREAD_GRAYSCALE) returns it.  labels == NULL: image only
 *               (preprocess(image), pre_test_image); Hl, Wl and labels_out are then not read
 *   h_off[b], w_off[b] : top-left corner of the crop_h x crop_w window in the padded arrays
 *   flip [B] or NULL : 1 = the window is read right to left (flip == -1, :231-234)
 * The padding is max(crop - size, 0) rows and columns at the bottom and right, from the label's size (the image's
 * without labels); the image gets the same.  ->
 *   images_out : [B][3][crop_h][crop_w] float32: float32(double(v) - mean[c]) * float32 scale inside the image
 *                (channel 2 - c of the pixel when swap_rb, else channel c), 0.0 in the padding
 *   labels_out : [B][1][crop_h][crop_w] float32: the label inside it, pad_label in the padding.  pad_label is
 *                saturate_cast<uchar>(ignore_label), what cv2.copyMakeBorder pads a uint8 label with
 * The arrays of pointers, sizes, offsets, flip and mean live on the host in both variants.  The images are read
 * through a table in device memory, so B is bounded by the engine only; the engine's shape, labels and retained
 * marginals are neither read nor changed, so the smallest engine (1 x 1, one label, max_batch = B) serves.
 * A negative offset, a window that leaves the padded image or the padded label (where the reference's slice comes
 * back short and numpy refuses to store it) or a pad_label outside 0..255 returns DSRG_E_INVALID before any copy or
 * launch.
 */
int dsrg_seg_data_forward_dev(dsrg_engine *e, const uint8_t *const *images_dev, const int *Hs, const int *Ws,
                              const uint8_t *const *labels_dev, const int *Hl, const int *Wl, int B, const int *h_off,
                              const int *w_off, const int32_t *flip, int crop_h, int crop_w,
                              const double *mean /* host, 3 */, float scale, int swap_rb, int pad_label,
                              float *images_out_dev, float *labels_out_dev, void *stream);
int dsrg_seg_data_forward_host(dsrg_engine *e, const uint8_t *const *images_host, const int *Hs, const int *Ws,
                               const uint8_t *const *labels_host, const int *Hl, const int *Wl, int B,
                               const int *h_off, const int *w_off, const int32_t *flip, int crop_h, int crop_w,
                               const double *mean /* host, 3 */, float scale, int swap_rb, int pad_label,
                               float *images_out_host, float *labels_out_host);

/* ------------------------------------------------------------------------------------------
 * Confusion matrix of a segmentation run, the scoring step of the evaluation tools:
 *   ConfusionMatrix (training/tools/evaluate.py:17-68, ap.py:19-72); its generateM (:61-68 / :65-72) counts
 *     m[gt[i], pred[i]] += 1 for every pixel with gt[i] < nclass, one Python iteration per pixel
 *   get_confusion_matrix (training/tools/test-coco.py:62-81): the same matrix via np.bincount(gt * K + pred)
 * An object owns a K x K uint64 matrix on `device` (-1: dsrg_current_device()), K <= DSRG_MAX_LABELS_WIDE, and
 * two uint64 counters of pixels that are not binned:
 *   invalid[0] : gt >= K other than 255 (the ignore label); such pixels are skipped, as generateM skips them
 *   invalid[1] : gt < K but pred outside [0, K) (numpy raises IndexError there; the Python layer raises)
 * The counts are exact and independent of the order of the calls.  Unlike test-coco.py, gt * K is never computed in
 * uint8: that product wraps mod 256 there for K = 81 (gt = 4, pred = 4 lands in bin 72).
 * Every call restores the caller's current device.
 * ------------------------------------------------------------------------------------------ */
typedef struct dsrg_confusion dsrg_confusion;

dsrg_confusion *dsrg_confusion_create(int device, int K);      /* ConfusionMatrix(nclass), evaluate.py:19-22 */
void dsrg_confusion_destroy(dsrg_confusion *c);
/* zero the matrix and the counters, queued on `stream` */
int dsrg_confusion_reset(dsrg_confusion *c, void *stream);
/* generateM over n pixels and accumulate (ConfM.addM(m) of evaluate.py:155-156): gt uint8, pred uint8 (pred_bytes
 * 1, a prediction PNG read back, evaluate.py:144) or int32 (4, the result of dsrg_predict_mask_dev).  Device
 * pointers may have any offset (int32 pred: 4-byte aligned); queued on `stream`. */
int dsrg_confusion_add_dev(dsrg_confusion *c, size_t n, const uint8_t *gt_dev, const void *pred_dev,
                           int pred_bytes /* 1 or 4 */, void *stream);
/* the same from host memory, streamed in chunks through the object's pinned staging (the copy of chunk k+1
 * overlaps the counting of chunk k); returns when the pixels are counted */
int dsrg_confusion_add_host(dsrg_confusion *c, size_t n, const uint8_t *gt, const void *pred, int pred_bytes);
/* wait for every add / reset so far and copy the K*K matrix (row = gt, column = pred) and the 2 invalid counters
 * out; either pointer may be NULL */
int dsrg_confusion_read(dsrg_confusion *c, uint64_t *matrix_out /* K*K */, uint64_t *invalid_out /* 2 */);

/* Host-only helpers of the *_host wire format (0/1 planes cross PCIe as 1 bit per value, see
 * csrc/wire.cu); exported for unit tests.  pack returns 1 if every value was exactly 0 or 1. */
int dsrg_wire_pack_mask(const float *src_host, uint32_t *dst_bits, size_t n);
void dsrg_wire_unpack_mask(const uint32_t *src_bits, float *dst_host, size_t n);
void dsrg_wire_apply_clamp_mask(const uint32_t *src_bits, float *probs_host, size_t n);

/*
 * CRFLayer.forward body (pylayers.py:63-88): same refinement, output log(result).
 *   log_out_dev : [B][M][H][W] float32 = log(renormalised marginals)
 *   result_dev  : optional [B][M][H][W] float32 copy of the marginals kept for backward (:90-92)
 */
int dsrg_crflayer_forward_dev(dsrg_engine *e, int B, float *probs_dev, const uint8_t *image_dev,
                              const dsrg_crf_params *params, float *log_out_dev,
                              float *result_dev, void *stream);

int dsrg_crflayer_forward_host(dsrg_engine *e, int B, float *probs_host, const uint8_t *image_host,
                               const dsrg_crf_params *params, float *log_out_host,
                               float *result_host);
/*
 * CRFLayer.backward (pylayers.py:90-92): grad = (1 - result) * top_diff over [B][M][H][W] float32, each element
 * rounded like numpy's float32 arithmetic (no contraction to FMA), so it is bit-identical to the reference's
 * statement on the same arrays.  result_dev is what dsrg_crflayer_forward_dev wrote to its `result` argument; the
 * batch size follows the two arrays it describes.
 */
int dsrg_crflayer_backward_dev(dsrg_engine *e, const float *result_dev, const float *top_diff_dev, int B,
                               float *grad_out_dev, void *stream);

/*
 * One refinement, two consumers.  In the reference's net CRFLayer and DSRGLayer are fed the same two blobs
 * (train-s.prototxt:758-786) and each runs the whole dense CRF on them (pylayers.py:82 and :326).  The raw
 * marginals of an engine's last mean-field pass stay on the device; these entry points let a second consumer
 * use them instead of repeating the pass:
 *   dsrg_srg_last_crf_host       : generate_seed_step over the batch on those marginals (float64 clamp +
 *                                  renormalisation fused in, exactly what dsrg_dsrg_forward_* does after its CRF)
 *   dsrg_srg_last_crf_dev        : the same on device arrays, queued on the caller's stream (no host
 *                                  synchronisation; labels [B][M], cues / seeds_out [B][M][H][W]); the batch
 *                                  size follows the arrays it describes
 *   dsrg_crf_last_marginals_host : the raw float32 marginals themselves
 * All return DSRG_E_STATE unless the engine's last pass was a CRF over exactly B images.
 */
int dsrg_srg_last_crf_host(dsrg_engine *e, int B, const float *labels_host, const float *cues_host, double th1,
                           double th2, float *seeds_out_host);
int dsrg_srg_last_crf_dev(dsrg_engine *e, const float *labels_dev, const float *cues_dev, int B, double th1,
                          double th2, float *seeds_out_dev, void *stream);
int dsrg_crf_last_marginals_host(dsrg_engine *e, int B, float *out_host, int out_layout);

/*
 * BalancedSeedLossLayer (pylayers.py:120-152).  Forward writes the LOCAL sums
 *   terms_out[0] = sum_n S_bg(n) / max(cnt_bg(n), 1e-4),  terms_out[1] = same for fg
 * so that loss = -(terms[0] + terms[1]) / N_global; with several GPUs the two floats are
 * all-reduced (SUM) first -- the only collective on the path.  Backward writes
 *   grad = top_diff * d loss / d probs = -top_diff * lab / (p * max(cnt,1e-4) * N_global).
 */
int dsrg_seedloss_forward_dev(dsrg_engine *e, int B, const float *probs_dev,
                              const float *seeds_dev, float *terms_out_dev, void *stream);
int dsrg_seedloss_backward_dev(dsrg_engine *e, int B, int n_global, const float *probs_dev,
                               const float *seeds_dev, float top_diff, float *grad_out_dev,
                               void *stream);

int dsrg_seedloss_forward_host(dsrg_engine *e, int B, const float *probs_host,
                               const float *seeds_host, float *terms_out_host /* 2 floats */);
int dsrg_seedloss_backward_host(dsrg_engine *e, int B, int n_global, const float *probs_host,
                                const float *seeds_host, float top_diff, float *grad_out_host);

/*
 * SeedLossLayer (pylayers.py:95-118), SEC's plain seeding loss: loss = -mean_n S(n) / cnt(n) with
 * S(n) = sum_{c,h,w} lab log p and cnt(n) = sum lab -- no max(cnt, 1e-4) floor, so an image without seeds gives
 * NaN like the reference.  Forward writes the LOCAL sum terms_out[0] = sum_n S(n) / cnt(n), so that
 * loss = -terms[0] / N_global.  Backward writes d loss / d probs = -lab / (p * cnt * N_global); the layer's top
 * diff is not applied (the reference ignores it).
 */
int dsrg_seedloss_plain_forward_dev(dsrg_engine *e, int B, const float *probs_dev, const float *seeds_dev,
                                    float *terms_out_dev /* 1 float */, void *stream);
int dsrg_seedloss_plain_backward_dev(dsrg_engine *e, int B, int n_global, const float *probs_dev,
                                     const float *seeds_dev, float *grad_out_dev, void *stream);
int dsrg_seedloss_plain_forward_host(dsrg_engine *e, int B, const float *probs_host, const float *seeds_host,
                                     float *terms_out_host /* 1 float */);
int dsrg_seedloss_plain_backward_host(dsrg_engine *e, int B, int n_global, const float *probs_host,
                                      const float *seeds_host, float *grad_out_host);

/*
 * ExpandLossLayer (pylayers.py:183-233), SEC's expansion loss by global weighted rank pooling (GWRP).  probs
 * [B][M][H][W] (channel 0 = background), labels [B][M] (the N x 1 x 1 M labels blob; class k >= 1 is present when
 * labels > 0.5).  G_q(x) = sum_i sort(x)_i q^(n-1-i) / Z, Z = sum_i q^i, n = H*W <= DSRG_GWRP_MAX_PLANE; the
 * reference's q_fg = 0.996, q_bg = 0.999 (:200, :207).  Forward writes the LOCAL sums
 *   terms_out[0] = sum_n sum_k s_k log G_fg(p_k) / P,  terms_out[1] = sum_n sum_k (1-s_k) log(1 - max p_k) / A,
 *   terms_out[2] = sum_n log G_bg(p_0)
 * (P, A: present / absent foreground classes of image n), so that loss = -(terms[0]+terms[1]+terms[2]) / N_global.
 * Backward writes d loss / d probs as Theano's T.grad forms it: through the sort permutation and, IN FULL, to every
 * element equal to a plane's max; P = 0 or A = 0 makes the loss NaN and the image's foreground gradient NaN.
 * Both are deterministic: two identical calls give bit-identical results.
 */
int dsrg_expandloss_forward_dev(dsrg_engine *e, int B, const float *probs_dev, const float *labels_dev, double q_fg,
                                double q_bg, float *terms_out_dev /* 3 floats */, void *stream);
int dsrg_expandloss_backward_dev(dsrg_engine *e, int B, int n_global, const float *probs_dev,
                                 const float *labels_dev, double q_fg, double q_bg, float *grad_out_dev,
                                 void *stream);
int dsrg_expandloss_forward_host(dsrg_engine *e, int B, const float *probs_host, const float *labels_host,
                                 double q_fg, double q_bg, float *terms_out_host /* 3 floats */);
int dsrg_expandloss_backward_host(dsrg_engine *e, int B, int n_global, const float *probs_host,
                                  const float *labels_host, double q_fg, double q_bg, float *grad_out_host);

/* Optional per-kernel timing for the roofline report: while enabled every kernel launch of the
 * engine is bracketed by CUDA events on its launching stream.  dsrg_engine_profile_read()
 * synchronises the device and returns, per kernel class (dsrg_profile_tag_count() of them, named by
 * dsrg_profile_tag_name()), the summed milliseconds and the number of launches since the last read. */
int dsrg_profile_tag_count(void);
const char *dsrg_profile_tag_name(int tag);
int dsrg_engine_profile(dsrg_engine *e, int enable);
int dsrg_engine_profile_read(dsrg_engine *e, float *ms_out, long long *count_out);

/* Introspection used by the lattice-level parity tests: vertex counts of the lattices built by
 * the last CRF call (spatial, then bilateral per image); either pointer may be NULL. */
int dsrg_engine_lattice_sizes(dsrg_engine *e, int B, int *v_spatial_out, int *v_bilateral_out);
/* Image b's lattice tables of the last CRF call (which = 0 spatial, shared by the batch; 1 bilateral), in the
 * engine's vertex numbering: off_out [d+1][N] the 1-based row of every (r, pixel) (0 is the zero row), nbr_out
 * [d+1][V+1][2] the two blur neighbours of rows 0..V (V from dsrg_engine_lattice_sizes) as rows of the same image,
 * 0 for a missing one.  Either pointer may be NULL.  For tests. */
int dsrg_engine_lattice_tables(dsrg_engine *e, int which, int b, int *off_out, int *nbr_out);
/* Per-pixel symmetric normalisation vectors (DenseKernel::norm_, pairwise.cpp:54-57) of the
 * last CRF call: which = 0 spatial [N] (shared by the batch), 1 bilateral [B][N]. */
int dsrg_engine_copy_norm(dsrg_engine *e, int which, int B, float *norm_out_host);

/* ------------------------------------------------------------------------------------------
 * Per-object API with the exact surface of the reference's C++ class DenseCRFWrapper
 * (CRF/include/densecrf_wrapper.h:3-28), which krahenbuhl2013/wrapper.pyx:20-60 binds.
 * Host pointers, borrowed for the duration of the call, like the original.  Creating an object is cheap
 * (the reference makes one per image, CRF.py:21): it allocates nothing on the device.
 * ------------------------------------------------------------------------------------------ */
typedef struct dsrg_densecrf dsrg_densecrf;

dsrg_densecrf *dsrg_densecrf_create(int W, int H, int nlabels);            /* densecrf_wrapper.cpp:5-8   */
void dsrg_densecrf_destroy(dsrg_densecrf *c);                              /* :10-12                     */
int dsrg_densecrf_npixels(const dsrg_densecrf *c);                         /* :14                        */
int dsrg_densecrf_nlabels(const dsrg_densecrf *c);                         /* :15                        */
int dsrg_densecrf_set_unary_energy(dsrg_densecrf *c, const float *unary_costs); /* :32-37, [N][M] energies */
int dsrg_densecrf_add_pairwise_energy(dsrg_densecrf *c, float w1, float theta_alpha_1,
                                      float theta_alpha_2, float theta_betta_1, float theta_betta_2,
                                      float theta_betta_3, float w2, float theta_gamma_1,
                                      float theta_gamma_2, const unsigned char *im);  /* :18-30 */
int dsrg_densecrf_map(dsrg_densecrf *c, int n_iters, int *labels);         /* :39-43 */
int dsrg_densecrf_inference(dsrg_densecrf *c, int n_iters, float *probs_out); /* :45-50 */
/* The objects borrow a process-wide engine per label count (created on first use, grown to the largest image
 * seen, serialised by a mutex); this frees those engines' device memory. */
void dsrg_densecrf_release_engines(void);

#ifdef __cplusplus
}
#endif
#endif /* DSRG_B200_H */
