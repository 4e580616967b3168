"""Inference pre- and post-processing of the reference's evaluation tools on the GPU: the network input of every
scale (preprocess(), training/tools/test-ms.py:68-81) and everything predict_mask() does after net.forward()
(training/tools/test-ms.py:84-111, training/tools/generate_train_gt.py:76-104).
The network forward pass stays with the caller; pass the fc8 score blobs as they come out of
``net.blobs['fc8-SEC'].data[0]`` ((M, h, w) float32).  No CPU fallback: needs the CUDA library."""
import numpy as np

from . import api as _api
from .pool import engine_for as _engine_for

EPS = 0.00001  # test-ms.py:103, generate_train_gt.py:90
MEAN_PIXEL = (104.0, 117.0, 123.0)  # test-ms.py:48 and the other tools


def net_input_size(H, W, size, relative=False):
    """The (h, w) of preprocess(image, size) for an H x W image: scipy's int(round(in * factor)) with Python's
    round, factor = size / float(in) (test-ms.py:73-74) or, with `relative`, the zoom factor itself
    (test-ms-f.py:105).  So 334 * 1.25 = 417.5 gives 418 and 334 * 0.75 = 250.5 gives 250."""
    fy, fx = (size, size) if relative else (size / float(H), size / float(W))
    return int(round(H * fy)), int(round(W * fx))


def preprocess(im, sizes, relative=False, M=21, mean_pixel=MEAN_PIXEL):
    """preprocess(image, size) of the evaluation tools (test-ms.py:68-81, test.py, test-coco.py, generate_train_gt.py,
    show-result.py; test-ms-f.py / test-coco-f.py with `relative` zoom factors) for every size of `sizes`, on the
    device in one launch: zoom(order=1), RGB -> BGR, - mean_pixel, HWC -> CHW, bit-exact with scipy.  `im` is the
    uint8 (H, W, 3) image as pylab.imread / cv2.imread return it.  Returns one (1, 3, h, w) float32 blob per size.
    Runs on the pooled engine that predict_mask_* with the same M will use for this image, so the post-processing
    that follows neither re-shapes the engine again nor drops its cached graphs."""
    if not isinstance(im, np.ndarray) or im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
        raise ValueError("image must be a uint8 (H, W, 3) array")
    mean = np.asarray(mean_pixel, np.float64)
    if mean.shape != (3,):
        raise ValueError("mean_pixel must have 3 elements")
    H, W = im.shape[:2]
    shapes = [net_input_size(H, W, s, relative) for s in sizes]
    if not shapes or min(min(s) for s in shapes) < 1:
        raise ValueError("every scale must give at least one row and column (got %s)" % shapes)
    eng = _engine_for(H, W, M)
    return eng.prepare_net_input_host(np.ascontiguousarray(im), shapes, mean)


def _blob(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.ndim != 3:
        raise ValueError("score blob must be (M, h, w)")
    return a


def _image(im, smooth):
    im = np.asarray(im)
    if im.ndim != 3 or im.shape[2] != 3:
        raise ValueError("image must be (H, W, 3)")
    return np.ascontiguousarray(im.astype('ubyte')) if smooth else None  # CRF.py:32


def predict_mask_ms(im, scores_per_scale, smooth=True, return_probs=False):
    """test-ms.py:84-111 after the forward passes: sum of zoomed score maps -> softmax -> clamp ->
    CRF(im, log(probs), scale_factor=1.0) -> argmax.  `scores_per_scale`: the (M,h,w) blobs of the
    241/321/401 passes (any number).  Returns the (H,W) label map (int64 like np.argmax)."""
    blobs = [_blob(s) for s in scores_per_scale]
    H, W = np.asarray(im).shape[:2]
    eng = _engine_for(H, W, blobs[0].shape[0])
    out = eng.predict_mask_host(blobs, _image(im, smooth), _api.crf_params(1.0), _api.POST_SUM_SCORES, EPS, smooth,
                                None, return_probs)
    if return_probs:
        return out[0].astype(np.int64), out[1]
    return out.astype(np.int64)


def predict_mask_gt(im, scores, labels, smooth=True, return_probs=False):
    """generate_train_gt.py:76-104 after net.forward(): softmax at network resolution -> zoom -> clamp ->
    CRF -> argmax restricted to [0] + labels, mapped back to label ids."""
    blob = _blob(scores)
    H, W = np.asarray(im).shape[:2]
    sel = [0] + [int(v) for v in np.asarray(labels).tolist()]   # :96-97
    eng = _engine_for(H, W, blob.shape[0])
    out = eng.predict_mask_host([blob], _image(im, smooth), _api.crf_params(1.0), _api.POST_ZOOM_PROBS, EPS, smooth,
                                sel, return_probs)
    if return_probs:
        return out[0].astype(np.int64), out[1]
    return out.astype(np.int64)
