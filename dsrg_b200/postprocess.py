"""Inference pre- and post-processing of the reference's evaluation tools on the GPU: the network input of every
scale (preprocess(), training/tools/test-ms.py:68-81) and everything predict_mask() does after net.forward()
(training/tools/test-ms.py:84-111, training/tools/generate_train_gt.py:76-104).
The network forward pass stays with the caller; pass the fc8 score blobs as they come out of
``net.blobs['fc8-SEC'].data[0]`` ((M, h, w) float32).  No CPU fallback: needs the CUDA library."""
import numpy as np

from . import api as _api
from ._lib import PREP_IMAGES_PER_LAUNCH as _PREP_IMAGES_PER_LAUNCH
from .pool import batch_capacity as _batch_capacity
from .pool import batch_engine_for as _batch_engine_for
from .pool import engine_for as _engine_for
from .pool import prep_engine_for as _prep_engine_for

EPS = 0.00001  # test-ms.py:103, generate_train_gt.py:90
_PREP_MAX_SCALES = 16   # DSRG_PREP_MAX_SCALES
_MAX_PLANE = 2 ** 31 - 1  # pixels of one image or network-input plane
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


def net_input_shapes(image_sizes, sizes, relative=False):
    """The (h, w) of every size of `sizes` for a list of (H, W) image sizes, which must agree across the list: one
    network batch per size.  Absolute sizes (size / H, size / W) always give (size, size); zoom factors give one
    shape only to images of one size.  ValueError otherwise, or when a scale rounds to no rows or columns."""
    image_sizes = [tuple(int(v) for v in hw) for hw in image_sizes]
    sizes = list(sizes)
    if not image_sizes or not 1 <= len(sizes) <= _PREP_MAX_SCALES:
        raise ValueError("need at least one image and 1 to %d sizes (got %d images, %d sizes)"
                         % (_PREP_MAX_SCALES, len(image_sizes), len(sizes)))
    if min(min(hw) for hw in image_sizes) < 1 or max(h * w for h, w in image_sizes) > _MAX_PLANE:
        raise ValueError("every image needs at least one row and column and fewer than 2^31 pixels")
    shapes = [net_input_size(image_sizes[0][0], image_sizes[0][1], s, relative) for s in sizes]
    for H, W in image_sizes[1:]:
        other = [net_input_size(H, W, s, relative) for s in sizes]
        if other != shapes:
            raise ValueError("sizes %s give a %dx%d image the network inputs %s but a %dx%d image %s: one batch needs "
                             "one shape per size" % (sizes, image_sizes[0][0], image_sizes[0][1], shapes, H, W, other))
    if min(min(s) for s in shapes) < 1 or max(h * w for h, w in shapes) > _MAX_PLANE:
        raise ValueError("every scale must give at least one row and column and fewer than 2^31 pixels (got %s)"
                         % shapes)
    return shapes


def prep_launches(B):
    """Kernel launches of one preprocess_batch* call of B images: DSRG_PREP_IMAGES_PER_LAUNCH images per launch."""
    return -(-int(B) // _PREP_IMAGES_PER_LAUNCH)


def _check_batch_args(M, mean_pixel):
    if not 1 <= int(M) <= 255:
        raise ValueError("M must lie in [1, 255], not %d" % M)
    mean = np.asarray(mean_pixel, np.float64)
    if mean.shape != (3,):
        raise ValueError("mean_pixel must have 3 elements")
    return mean


def preprocess_batch(ims, sizes, relative=False, M=21, mean_pixel=MEAN_PIXEL):
    """preprocess(image, size) for a list of uint8 (H_i, W_i, 3) images of any sizes, every size of `sizes` in one
    launch: one (B, 3, h, w) float32 array per size, which a Caffe tool can hand to one forward pass after
    net.blobs['images'].reshape(B, 3, h, w).  Image b of each is bit-identical to preprocess(ims[b], sizes).  With
    `relative` zoom factors every image must give the same shape (ValueError otherwise).  M is the label count
    preprocess() takes; the network input does not depend on it, and the call runs on an engine of its own that
    grows in batch only, so no post-processing engine grows to the largest image of the list."""
    ims = list(ims)
    for im in ims:
        if not isinstance(im, np.ndarray) or im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
            raise ValueError("every image must be a uint8 (H, W, 3) array")
    mean = _check_batch_args(M, mean_pixel)
    shapes = net_input_shapes([im.shape[:2] for im in ims], sizes, relative)
    from . import _lib
    eng = _prep_engine_for(len(ims), _lib.lib().dsrg_current_device())
    return eng.prepare_net_input_batch_host([np.ascontiguousarray(im) for im in ims], shapes, mean)


def preprocess_batch_dev(images, sizes, relative=False, M=21, mean_pixel=MEAN_PIXEL, out=None):
    """preprocess_batch on the device, queued on the current CUDA stream of the images' device without a host
    synchronisation (so it can be captured in a CUDA graph once a batch of this size has run):
      images : a contiguous (B, H, W, 3) uint8 CUDA tensor, or a list of B contiguous (H_i, W_i, 3) ones on one device
      out    : optional list of one contiguous (B, 3, h, w) float32 tensor per size to write into
    Returns one (B, 3, h, w) float32 tensor per size.  Every argument is checked (ValueError) before anything is
    queued."""
    import torch
    if isinstance(images, torch.Tensor):
        if not (images.is_cuda and images.dtype == torch.uint8 and images.dim() == 4 and images.shape[3] == 3
                and images.is_contiguous() and images.shape[0] > 0):
            raise ValueError("images must be a contiguous (B, H, W, 3) uint8 CUDA tensor")
        images = list(images.unbind(0))
    else:
        images = list(images)
        if not images:
            raise ValueError("need at least one image")
    dev = images[0].device if isinstance(images[0], torch.Tensor) else None
    for im in images:
        if not (isinstance(im, torch.Tensor) and im.is_cuda and im.device == dev and im.dtype == torch.uint8
                and im.dim() == 3 and im.shape[2] == 3 and im.is_contiguous()):
            raise ValueError("every image must be a contiguous (H, W, 3) uint8 CUDA tensor, all on one device")
    mean = _check_batch_args(M, mean_pixel)
    shapes = net_input_shapes([im.shape[:2] for im in images], sizes, relative)
    B = len(images)
    if out is None:
        out = [torch.empty((B, 3, h, w), dtype=torch.float32, device=dev) for h, w in shapes]
    else:
        out = list(out)
        if len(out) != len(shapes) or any(
                not (isinstance(o, torch.Tensor) and o.device == dev and o.dtype == torch.float32
                     and tuple(o.shape) == (B, 3, h, w) and o.is_contiguous()) for o, (h, w) in zip(out, shapes)):
            raise ValueError("out must hold one contiguous float32 tensor on %s per size, of shapes %s"
                             % (dev, [(B, 3, h, w) for h, w in shapes]))
    eng = _prep_engine_for(B, dev.index)
    with torch.cuda.device(dev):
        eng.prepare_net_input_batch_dev(images, out, mean)
    return out


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


# ---- many images per pass ----

def _chunks(keys, batch):
    """Indices of `keys` grouped by equal key (groups in order of first appearance, indices ascending), each group
    cut into chunks of at most `batch`."""
    groups = {}
    for i, k in enumerate(keys):
        groups.setdefault(k, []).append(i)
    return [idx[a:a + batch] for idx in groups.values() for a in range(0, len(idx), batch)]


def _run_batched(ims, blobs_per_image, sels, mode, smooth, batch, return_probs):
    """Group the images by (H, W, score shapes), run each chunk as one batched pass, return per image in input
    order.  `sels`: None or one selection list per image."""
    n = len(ims)
    if len(blobs_per_image) != n or (sels is not None and len(sels) != n):
        raise ValueError("one set of score blobs%s per image" % ("" if sels is None else " and labels"))
    batch = int(batch)
    if batch < 1:
        raise ValueError("batch must be at least 1")
    shapes = []
    for im, blobs in zip(ims, blobs_per_image):
        shape = np.shape(im)
        if len(shape) != 3 or shape[2] != 3:
            raise ValueError("image must be (H, W, 3)")
        if not blobs or any(b.shape[0] != blobs[0].shape[0] for b in blobs):
            raise ValueError("every image needs at least one score blob, all with the same label count")
        shapes.append((tuple(shape[:2]), tuple(b.shape for b in blobs)))
    chunks = _chunks(shapes, batch)
    # size each label count's engine for the largest chunk and image once, so no chunk re-creates it
    need = {}
    for idx in chunks:
        (H, W), bs = shapes[idx[0]]
        B0, H0, W0 = need.get(bs[0][0], (0, 0, 0))
        need[bs[0][0]] = (max(B0, len(idx)), max(H0, H), max(W0, W))
    for M, (B0, H0, W0) in need.items():
        _batch_engine_for(B0, H0, W0, M)
    labels, probs = [None] * n, [None] * n
    params = _api.crf_params(1.0)
    for idx in chunks:
        (H, W), bs = shapes[idx[0]]
        M = bs[0][0]
        eng = _batch_engine_for(len(idx), H, W, M)
        scores = [np.stack([blobs_per_image[i][k] for i in idx]) for k in range(len(bs))]
        images = np.stack([_image(ims[i], True) for i in idx]) if smooth else None
        sel = None
        if sels is not None:
            sel = np.full((len(idx), M), -1, np.int32)
            for r, i in enumerate(idx):
                sel[r, :len(sels[i])] = sels[i]
        out = eng.predict_mask_batch_host(scores, images, params, mode, EPS, smooth, sel, return_probs)
        res, pr = out if return_probs else (out, None)
        for r, i in enumerate(idx):
            labels[i] = res[r].astype(np.int64)
            if return_probs:
                probs[i] = pr[r]
    return (labels, probs) if return_probs else labels


def predict_masks_ms(ims, scores_per_image, smooth=True, batch=16, return_probs=False):
    """predict_mask_ms over a list of images, up to `batch` of them per device pass: ims[i] is an (H,W,3) image and
    scores_per_image[i] its list of (M,h,w) score blobs, of any sizes.  Images with the same (H, W) and score shapes
    share passes.  Returns the list of (H,W) int64 label maps in input order [and the list of (H,W,M) float32
    probabilities].  With smooth=False the results are bit-identical to predict_mask_ms image by image."""
    blobs = [[_blob(s) for s in sc] for sc in scores_per_image]
    return _run_batched(list(ims), blobs, None, _api.POST_SUM_SCORES, smooth, batch, return_probs)


def predict_masks_gt(ims, scores, labels_per_image, smooth=True, batch=16):
    """predict_mask_gt over a list of images, up to `batch` of them per device pass: scores[i] is image i's (M,h,w)
    blob and labels_per_image[i] its tags.  Returns the list of (H,W) int64 label maps in input order."""
    blobs = [[_blob(s)] for s in scores]
    sels = []
    for blob, tags in zip(blobs, labels_per_image):
        M = blob[0].shape[0]
        sel = [0] + [int(v) for v in np.asarray(tags).reshape(-1).tolist()]   # generate_train_gt.py:96-97
        if min(sel) < 0 or max(sel) >= M:
            raise ValueError("label ids must lie in [0, %d), got %s" % (M, sel))
        # a repeated id can never be the first maximum again: keeping only its first occurrence changes nothing
        sels.append(list(dict.fromkeys(sel)))
    return _run_batched(list(ims), blobs, sels, _api.POST_ZOOM_PROBS, smooth, batch, False)


_MODES = {"ms": _api.POST_SUM_SCORES, "gt": _api.POST_ZOOM_PROBS}


def _learned(ref, B, M, H, W, kw):
    """(params, features, compat) of the learned-CRF keywords in kw that are given, checked as nn.dense_crf_inference
    checks them, with the weights and sigmas read on the host once; None when none is given (CRF()'s own pass)."""
    kw = {k: v for k, v in kw.items() if v is not None}
    if not kw:
        return None
    from . import nn as _nn
    params = _api.crf_params(1.0)
    feats, compat = _nn._learned_crf(ref, B, M, H, W, params, **kw)
    return params, feats, compat


def _smooth_for(smooth, kw):
    given = sorted(k for k, v in kw.items() if v is not None)
    if given and not smooth:
        raise ValueError("%s configure the CRF: they need smooth=True" % ", ".join(given))


def predict_mask_batch_dev(images, scores, labels=None, mode="ms", smooth=True, out=None, *, w1=None, w2=None,
                           compat_bi=None, compat_sp=None, theta_bi=None, theta_sp=None, features_bi=None):
    """The post-processing of a batch that never leaves the device, queued on the current CUDA stream (so it can be
    captured in a CUDA graph).
      images : (B,H,W,3) uint8 CUDA tensor
      scores : list of (B,M,h,w) float32 CUDA tensors, one batched forward per scale ("ms": 1 to 16 of them,
               test-ms.py; "gt": exactly one, generate_train_gt.py)
      labels : optional (B,M) or (B,1,1,M) 0/1 tag tensor (the labels blob): image b's arg-max runs over label 0 and
               the labels tagged > 0.5, in ascending order.  The selection is built on the device, without a host
               synchronisation, and read when the pass runs
      out    : optional (B,H,W) int32 CUDA tensor to write into (a fixed output lets the engine replay its own graph)
    Returns the (B,H,W) int32 label maps, which api.Confusion.add_dev counts directly.  Every argument is checked
    (ValueError) before anything is queued.

    The keyword-only arguments run the learned CRF of nn.dense_crf_inference in place of CRF()'s, with the meanings
    they have there (smooth only): the Potts weights w1 / w2 or the matrices compat_bi / compat_sp, the bandwidths
    theta_bi / theta_sp and the bilateral features features_bi ((B, 5, H, W) float32; the images then give only the
    shape).  The sigmas are absolute, at the image's resolution: a CRF learned on 41x41 maps with scale factor 12
    passes theta * 12.  An image whose feature lattice leaves the packed key range gets -1 in every pixel.  With all
    of them None the pass is CRF()'s, as before."""
    kw = dict(w1=w1, w2=w2, compat_bi=compat_bi, compat_sp=compat_sp, theta_bi=theta_bi, theta_sp=theta_sp,
              features_bi=features_bi)
    _smooth_for(smooth, kw)
    return _predict_mask_batch(images, scores, labels, mode, smooth, out,
                               lambda B, M, H, W: _learned(images, B, M, H, W, kw))


def _predict_mask_batch(images, scores, labels, mode, smooth, out, learned):
    """predict_mask_batch_dev's pass; learned(B, M, H, W) checks and resolves the learned CRF (see _learned) once the
    shapes are known, before anything is queued."""
    import torch
    if mode not in _MODES:
        raise ValueError("mode must be 'ms' or 'gt', not %r" % (mode,))
    if not (isinstance(images, torch.Tensor) and images.is_cuda and images.dtype == torch.uint8 and images.dim() == 4
            and images.shape[3] == 3 and images.is_contiguous()):
        raise ValueError("images must be a contiguous (B, H, W, 3) uint8 CUDA tensor")
    B, H, W = (int(v) for v in images.shape[:3])
    dev = images.device
    scores = list(scores)
    if not 1 <= len(scores) <= 16 or (mode == "gt" and len(scores) != 1):
        raise ValueError("mode %r takes %s score tensors, got %d" % (mode, "1" if mode == "gt" else "1 to 16",
                                                                     len(scores)))
    for s in scores:
        if not (isinstance(s, torch.Tensor) and s.device == dev and s.dtype == torch.float32 and s.dim() == 4
                and s.is_contiguous() and s.shape[0] == B and s.shape[1] == scores[0].shape[1] and min(s.shape) > 0):
            raise ValueError("every score map must be a contiguous (B, M, h, w) float32 tensor on %s with B = %d and "
                             "one M" % (dev, B))
    M = int(scores[0].shape[1])
    if B < 1 or H < 1 or W < 1 or M > 255:
        raise ValueError("need B, H, W >= 1 and at most 255 labels (got B=%d, %dx%d, M=%d)" % (B, H, W, M))
    if labels is not None and not (isinstance(labels, torch.Tensor) and labels.device == dev and
                                   tuple(labels.shape) in ((B, M), (B, 1, 1, M))):
        raise ValueError("labels must be a (B, M) or (B, 1, 1, M) tensor on %s" % dev)
    if out is not None and not (isinstance(out, torch.Tensor) and out.device == dev and out.dtype == torch.int32
                                and tuple(out.shape) == (B, H, W) and out.is_contiguous()):
        raise ValueError("out must be a contiguous (B, H, W) int32 tensor on %s" % dev)
    resolved = learned(B, M, H, W)
    eng = _batch_engine_for(B, H, W, M, dev.index)
    hc, wc = eng.capacity
    for s in scores:
        if s.shape[2] * s.shape[3] > hc * wc:
            raise ValueError("score map %dx%d has more pixels than the engine holds (%d)" % (s.shape[2], s.shape[3],
                                                                                           hc * wc))
    sel = None
    if labels is not None:
        present = labels.reshape(B, M) > 0.5
        present[:, 0] = True
        ids = torch.arange(M, device=dev, dtype=torch.int32).expand(B, M)
        order = torch.sort(torch.where(present, ids, ids + M), dim=1).values   # tagged ids first, ascending
        sel = torch.where(order < M, order, torch.full_like(order, -1)).contiguous()
    if out is None:
        out = torch.empty((B, H, W), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        if resolved is not None:
            params, feats, compat = resolved
            eng.predict_mask_batch_learned_dev(scores, None if feats is not None else images, out, params,
                                               _MODES[mode], EPS, features=feats, compat=compat, sel=sel)
        else:
            eng.predict_mask_batch_dev(scores, images, out, _api.crf_params(1.0), _MODES[mode], EPS, smooth, sel)
    return out


def predict_masks_dev(images, scores, labels=None, mode="ms", smooth=True, *, w1=None, w2=None, compat_bi=None,
                      compat_sp=None, theta_bi=None, theta_sp=None, features_bi=None):
    """predict_mask_batch_dev over a batch of images of mixed sizes, the device analogue of predict_masks_ms /
    predict_masks_gt after one batched forward per scale (preprocess_batch_dev gives every image the same network
    input shape):
      images : list of B contiguous (H_i, W_i, 3) uint8 CUDA tensors on one device
      scores : list of (B, M, h, w) float32 CUDA tensors, one per scale ("ms": 1 to 16, "gt": exactly one)
      labels : optional (B, M) or (B, 1, 1, M) 0/1 tag tensor, as for predict_mask_batch_dev
    The images are grouped by (H, W) on the host from the tensor shapes; each group's rows are gathered with
    torch.stack over views (nothing is copied from the host) and run as one predict_mask_batch_dev pass.  Returns the
    (H_i, W_i) int32 label maps in input order, queued on the current stream.  Every argument is checked (ValueError)
    before anything is queued.  The batch engine's capacity is ensured once for the largest group and image (outside
    a capture: run the largest batch and image once first); each group then selects its size without waiting for
    the device (dsrg_engine_set_size_ordered), so nothing synchronises the host and a call can be captured.
    The keyword-only arguments are predict_mask_batch_dev's learned CRF; features_bi is then a list of (5, H_i, W_i)
    float32 tensors aligned with images, grouped with them.  They are checked, and a weight or sigma tensor read on the
    host, once per call."""
    import torch
    kw = dict(w1=w1, w2=w2, compat_bi=compat_bi, compat_sp=compat_sp, theta_bi=theta_bi, theta_sp=theta_sp)
    _smooth_for(smooth, dict(kw, features_bi=features_bi))
    if mode not in _MODES:
        raise ValueError("mode must be 'ms' or 'gt', not %r" % (mode,))
    images = list(images)
    if not images or not isinstance(images[0], torch.Tensor):
        raise ValueError("images must be a non-empty list of CUDA tensors")
    dev = images[0].device
    for im in images:
        if not (isinstance(im, torch.Tensor) and im.is_cuda and im.device == dev and im.dtype == torch.uint8
                and im.dim() == 3 and im.shape[2] == 3 and min(im.shape) > 0 and im.is_contiguous()):
            raise ValueError("every image must be a contiguous (H, W, 3) uint8 CUDA tensor, all on one device")
    B = len(images)
    scores = list(scores)
    if not 1 <= len(scores) <= 16 or (mode == "gt" and len(scores) != 1):
        raise ValueError("mode %r takes %s score tensors, got %d" % (mode, "1" if mode == "gt" else "1 to 16",
                                                                     len(scores)))
    for s in scores:
        if not (isinstance(s, torch.Tensor) and s.device == dev and s.dtype == torch.float32 and s.dim() == 4
                and s.is_contiguous() and s.shape[0] == B and s.shape[1] == scores[0].shape[1] and min(s.shape) > 0):
            raise ValueError("every score map must be a contiguous (B, M, h, w) float32 tensor on %s with B = %d and "
                             "one M" % (dev, B))
    M = int(scores[0].shape[1])
    if M > 255:
        raise ValueError("at most 255 labels, not %d" % M)
    if labels is not None and not (isinstance(labels, torch.Tensor) and labels.device == dev and
                                   tuple(labels.shape) in ((B, M), (B, 1, 1, M))):
        raise ValueError("labels must be a (B, M) or (B, 1, 1, M) tensor on %s" % dev)
    sizes = [tuple(int(v) for v in im.shape[:2]) for im in images]
    if features_bi is not None:
        features_bi = list(features_bi)
        if len(features_bi) != B or any(
                not (isinstance(f, torch.Tensor) and f.device == dev and f.dtype == torch.float32
                     and tuple(f.shape) == (5,) + hw) for f, hw in zip(features_bi, sizes)):
            raise ValueError("features_bi must be a list of %d float32 tensors on %s, of shapes %s"
                             % (B, dev, [(5,) + hw for hw in sizes]))
    resolved = _learned(images[0], B, M, 1, 1, kw)   # the features go with their group below
    if resolved is None and features_bi is not None:
        resolved = (_api.crf_params(1.0), None, None)
    groups = _chunks(sizes, B)
    need = (max(len(g) for g in groups), max(h for h, _ in sizes), max(w for _, w in sizes))
    _, hc, wc = _batch_capacity(*need, M, dev.index)
    for s in scores:
        if s.shape[2] * s.shape[3] > hc * wc:
            raise ValueError("score map %dx%d has more pixels than the engine holds (%d)" % (s.shape[2], s.shape[3],
                                                                                           hc * wc))
    # the engine's capacity once for the largest group and image, so no group re-creates it; each group then selects
    # its own size, stream-ordered
    _batch_engine_for(*need, M, dev.index, select=False)
    out = [None] * B
    for idx in groups:
        if idx == list(range(B)):   # one size: the caller's tensors as they are
            g_images, g_scores, g_labels = torch.stack(images), scores, labels
        else:
            g_images = torch.stack([images[i] for i in idx])
            g_scores = [torch.stack([s[i] for i in idx]) for s in scores]
            g_labels = None if labels is None else torch.stack([labels[i] for i in idx])
        g_learned = None
        if resolved is not None:
            g_features = None if features_bi is None else torch.stack([features_bi[i] for i in idx])
            g_learned = (resolved[0], g_features, resolved[2])
        res = _predict_mask_batch(g_images, g_scores, g_labels, mode, smooth, None, lambda *_: g_learned)
        for r, i in enumerate(idx):
            out[i] = res[r]
    return out
