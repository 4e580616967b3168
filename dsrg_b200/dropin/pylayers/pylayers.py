"""Drop-in Caffe Python layers for DSRG's pixel-labelling hot path, H100-backed.

Same class names, bottoms/tops, ``param_str`` keys, side effects and error behaviour as the
reference's pylayers/pylayers/pylayers.py, so ``python_param { module: 'pylayers' layer: ... }``
in train-s.prototxt:746-812 keeps working:

* ``CRFLayer``               (pylayers.py:54-92)   -> dsrg_crflayer_forward_host
* ``DSRGLayer``              (pylayers.py:277-344) -> dsrg_dsrg_forward_host
* ``BalancedSeedLossLayer``  (pylayers.py:120-152) -> dsrg_seedloss_{forward,backward}_host
* ``generate_seed_step``     (pylayers.py:237-275) -> dsrg_srg_batch_host (batch of one)
* ``SoftmaxLayer`` / ``ConstrainLossLayer`` (pylayers.py:23-51, :154-180), the producer and the
  other consumer of the hot path's blobs (SURVEY 8f rank 1) -> dsrg_softmax_* / dsrg_constrainloss_*,
  so that the module covers every Python layer train-s.prototxt names except the data layer.
* ``SeedLossLayer`` / ``ExpandLossLayer`` (pylayers.py:95-118, :183-233), SEC's seeding and expansion losses
  (the seed-loss blocks train-s.prototxt:821-910 keeps commented out, and SEC-style baselines)
  -> dsrg_seedloss_plain_* / dsrg_expandloss_*.
* ``AnnotationLayer`` / ``AnnotationLayerCOCO`` (pylayers.py:346-387, :389-512), the VOC and COCO training inputs
  -> dsrg_annotation_forward_* / dsrg_annotation_coco_forward_*.
* The package's ``layer`` submodule (pylayers/pylayers/layer.py) holds ``ImageSegDataLayer``, the stage-2 training
  input of train-f.prototxt -> dsrg_seg_data_forward_*; it reads its files through ``_read`` / ``_imread`` below.

The blobs Caffe hands to a Python layer are host numpy views, so the ``*_host`` entry points of
the C ABI are used: one H2D of the bottoms and one D2H of the tops per call, everything else --
including the image zoom / mean / round preprocessing -- on the GPU.  There is no multiprocessing.Pool (pylayers.py:292) and no CPU fallback.
"""
import ast
import re

import numpy as np
import yaml

import caffe  # the layers subclass caffe.Layer exactly like the reference (pylayers.py:1)

from dsrg_b200 import api as _api

min_prob = 0.0001  # pylayers.py:20

_ENGINES = {}


def _engine(n, c, h, w):
    """One engine per blob shape and device, created on first use and kept (layers are long-lived).  The device
    is the solver thread's current CUDA device -- the one ``caffe.set_device`` chose (training/tools/train.py:77-79)
    -- or DSRG_B200_DEVICE; every C entry point restores the thread's current device before it returns."""
    from dsrg_b200 import _lib
    key = (int(n), int(c), int(h), int(w), int(_lib.lib().dsrg_current_device()))
    if key not in _ENGINES:
        _ENGINES[key] = _api.Engine(key[0], key[2], key[3], key[1], device=key[4])
    return _ENGINES[key]


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


_PINNED_REGIONS = {}   # data pointer -> (nbytes, the array) of blob buffers page-locked with dsrg_host_register


def _pin(a):
    """Page-lock a blob's buffer once (Caffe keeps its blobs for the life of the net; in GPU mode their CPU side
    already is pinned memory): the host entry points then stream it at the PCIe rate instead of going through the
    driver's staged pageable copies.  DSRG_B200_PIN_BLOBS=0 turns it off; failures are ignored.
    The table holds a reference to every array it registered, so a registered buffer is never freed: memory that is
    freed while still registered and then handed to another array makes the driver refuse later copies from it
    (cudaErrorInvalidValue).  At most 16 arrays are held; the oldest is unregistered and released first."""
    import os
    if os.environ.get("DSRG_B200_PIN_BLOBS", "1") == "0" or not isinstance(a, np.ndarray) or a.nbytes < (1 << 20):
        return a
    from dsrg_b200 import _lib
    ptr = a.ctypes.data
    if _PINNED_REGIONS.get(ptr, (None,))[0] != a.nbytes:
        L = _lib.lib()
        if ptr in _PINNED_REGIONS:
            L.dsrg_host_unregister(ptr)
            del _PINNED_REGIONS[ptr]
        while len(_PINNED_REGIONS) >= 16:      # blobs come and go in tests; a net has a handful
            old = next(iter(_PINNED_REGIONS))
            L.dsrg_host_unregister(old)
            del _PINNED_REGIONS[old]
        if L.dsrg_host_register(ptr, a.nbytes) == 0:
            _PINNED_REGIONS[ptr] = (a.nbytes, a)
    return a


_IMAGE_BUFS = {}


def _fingerprint(a):
    """Cheap identity of a blob's current content: buffer address, shape and a strided sample of ~16 K values.
    Used to recognise that DSRGLayer is fed the very blobs CRFLayer has just refined (train-s.prototxt:758-786)."""
    flat = a.reshape(-1)
    step = max(1, flat.size // 16384)
    return (a.ctypes.data, a.shape, str(a.dtype), hash(flat[::step].tobytes()))


_LAST_CRF = {}   # what the engine's retained mean-field result was computed from


def _share_crf():
    import os
    return os.environ.get("DSRG_B200_SHARE_CRF", "1") != "0"


def _prepare_image(im, eng):
    """pylayers.py:70-75 / :315-319 (bilinear zoom to the map size, + mean pixel, np.round) and the
    ubyte cast of CRF.py:32, on the device: dsrg_prepare_image_host is byte-identical to the
    reference's scipy.ndimage.zoom(order=1) pipeline (tests/test_gpu_dropin.py)."""
    key = (id(eng), im.shape[0])
    if key not in _IMAGE_BUFS:   # pinned once per engine: the uint8 image comes back and goes in again with the pass
        _IMAGE_BUFS[key] = _api.pinned_empty((im.shape[0], eng.H, eng.W, 3), np.uint8)
    return eng.prepare_image_host(_f32(im), (104.0, 117.0, 123.0), out=_IMAGE_BUFS[key])


def _clamped_writeback(blob_data, probs):
    """The reference clamps the bottom blob in place (pylayers.py:67, :312); the host entry point applied the
    clamp to the array it was given -- which is the blob itself unless _f32 had to make a contiguous copy."""
    if probs is not blob_data and not np.shares_memory(probs, blob_data):
        blob_data[...] = probs


class SoftmaxLayer(caffe.Layer):
    """pylayers.py:23-51 -> dsrg_softmax_{forward,backward}_host."""

    def setup(self, bottom, top):
        if len(bottom) != 1:
            raise Exception("Need two inputs to compute distance.")

    def reshape(self, bottom, top):
        top[0].reshape(*bottom[0].data.shape)

    def forward(self, bottom, top):
        top[0].data[...] = _engine(*bottom[0].data.shape).softmax_forward_host(_f32(bottom[0].data))

    def backward(self, top, prop_down, bottom):
        bottom[0].diff[...] = _engine(*bottom[0].data.shape).softmax_backward_host(_f32(bottom[0].data),
                                                                                  _f32(top[0].diff))


class CRFLayer(caffe.Layer):
    """pylayers.py:54-92."""

    def setup(self, bottom, top):
        if len(bottom) != 2:
            raise Exception("The layer needs two inputs!")

    def reshape(self, bottom, top):
        top[0].reshape(*bottom[0].data.shape)

    def forward(self, bottom, top):
        n, c, h, w = bottom[0].data.shape
        probs = _f32(bottom[0].data)
        eng = _engine(n, c, h, w)
        im = _prepare_image(bottom[1].data[...], eng)
        log_out = np.empty((n, c, h, w), np.float32)
        self.result = np.empty((n, c, h, w), np.float32)
        eng.crflayer_forward_host(probs, im, _api.crf_params(12.0), log_out, self.result)  # scale_factor=12.0 (:82)
        _clamped_writeback(bottom[0].data, probs)
        top[0].data[...] = log_out
        # the engine keeps the raw marginals: a DSRGLayer fed the same two blobs need not repeat the CRF
        _LAST_CRF.clear()
        _LAST_CRF.update(engine=eng, n=n, scale=12.0, probs=_fingerprint(bottom[0].data),
                         image=_fingerprint(bottom[1].data))

    def backward(self, top, prop_down, bottom):
        grad = (1 - self.result) * top[0].diff[...]
        bottom[0].diff[...] = grad


class BalancedSeedLossLayer(caffe.Layer):
    """pylayers.py:120-152.  Default = the reference's semantics: the mean over THIS solver's batch (one Caffe
    solver per GPU, gradients averaged by the trainer).  ``param_str: "{'global_batch': True}"`` (or
    DSRG_B200_GLOBAL_LOSS=1) opts into the mean over the global batch of a torch.distributed job instead: the two
    local sums and the local image count are all-reduced once, in forward (dsrg_b200/shard.py); backward reuses
    the count and issues no collective."""

    def setup(self, bottom, top):
        if len(bottom) != 2:
            raise Exception("The layer needs two inputs!")
        import os
        params = yaml.safe_load(self.param_str) if getattr(self, "param_str", "") else None
        self._global = bool((params or {}).get("global_batch", os.environ.get("DSRG_B200_GLOBAL_LOSS", "0") == "1"))
        self._n_global = None

    def reshape(self, bottom, top):
        top[0].reshape(1)

    def forward(self, bottom, top):
        n, c, h, w = bottom[0].data.shape
        terms = _engine(n, c, h, w).seedloss_forward_host(_f32(bottom[0].data), _f32(bottom[1].data))
        n_global = n
        if self._global:
            terms, n_global = _allreduce_terms(terms, n)
        self._n_global = n_global
        top[0].data[...] = -(float(terms[0]) + float(terms[1])) / n_global

    def backward(self, top, prop_down, bottom):
        n, c, h, w = bottom[0].data.shape
        n_global = self._n_global if (self._global and self._n_global) else n
        # like the reference (pylayers.py:150-152) the incoming top diff is NOT applied
        bottom[0].diff[...] = _engine(n, c, h, w).seedloss_backward_host(_f32(bottom[0].data), _f32(bottom[1].data),
                                                                           n_global=n_global, top_diff=1.0)


class SeedLossLayer(caffe.Layer):
    """pylayers.py:95-118, SEC's seeding loss -> dsrg_seedloss_plain_{forward,backward}_host.  The mean over this
    solver's batch of sum(lab log p) / sum(lab); no floor on the count, so an image without seeds gives NaN like the
    reference."""

    def setup(self, bottom, top):
        if len(bottom) != 2:
            raise Exception("The layer needs two inputs!")

    def reshape(self, bottom, top):
        top[0].reshape(1)

    def forward(self, bottom, top):
        n = bottom[0].data.shape[0]
        terms = _engine(*bottom[0].data.shape).seedloss_plain_forward_host(_f32(bottom[0].data), _f32(bottom[1].data))
        top[0].data[...] = -float(terms[0]) / n

    def backward(self, top, prop_down, bottom):
        # like the reference (pylayers.py:116-118) the incoming top diff is NOT applied
        bottom[0].diff[...] = _engine(*bottom[0].data.shape).seedloss_plain_backward_host(_f32(bottom[0].data),
                                                                                          _f32(bottom[1].data))


class ExpandLossLayer(caffe.Layer):
    """pylayers.py:183-233, SEC's expansion loss (global weighted rank pooling, q_fg = 0.996, q_bg = 0.999)
    -> dsrg_expandloss_{forward,backward}_host.  Bottoms: probs (N, 21, 41, 41) and the labels blob (N, 1, 1, 21).
    The reference's graph reshapes to (-1, 20, 41*41) (:201, :208): any other shape fails inside Theano or mixes
    planes of different images, so it is refused here."""

    Q_FG, Q_BG = 0.996, 0.999   # pylayers.py:200, :207

    def setup(self, bottom, top):
        if len(bottom) != 2:
            raise Exception("The layer needs two inputs!")

    def reshape(self, bottom, top):
        top[0].reshape(1)

    @staticmethod
    def _check(bottom):
        shape = bottom[0].data.shape
        if len(shape) != 4 or shape[1] != 21 or shape[2] * shape[3] != 41 * 41:
            raise Exception("ExpandLossLayer needs probs of shape (N, 21, H, W) with H*W = 41*41 (pylayers.py:201), "
                            "got %s" % (shape,))
        if bottom[1].data.size != shape[0] * 21:
            raise Exception("ExpandLossLayer needs labels of shape (N, 1, 1, 21), got %s" % (bottom[1].data.shape,))
        return shape

    def forward(self, bottom, top):
        shape = self._check(bottom)
        terms = _engine(*shape).expandloss_forward_host(_f32(bottom[0].data), _f32(bottom[1].data),
                                                        self.Q_FG, self.Q_BG)
        top[0].data[...] = -(float(terms[0]) + float(terms[1]) + float(terms[2])) / shape[0]

    def backward(self, top, prop_down, bottom):
        shape = self._check(bottom)
        # like the reference (pylayers.py:231-233) the incoming top diff is NOT applied
        bottom[0].diff[...] = _engine(*shape).expandloss_backward_host(_f32(bottom[0].data), _f32(bottom[1].data),
                                                                       q_fg=self.Q_FG, q_bg=self.Q_BG)


def _allreduce_terms(terms, n_local):
    """One process per GPU: the balanced loss is a mean over the GLOBAL batch, so the two local sums
    are all-reduced (the path's only collective, dsrg_b200/shard.py).  Single process: identity."""
    from dsrg_b200 import shard
    return shard.allreduce_loss_terms(terms, n_local)


class ConstrainLossLayer(caffe.Layer):
    """pylayers.py:154-180 -> dsrg_constrainloss_{forward,backward}_host."""

    def setup(self, bottom, top):
        if len(bottom) != 2:
            raise Exception("The layer needs two inputs!")

    def reshape(self, bottom, top):
        top[0].reshape(1)

    def forward(self, bottom, top):
        top[0].data[...] = _engine(*bottom[0].data.shape).constrainloss_forward_host(_f32(bottom[0].data),
                                                                                    _f32(bottom[1].data))

    def backward(self, top, prop_down, bottom):
        gp, gl = _engine(*bottom[0].data.shape).constrainloss_backward_host(_f32(bottom[0].data), _f32(bottom[1].data))
        bottom[0].diff[...] = gp
        bottom[1].diff[...] = gl


def generate_seed_step(item):
    """pylayers.py:237-275 for ONE image: item = [labels (C,), seed_c (C,H,W), probs (C,H,W), th1, th2].
    Mutates and returns seed_c like the reference."""
    labels, seed_c, probs_refinement, th1, th2 = item
    c, h, w = seed_c.shape
    eng = _engine(1, c, h, w)
    # the reference compares float64 values; float32 inputs are compared exactly as given
    p32 = _f32(probs_refinement)[None]
    if not np.array_equal(p32[0].astype(np.float64), np.asarray(probs_refinement, np.float64)):
        raise ValueError("generate_seed_step: probs must be representable in float32 "
                         "(use DSRGLayer / dsrg_dsrg_forward for the fused float64 renormalisation)")
    out = eng.srg_host(_f32(labels)[None], p32, _f32(seed_c)[None], th1, th2)
    seed_c[...] = out[0]
    return seed_c


class DSRGLayer(caffe.Layer):
    """pylayers.py:277-344."""

    def setup(self, bottom, top):
        if len(bottom) != 4:
            raise Exception("The layer needs four inputs!")
        # parse the layer parameter string, which must be valid YAML (pylayers.py:284-291)
        layer_params = yaml.safe_load(self.param_str)
        self._th1 = layer_params['th1']
        self._th2 = layer_params['th2']
        if 'iters' not in layer_params:
            layer_params['iters'] = -1
        self._max_iters = layer_params['iters']
        self._iter_index = 0
        # extension (not in the reference, whose refinement() hard-codes 12.0, pylayers.py:335): the CRF scale
        self._scale_factor = float(layer_params.get('scale_factor', 12.0))

    def reshape(self, bottom, top):
        top[0].reshape(*bottom[1].data.shape)

    def forward(self, bottom, top):
        img_labels, probs, cues, im = bottom[0].data, bottom[1].data, bottom[2].data, bottom[3].data
        out = top[0].data
        direct = isinstance(out, np.ndarray) and out.dtype == np.float32 and out.flags["C_CONTIGUOUS"]
        seed_c = self.generate_seed(img_labels, probs, cues, im, seeds_out=_pin(out) if direct else None)
        self._iter_index = self._iter_index + 1
        if seed_c is not out:
            top[0].data[...] = seed_c

    def backward(self, top, prop_down, bottom):
        bottom[1].diff[...] = top[0].diff

    def generate_seed(self, labels, probs, cues, im, seeds_out=None):
        """refinement (pylayers.py:310-331) + SRG over the batch (:333-344), fused on the device."""
        num, channels, height, width = probs.shape
        eng = _engine(num, channels, height, width)
        scale = getattr(self, "_scale_factor", 12.0)
        if (_share_crf() and _LAST_CRF.get("engine") is eng and _LAST_CRF.get("n") == num and _LAST_CRF.get("scale") == scale
                and _LAST_CRF.get("probs") == _fingerprint(probs) and _LAST_CRF.get("image") == _fingerprint(im)):
            # same blobs as the CRFLayer that ran just before (already clamped in place by it): one refinement
            # serves both layers; any other CRF call on this engine invalidates the retained result (DSRG_E_STATE)
            try:
                return eng.srg_last_crf_host(_f32(labels).reshape(num, channels), _pin(_f32(cues)), self._th1, self._th2,
                                             seeds_out=seeds_out)
            except _api.DsrgError:
                pass
        _LAST_CRF.clear()
        p = _pin(_f32(probs))
        image = _prepare_image(_pin(_f32(im)), eng)
        seeds = eng.dsrg_forward_host(_f32(labels).reshape(num, channels), p, _pin(_f32(cues)), image,
                                      _api.crf_params(getattr(self, "_scale_factor", 12.0)), self._th1, self._th2,
                                      seeds_out=seeds_out)
        _clamped_writeback(probs, p)
        return seeds


class AnnotationLayer(caffe.Layer):
    """pylayers.py:346-387 -> dsrg_annotation_forward_host.  The pickle of localisation cues is read on
    the host like the reference does (cPickle -> pickle, latin1 for the Python-2 file); `np.random.choice`
    is drawn per image in the reference's order, so a seeded run mirrors the same images.
    ``param_str`` keys: `cues` (file name, default 'localization_cues.pickle'), `mirror`; additionally
    `root` (directory of the cue files; default: the reference's ../../training/localization_cues
    relative to this module, or $DSRG_CUES_DIR)."""

    def setup(self, bottom, top):
        import os
        import os.path as osp
        import pickle
        if len(bottom) != 2:
            raise Exception("The layer needs two inputs!")

        layer_params = yaml.safe_load(self.param_str)
        if 'cues' not in layer_params:
            layer_params['cues'] = 'localization_cues.pickle'
        self._cue_name = layer_params['cues']

        if 'mirror' not in layer_params:
            layer_params['mirror'] = False
        self.is_mirror = layer_params['mirror']

        this_dir = osp.dirname(__file__)
        root = layer_params.get('root') or os.environ.get('DSRG_CUES_DIR') or \
            osp.join(this_dir, '../../training', 'localization_cues')
        with open(osp.join(root, self._cue_name), 'rb') as f:
            self.data_file = pickle.load(f, encoding='latin1')

    def reshape(self, bottom, top):
        top[0].reshape(bottom[0].data.shape[0], 1, 1, 21)
        top[1].reshape(bottom[0].data.shape[0], 21, 41, 41)
        top[2].reshape(*bottom[1].data.shape)

    def forward(self, bottom, top):
        ids = np.asarray(bottom[0].data[...]).reshape(-1)
        tags, cues, flips = [], [], []
        for image_id in ids:
            tags.append(self.data_file['%i_labels' % image_id])
            cues.append(self.data_file['%i_cues' % image_id])
            if self.is_mirror:
                flips.append(int(np.random.choice(2) * 2 - 1 == -1))      # pylayers.py:385
        n = len(ids)
        eng = _engine(n, 21, 41, 41)
        labels, dense, images = eng.annotation_forward_host(tags, cues, flips if self.is_mirror else None,
                                                            _f32(bottom[1].data))
        top[0].data[...] = labels
        top[1].data[...] = dense
        top[2].data[...] = images

    def backward(self, top, propagate_down, bottom):
        pass


_IMREAD_GRAYSCALE, _IMREAD_COLOR = 0, 1   # cv2's values of the two flags


def _imread(path, flag):
    """cv2.imread(path, flag).  OpenCV is imported on first use, so that the module loads without it; tests and
    tools that feed decoded arrays replace this function."""
    import cv2
    return cv2.imread(path, flag)


def _read(path, flag):
    im = _imread(path, flag)
    if im is None:
        raise IOError("cannot read %r" % path)
    im = np.asarray(im)
    if im.dtype != np.uint8 or im.ndim != (3 if flag == _IMREAD_COLOR else 2) or (im.ndim == 3 and im.shape[2] != 3):
        raise ValueError("%r: expected %s uint8, got %s %s" % (
            path, "(H, W, 3)" if flag == _IMREAD_COLOR else "(H, W)", im.shape, im.dtype))
    return im


class AnnotationLayerCOCO(caffe.Layer):
    """pylayers.py:389-512 -> dsrg_annotation_coco_forward_host.  The files are decoded on the host (``_imread``)
    and the random numbers drawn there in the reference's order: ``numpy.random.shuffle`` of the list when an epoch
    is over, then per image ``np.random.choice`` when mirroring.  The zoom, the mean, the mirror, the cue planes and
    the tags of the whole batch are one device call.  ``param_str`` keys as in the reference: `source`, `root`,
    `batch_size`, `mean` (3 values) and `new_size` are required; `mirror` defaults to False, `ignore_label` to
    255."""

    K = 81

    def setup(self, bottom, top):
        layer_params = ast.literal_eval(self.param_str)
        self.source = layer_params['source']
        self.root_folder = layer_params['root']
        self.batch_size = layer_params['batch_size']
        self.is_mirror = layer_params.get('mirror', False)
        self.mean = layer_params['mean']
        self.new_h, self.new_w = layer_params['new_size']
        self.ignore_label = layer_params.get('ignore_label', 255)
        # image - self.mean subtracts per channel in float64 only when mean has three values; numpy would subtract
        # a scalar in float32
        if np.asarray(self.mean).shape != (3,):
            raise ValueError("mean must have 3 values, got %r" % (self.mean,))
        self._mean = np.asarray(self.mean, np.float64)
        with open(self.source) as f:
            self.indexlist = [line.strip().split() for line in f]
        self._cur = 0
        top[0].reshape(self.batch_size, 1, 1, self.K)
        top[1].reshape(self.batch_size, self.K, self.new_h // 8 + 1, self.new_w // 8 + 1)
        top[2].reshape(self.batch_size, 3, self.new_h, self.new_w)

    def reshape(self, bottom, top):
        pass

    def backward(self, top, propagate_down, bottom):
        pass

    def forward(self, bottom, top):
        B = self.batch_size
        h, w = self.new_h // 8 + 1, self.new_w // 8 + 1
        images, labels, flips = [], np.empty((B, h, w), np.uint8), []
        for itt in range(B):
            if self._cur == len(self.indexlist):                                      # pylayers.py:447-449
                self._cur = 0
                np.random.shuffle(self.indexlist)
            image_file_path, label_file_path = self.indexlist[self._cur]
            image = _read(self.root_folder + image_file_path, _IMREAD_COLOR)
            label = _read(self.root_folder + label_file_path, _IMREAD_GRAYSCALE)
            self._cur += 1
            if self.is_mirror:
                flips.append(int(np.random.choice(2) * 2 - 1 == -1))                 # pylayers.py:501
            images.append(image)
            labels[itt] = label   # broadcasts like top[1].data[itt, ...] = cues (:439); ValueError otherwise
        tops = [t.data for t in top[:3]]
        direct = all(isinstance(t, np.ndarray) and t.dtype == np.float32 and t.flags["C_CONTIGUOUS"] for t in tops)
        eng = _engine(B, self.K, h, w)
        try:
            got = eng.annotation_coco_forward_host(images, labels, (self.new_h, self.new_w), self._mean,
                                                   flips if self.is_mirror else None, self.ignore_label,
                                                   out=tops if direct else None)
        except _api.DsrgError as e:
            m = re.search(r"index -?\d+ is out of bounds for axis 0 with size \d+", str(e))
            if m:
                raise IndexError(m.group(0)) from None
            raise
        if not direct:
            for t, g in zip(top, got):
                t.data[...] = g
