"""Drop-in for pylayers/pylayers/layer.py: ``ImageSegDataLayer``, the stage-2 training input that
training/experiment/seed_mc/train-f.prototxt names (``module: 'pylayers.layer'``), with ``BatchLoader``,
``SimpleTransformer`` and ``print_info`` under the reference's names, ``param_str`` keys, defaults and printed lines
-> dsrg_seg_data_forward_host.

Decoding (``_imread`` of ``.pylayers``, cv2 imported on first use) and the random draws stay on the host, in the
reference's order: Python's ``random.shuffle`` of the list when an epoch is over, then per image the two
``random.randint`` of the crop window (phase 'Train') and ``np.random.choice`` of the mirror.  The mean, the scale,
the padding, the crop, the mirror and the CHW layout of a whole batch are one device call, bit-exact with the
reference's numpy and cv2 statements.

Narrower than the reference:
* images are uint8 (H, W, 3) and labels uint8 (H, W), what cv2.imread returns;
* ``mean`` is 3 values (ValueError otherwise) and ``scale`` a Python number;
* a crop window that leaves the padded image raises ValueError, also in ``SimpleTransformer.preprocess``, where the
  reference returns the short slice its layer then fails to store (numpy would broadcast a slice of one row or one
  column; that is refused too);
* parity is with the reference run on Python 3: Python 2's ``random`` draws other crops from the same seed.
"""
import ast
import random

import numpy as np

import caffe  # the layer subclasses caffe.Layer exactly like the reference (layer.py:8)

from . import pylayers as _pl


def _engine(batch):
    """The call reads nothing of an engine's shape: the smallest one dsrg_engine_create accepts, not a CRF-sized one
    next to the training network."""
    return _pl._engine(batch, 1, 1, 1)


def _pad_byte(ignore_label):
    """saturate_cast<uchar>(ignore_label): what cv2.copyMakeBorder pads a uint8 label with (round half to even,
    then clamp to 0..255)."""
    return int(np.clip(np.rint(float(ignore_label)), 0, 255))


def _mean3(mean):
    # image -= mean subtracts per channel in float64 only when mean has three values
    m = np.asarray(mean, np.float64)
    if m.shape != (3,):
        raise ValueError("mean must have 3 values, got %r" % (mean,))
    return m


def _uint8(a, ndim):
    a = np.ascontiguousarray(a)
    if a.dtype != np.uint8 or a.ndim != ndim or (ndim == 3 and a.shape[2] != 3):
        raise ValueError("expected a %s uint8 array, got %s %s" % ("(H, W, 3)" if ndim == 3 else "(H, W)",
                                                                 a.shape, a.dtype))
    return a


def _slice_len(n, start, length):
    return len(range(n)[start:start + length])


class ImageSegDataLayer(caffe.Layer):
    """layer.py:17-74 -> dsrg_seg_data_forward_host, one call per batch.  ``param_str`` keys as in the reference
    (parsed with ``ast.literal_eval``): `batch_size`, `root_folder` and `source` are required; `crop_size`
    (505, 505), `mean` [128, 128, 128], `scale` 1.0, `mirror` False, `phase` 'Train' and `ignore_label` 255 are
    the defaults."""

    def setup(self, bottom, top):
        self.top_names = ['data', 'label']
        params = ast.literal_eval(self.param_str)
        SimpleTransformer.check_params(params)
        self.batch_size = params['batch_size']
        self.input_shape = params['crop_size']
        self.batch_loader = BatchLoader(params)
        top[0].reshape(self.batch_size, 3, self.input_shape[0], self.input_shape[1])
        top[1].reshape(self.batch_size, 1, self.input_shape[0], self.input_shape[1])
        print_info("ImageSegDataLayer", params)

    def forward(self, bottom, top):
        loader, t = self.batch_loader, self.batch_loader.transformer
        images, labels, h_off, w_off, flips = [], [], [], [], []
        for itt in range(self.batch_size):
            image, label = loader._next_pair()
            h, w, f = t._draw(image.shape, label.shape)   # numpy's ValueError here stops the batch at this image
            images.append(image)
            labels.append(label)
            h_off.append(h)
            w_off.append(w)
            flips.append(f)
        tops = [t_.data for t_ in top[:2]]
        shapes = [(self.batch_size, 3, t.crop_h, t.crop_w), (self.batch_size, 1, t.crop_h, t.crop_w)]
        direct = all(isinstance(a, np.ndarray) and a.dtype == np.float32 and a.flags["C_CONTIGUOUS"] and
                     a.shape == s for a, s in zip(tops, shapes))
        got = t._run(_engine(self.batch_size), images, labels, h_off, w_off, flips, out=tops if direct else None)
        if not direct:
            for t_, g in zip(top, got):
                t_.data[...] = g

    def reshape(self, bottom, top):
        pass

    def backward(self, top, propagate_down, bottom):
        pass


class BatchLoader(object):
    """layer.py:77-116: the list of (image, label) paths, the epoch wrap with Python's ``random.shuffle``, and the
    files read by plain string concatenation of `root_folder` and the path."""

    def __init__(self, params):
        self.batch_size = params['batch_size']
        self.root_folder = params['root_folder']
        self.source = params['source']
        with open(self.source) as f:
            self.indexlist = [line.strip().split() for line in f]
        self._cur = 0
        self.transformer = SimpleTransformer(params)
        print("BatchLoader initialized with {} images".format(len(self.indexlist)))

    def _next_pair(self):
        if self._cur == len(self.indexlist):                                          # layer.py:104-106
            self._cur = 0
            random.shuffle(self.indexlist)
        image_file_path, label_file_path = self.indexlist[self._cur]
        image = _pl._read(self.root_folder + image_file_path, _pl._IMREAD_COLOR)
        label = _pl._read(self.root_folder + label_file_path, _pl._IMREAD_GRAYSCALE)
        self._cur += 1
        return image, label

    def load_next_image(self):
        """The next (image (3, crop_h, crop_w), label (crop_h, crop_w)) float32 pair: a device call of one image."""
        image, label = self._next_pair()
        return self.transformer.preprocess(image, label)


class SimpleTransformer:
    """layer.py:119-251.  Every path is a device call; the arithmetic is the reference's: float32(double(v) - mean)
    times float32(scale), padding of 0.0 after both, the label padded with saturate_cast<uchar>(ignore_label)."""

    def __init__(self, params):
        SimpleTransformer.check_params(params)
        self.mean = params['mean']
        self.is_mirror = params['mirror']
        self.crop_h, self.crop_w = params['crop_size']
        self.scale = params['scale']
        self.phase = params['phase']
        self.ignore_label = params['ignore_label']
        _mean3(self.mean)

    def set_mean(self, mean):
        _mean3(mean)
        self.mean = mean

    def set_scale(self, scale):
        self.scale = scale

    def _center(self, shape):
        """Offsets of the centred window in an image padded to at least the crop (layer.py:152-163)."""
        rows, cols = max(shape[0], self.crop_h), max(shape[1], self.crop_w)
        return (rows - self.crop_h) // 2, (cols - self.crop_w) // 2

    def _draw(self, image_shape, label_shape):
        """The crop window and the mirror of preprocess(image, label), drawn in the reference's order
        (layer.py:202-234).  Raises numpy's ValueError, after the draws, when the window leaves the padded image."""
        pad_h, pad_w = max(self.crop_h - label_shape[0], 0), max(self.crop_w - label_shape[1], 0)
        rows, cols = label_shape[0] + pad_h, label_shape[1] + pad_w
        if self.phase == 'Train':
            h_off = random.randint(0, rows - self.crop_h)
            w_off = random.randint(0, cols - self.crop_w)
        else:
            h_off, w_off = (rows - self.crop_h) // 2, (cols - self.crop_w) // 2
        flip = 0
        if self.is_mirror:
            flip = int(np.random.choice(2) * 2 - 1 == -1)
        got = (3, _slice_len(image_shape[0] + pad_h, h_off, self.crop_h),
               _slice_len(image_shape[1] + pad_w, w_off, self.crop_w))
        if got[1:] != (self.crop_h, self.crop_w):
            # what top[0].data[itt, ...] = im raises (layer.py:60)
            np.empty((3, self.crop_h, self.crop_w), np.float32)[...] = np.empty(got, np.float32)
            raise ValueError("a crop window of %s in the padded image is not supported (the reference would repeat "
                             "its one row or column)" % (got,))
        return h_off, w_off, flip

    def _run(self, eng, images, labels, h_off, w_off, flips, swap_rb=False, scale=None, out=None):
        return eng.seg_data_forward_host(
            images, labels, h_off, w_off, (self.crop_h, self.crop_w), _mean3(self.mean),
            float(self.scale if scale is None else scale), flips, swap_rb, _pad_byte(self.ignore_label), out=out)

    def pre_test_image(self, image):
        """layer.py:147-167: channels swapped before the mean, no scale, padding from the image, centred crop ->
        (3, crop_h, crop_w) float32."""
        image = _uint8(image, 3)
        h, w = self._center(image.shape)
        return self._run(_engine(1), [image], None, [h], [w], None, swap_rb=True, scale=1.0)[0][0]

    def preprocess(self, image, label=None):
        """layer.py:169-236.  Without a label: padding from the image and a centred crop, no mirror ->
        (3, crop_h, crop_w) float32.  With one: the window and the mirror drawn as in the reference ->
        (image (3, crop_h, crop_w), label (crop_h, crop_w)) float32."""
        image = _uint8(image, 3)
        if label is None:
            h, w = self._center(image.shape)
            return self._run(_engine(1), [image], None, [h], [w], None)[0][0]
        label = _uint8(label, 2)
        h, w, f = self._draw(image.shape, label.shape)
        im, lab = self._run(_engine(1), [image], [label], [h], [w], [f])
        return im[0], lab[0, 0]

    @classmethod
    def check_params(cls, params):
        """Writes the defaults of the keys the caller left out into the caller's dict (layer.py:238-251)."""
        for key, value in _DEFAULTS:
            if key not in params:
                params[key] = list(value) if isinstance(value, list) else value


_DEFAULTS = (('crop_size', (505, 505)), ('mean', [128, 128, 128]), ('scale', 1.0), ('mirror', False),
             ('phase', 'Train'), ('ignore_label', 255))


def print_info(name, params):
    print("{} initialized for split: {}, with bs: {}, im_shape: {}.".format(
        name, params['source'], params['batch_size'], params['crop_size']))
