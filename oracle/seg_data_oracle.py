"""TEST INFRASTRUCTURE ONLY -- numpy restatement of ImageSegDataLayer.forward (pylayers/pylayers/layer.py:51-61) and
of SimpleTransformer's three paths (:147-236), the stage-2 training input: mean and scale, bottom/right padding
(np.pad where the reference calls cv2.copyMakeBorder, so no cv2 is needed), the crop window, the CHW layout and the
mirror, with Python's ``random`` (shuffle, randint) and ``numpy.random`` (the mirror) drawn in the reference's order.
Only tests/ and tools/ may import it.

Parity status: pinned against the reference's own classes executed in place (oracle/ref_seg_layer.py ->
tests/golden/seg_data_ref.npz, compared bit for bit in tests/test_seg_data_cpu.py), and the padding against
cv2.copyMakeBorder itself.
"""
import random

import numpy as np

DEFAULTS = {"crop_size": (505, 505), "mean": [128, 128, 128], "scale": 1.0, "mirror": False, "phase": "Train",
            "ignore_label": 255}


def pad_byte(ignore_label):
    """saturate_cast<uchar>(ignore_label), the value cv2.copyMakeBorder writes into a uint8 label."""
    return int(np.clip(np.rint(ignore_label), 0, 255))


def pad_bottom_right(a, pad_h, pad_w, value):
    """cv2.copyMakeBorder(a, 0, pad_h, 0, pad_w, BORDER_CONSTANT, value) for a 2-D array or an (H, W, 3) one."""
    if pad_h <= 0 and pad_w <= 0:
        return a
    return np.pad(a, ((0, pad_h), (0, pad_w)) + ((0, 0),) * (a.ndim - 2), constant_values=value)


def centred(n, crop):
    """Offset of the centred window in an axis of n (>= crop) values: Python 2's `/` on ints."""
    return (n - crop) // 2


def crop_chw(image, h_off, w_off, crop_h, crop_w):
    """The window of the padded (H, W, 3) image, float32, CHW.  It comes back short where the window leaves it."""
    return np.asarray(image[h_off:h_off + crop_h, w_off:w_off + crop_w], np.float32).transpose(2, 0, 1)


def normalised(image, mean, scale=None, swap=False):
    """float32 image (channels reversed first when `swap`), minus the mean -- numpy computes it in float64 against a
    list or tuple of 3 and stores float32 -- then times scale in float32."""
    image = np.asarray(image, np.float32)
    if swap:
        image = image[:, :, [2, 1, 0]]
    image = (image - np.asarray(mean)).astype(np.float32)
    if scale is not None:
        image = image * np.float32(scale)
    return image


def transform(image, label, crop_size, mean, scale, h_off, w_off, flip, ignore_label=255):
    """preprocess(image, label) with the window (h_off, w_off) and the mirror (flip: 1 = reversed) given.
    Returns (image (3, crop_h, crop_w), label (crop_h, crop_w)) float32; the image is short where the window leaves
    the padded image."""
    crop_h, crop_w = crop_size
    pad_h, pad_w = max(crop_h - label.shape[0], 0), max(crop_w - label.shape[1], 0)
    image = pad_bottom_right(normalised(image, mean, scale), pad_h, pad_w, 0.0)
    label = pad_bottom_right(label, pad_h, pad_w, pad_byte(ignore_label))
    image = crop_chw(image, h_off, w_off, crop_h, crop_w)
    label = np.asarray(label[h_off:h_off + crop_h, w_off:w_off + crop_w], np.float32)
    if flip:
        image, label = image[:, :, ::-1], label[:, ::-1]
    return image, label


def draw(label_shape, crop_size, phase="Train", mirror=False):
    """(h_off, w_off, flip) of preprocess(image, label): random.randint twice in phase 'Train', centred otherwise,
    then np.random.choice(2) when mirroring (flip = 1 where it gives -1)."""
    crop_h, crop_w = crop_size
    rows, cols = max(label_shape[0], crop_h), max(label_shape[1], crop_w)
    if phase == "Train":
        h_off = random.randint(0, rows - crop_h)
        w_off = random.randint(0, cols - crop_w)
    else:
        h_off, w_off = centred(rows, crop_h), centred(cols, crop_w)
    flip = 0
    if mirror:
        flip = int(np.random.choice(2) * 2 - 1 == -1)
    return h_off, w_off, flip


def params_of(params):
    p = dict(DEFAULTS)
    p.update(params)
    return p


def preprocess(image, label, params):
    """SimpleTransformer.preprocess: with a label, the draws and transform(); without, a centred crop of the image
    padded from its own shape, no mirror."""
    p = params_of(params)
    crop_h, crop_w = p["crop_size"]
    if label is None:
        pad_h, pad_w = max(crop_h - image.shape[0], 0), max(crop_w - image.shape[1], 0)
        im = pad_bottom_right(normalised(image, p["mean"], p["scale"]), pad_h, pad_w, 0.0)
        return crop_chw(im, centred(im.shape[0], crop_h), centred(im.shape[1], crop_w), crop_h, crop_w)
    h_off, w_off, flip = draw(label.shape, (crop_h, crop_w), p["phase"], p["mirror"])
    return transform(image, label, (crop_h, crop_w), p["mean"], p["scale"], h_off, w_off, flip, p["ignore_label"])


def pre_test_image(image, params):
    """SimpleTransformer.pre_test_image: channels reversed before the mean, no scale, centred crop."""
    p = params_of(params)
    crop_h, crop_w = p["crop_size"]
    pad_h, pad_w = max(crop_h - image.shape[0], 0), max(crop_w - image.shape[1], 0)
    im = pad_bottom_right(normalised(image, p["mean"], swap=True), pad_h, pad_w, 0.0)
    return crop_chw(im, centred(im.shape[0], crop_h), centred(im.shape[1], crop_w), crop_h, crop_w)


def seg_data_forward(read, indexlist, cur, root, batch_size, params):
    """ImageSegDataLayer.forward on `read(path, flag)` (cv2.imread's place; flag 1 = colour, 0 = grey).  Shuffles
    `indexlist` in place with random.shuffle like the reference.  Returns (top0 (B, 3, crop_h, crop_w),
    top1 (B, 1, crop_h, crop_w) float32, the new _cur); a window that leaves the padded image raises numpy's
    ValueError at the store, as in the reference."""
    crop_h, crop_w = params_of(params)["crop_size"]
    top0 = np.zeros((batch_size, 3, crop_h, crop_w), np.float32)
    top1 = np.zeros((batch_size, 1, crop_h, crop_w), np.float32)
    for itt in range(batch_size):
        if cur == len(indexlist):
            cur = 0
            random.shuffle(indexlist)
        image_path, label_path = indexlist[cur]
        image, label = read(root + image_path, 1), read(root + label_path, 0)
        cur += 1
        im, lab = preprocess(image, label, params)
        top0[itt, ...] = im
        top1[itt, ...] = lab
    return top0, top1, cur
