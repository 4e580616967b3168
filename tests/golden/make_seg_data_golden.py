"""tests/golden/make_seg_data_golden.py -- regenerates tests/golden/seg_data_ref.npz.

Runs only where the reference and cv2 are present: the reference's own ImageSegDataLayer.forward and
SimpleTransformer (pylayers/pylayers/layer.py) are executed in place (oracle/ref_seg_layer.py) on the seeded
in-memory files below, after random.seed(seed) and np.random.seed(seed).  Stored per case: both tops in full when
they are small and as the SHA-256 digest of their float32 bytes otherwise, and for the layer cases the layer's _cur
afterwards and the order the list was shuffled into.  The file pins oracle/seg_data_oracle (tests/test_seg_data_cpu.py)
and the device's dsrg_seg_data_forward_* through the drop-in layer (tests/test_gpu_seg_data.py).

usage: python tests/golden/make_seg_data_golden.py
"""
import hashlib
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "seg_data_ref.npz")
FULL_MAX = 8192   # tops of at most this many values are stored in full
DATA_ROOT = "/data/voc/"   # joined to the list's paths by string concatenation, like the reference
MEAN = (104.008, 116.669, 122.675)

# (name, kind, image sizes, label sizes (None: the image's), batch, params, seed).  kind: "layer" (one forward of
# ImageSegDataLayer over a list of those files), "preprocess" (SimpleTransformer.preprocess(image) without a label)
# or "pre_test" (pre_test_image).  params are the layer's param_str keys besides batch_size, root_folder and source.
CASES = [
    ("pad_h", "layer", [(20, 40), (18, 50)], None, 2, {"crop_size": (25, 31), "mean": MEAN, "mirror": True}, 1),
    ("pad_both", "layer", [(12, 15), (9, 30)], None, 2, {"crop_size": (17, 21), "mean": MEAN}, 2),
    ("img_larger", "layer", [(30, 40), (26, 33)], [(22, 35), (26, 30)], 2,
     {"crop_size": (24, 24), "mean": MEAN, "mirror": True}, 3),
    ("train_window", "layer", [(40, 52), (37, 60)], None, 2, {"crop_size": (17, 23), "mean": MEAN, "mirror": True}, 4),
    ("test_odd", "layer", [(40, 52), (41, 53)], None, 2,
     {"crop_size": (16, 21), "mean": MEAN, "mirror": True, "phase": "Test"}, 5),
    ("wrap", "layer", [(10, 12), (11, 9), (8, 14)], None, 8, {"crop_size": (9, 9), "mean": MEAN, "mirror": True}, 22),
    ("ignore300", "layer", [(7, 9), (12, 5)], None, 2, {"crop_size": (10, 12), "mean": MEAN, "ignore_label": 300}, 7),
    ("ignore_m5", "layer", [(7, 9)], None, 1, {"crop_size": (10, 12), "mean": MEAN, "ignore_label": -5}, 8),
    ("ignore_half", "layer", [(7, 9)], None, 1, {"crop_size": (10, 12), "mean": MEAN, "ignore_label": 254.5}, 9),
    ("scale017", "layer", [(15, 20), (20, 15)], None, 2, {"crop_size": (18, 18), "scale": 0.017, "mirror": True}, 10),
    ("thin", "layer", [(1, 9), (13, 1)], None, 2, {"crop_size": (3, 5), "mean": MEAN, "mirror": True}, 11),
    ("thin_crop", "layer", [(1, 9), (7, 1)], None, 2, {"crop_size": (1, 1), "mean": MEAN, "mirror": True}, 12),
    ("batch18", "layer", [(9, 12), (15, 7), (1, 1), (6, 20), (30, 3)], None, 18,
     {"crop_size": (11, 13), "mean": MEAN, "mirror": True}, 13),
    ("voc321", "layer", [(375, 500), (500, 375), (333, 500)], None, 3,
     {"crop_size": (321, 321), "mean": (104.0, 117.0, 123.0), "mirror": True}, 14),
    ("nolabel", "preprocess", [(10, 14), (21, 26), (1, 1)], None, 3, {"crop_size": (17, 17), "mean": MEAN,
                                                                      "scale": 0.5}, 15),
    ("pre_test", "pre_test", [(10, 14), (20, 25), (16, 1)], None, 3, {"crop_size": (16, 16), "mean": MEAN}, 16),
]


def case_files(case):
    """(files {path: array}, indexlist, root) of a case: noise images (synth.make_image) and label maps with the
    background, two classes and ignore pixels (255)."""
    from dsrg_b200 import synth
    name, kind, sizes, label_sizes, B, params, seed = case
    rng = np.random.RandomState(9000 + seed)
    files, indexlist = {}, []
    for i, (H, W) in enumerate(sizes):
        im_path, lab_path = "JPEGImages/%s_%d.jpg" % (name, i), "SegmentationClassAug/%s_%d.png" % (name, i)
        files[DATA_ROOT + im_path] = synth.make_image(np.random.RandomState(7000 + 10 * seed + i), H, W, "noise")
        values = np.array([0] + list(rng.choice(np.arange(1, 21), 2, replace=False)) + [255])
        shape = (H, W) if label_sizes is None else label_sizes[i]
        files[DATA_ROOT + lab_path] = values[rng.randint(0, len(values), shape)].astype(np.uint8)
        indexlist.append([im_path, lab_path])
    return files, indexlist, DATA_ROOT


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()


def order_of(indexlist, original):
    return np.array([original.index(e) for e in indexlist], np.int64)


def store(out, key, a):
    out["shape" + key] = np.array(a.shape, np.int64)
    if a.size <= FULL_MAX:
        out["full" + key] = np.asarray(a, np.float32)
    else:
        out["sha" + key] = np.array(digest(a))


def run_reference(case):
    """The reference's own outputs of a case: (top0, top1 (None for the image-only kinds), _cur, order)."""
    from oracle import ref_seg_layer
    name, kind, sizes, label_sizes, B, params, seed = case
    files, indexlist, root = case_files(case)
    original = [list(e) for e in indexlist]
    random.seed(seed)
    np.random.seed(seed)
    if kind == "layer":
        t0, t1, cur = ref_seg_layer.seg_layer_forward(files, indexlist, 0, root, B, params)
        return t0, t1, cur, order_of(indexlist, original)
    t = ref_seg_layer.transformer(dict(params))
    fn = t.preprocess if kind == "preprocess" else t.pre_test_image
    images = [files[root + im] for im, _ in indexlist]
    return np.stack([fn(np.array(im)) for im in images]), None, None, None


def main():
    from oracle import ref_seg_layer
    if not ref_seg_layer.available():
        sys.exit("the reference or cv2 is not available")
    out = {}
    for case in CASES:
        name = case[0]
        t0, t1, cur, order = run_reference(case)
        store(out, "0_" + name, t0)
        if t1 is not None:
            store(out, "1_" + name, t1)
            out["cur_" + name] = np.array(cur, np.int64)
            out["order_" + name] = order
    np.savez_compressed(OUT, **out)
    print("wrote %s (%d arrays, %d bytes)" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
