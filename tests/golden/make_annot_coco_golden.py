"""tests/golden/make_annot_coco_golden.py -- regenerates tests/golden/annot_coco_ref.npz.

Runs only where the reference is mounted: the reference's own AnnotationLayerCOCO.forward (pylayers.py:432-512) is
executed in place (oracle/ref_coco_layer.py) on the seeded in-memory files below, one forward per case after
np.random.seed(seed).  Stored per case: the tag and cue tops in full (the cues as uint8 0/1),
the image top in full when it is small and as the SHA-256 digest of its float32 bytes otherwise, the layer's _cur
afterwards and the order the list was shuffled into.  The file pins oracle/annot_coco_oracle.annotation_coco_forward
(tests/test_annot_coco_cpu.py) and the device's dsrg_annotation_coco_forward_* through the drop-in layer
(tests/test_gpu_annot_coco.py).

usage: python tests/golden/make_annot_coco_golden.py
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "annot_coco_ref.npz")
FULL_MAX = 8192   # image tops of at most this many values are stored in full
DATA_ROOT = "/data/coco/"   # joined to the list's paths by string concatenation, like the reference

# (name, image sizes of the list's entries, label-map shape overrides {entry: (h, w)}, batch, new_size, mirror,
#  ignore_label, seed)
CASES = [
    ("wrap", [(20, 30), (1, 9), (13, 1)], {}, 4, (17, 23), True, 255, 1),        # epoch wrap + shuffle, H or W = 1
    ("ignore7", [(11, 14), (9, 9)], {}, 2, (16, 16), False, 7, 2),                # non-default ignore_label
    ("cval", [(40, 51)], {}, 1, (45, 45), False, 255, 3),                         # 51 -> 45: scipy's 0 column
    ("batch18", [(9, 12), (15, 7), (1, 1), (6, 20), (30, 3)], {2: (1, 2), 4: (2, 1)}, 18, (9, 11), True, 255, 4),
    ("voc", [(375, 500), (500, 375), (333, 500)], {}, 3, (321, 321), True, 255, 10),
    ("coco", [(480, 640), (640, 480), (427, 640), (612, 612)], {}, 4, (321, 321), True, 255, 20),
]
MEAN = (104.008, 116.669, 122.675)


def case_files(case):
    """(files {path: array}, indexlist, root) of a case: noise images (synth.make_image) and label maps with the
    background, two classes and, unless ignore_label is one of the classes, ignore pixels."""
    from dsrg_b200 import synth
    name, sizes, shapes, B, new_size, mirror, ignore, seed = case
    rng = np.random.RandomState(9000 + seed)
    h, w = new_size[0] // 8 + 1, new_size[1] // 8 + 1
    files, indexlist = {}, []
    for i, (H, W) in enumerate(sizes):
        im_path, lab_path = "JPEGImages/%s_%d.jpg" % (name, i), "Annotations/%s_%d.png" % (name, i)
        files[DATA_ROOT + im_path] = synth.make_image(np.random.RandomState(7000 + 10 * seed + i), H, W, "noise")
        values = np.array([0] + list(rng.choice(np.arange(1, 81), 2, replace=False)) + [ignore if ignore > 80 else 7])
        files[DATA_ROOT + lab_path] = values[rng.randint(0, len(values), shapes.get(i, (h, w)))].astype(np.uint8)
        indexlist.append([im_path, lab_path])
    return files, indexlist, DATA_ROOT


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()


def order_of(indexlist, original):
    return np.array([original.index(e) for e in indexlist], np.int64)


def main():
    from oracle import ref_coco_layer
    if not ref_coco_layer.available():
        sys.exit("the reference is not mounted")
    out = {}
    for case in CASES:
        name, sizes, shapes, B, new_size, mirror, ignore, seed = case
        files, indexlist, root = case_files(case)
        original = [list(e) for e in indexlist]
        np.random.seed(seed)
        t0, t1, t2, cur = ref_coco_layer.annotation_coco_layer_forward(files, indexlist, 0, root, B, MEAN, new_size,
                                                                       mirror, ignore)
        out["labels_" + name] = t0
        out["cues_" + name] = t1.astype(np.uint8)
        out["shape_" + name] = np.array(t2.shape, np.int64)
        if t2.size <= FULL_MAX:
            out["full_" + name] = t2
        else:
            out["sha_" + name] = np.array(digest(t2))
        out["cur_" + name] = np.array(cur, np.int64)
        out["order_" + name] = order_of(indexlist, original)
    np.savez_compressed(OUT, **out)
    print("wrote %s (%d arrays, %d bytes)" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
