"""tests/golden/make_prep_golden.py -- regenerates tests/golden/prep_ref.npz.

Runs only where the reference is mounted: the reference's own preprocess() of the evaluation tools
(training/tools/test-ms.py, test-ms-f.py, test-coco.py, generate_train_gt.py) is executed in place
(oracle/prep_oracle.py) on the seeded images below.  Small outputs are frozen in full, the VOC- and COCO-sized ones
as SHA-256 digests of their float32 bytes.  The file pins oracle/prep_oracle.preprocess (tests/test_prep_cpu.py) and
the device's dsrg_prepare_net_input_* (tests/test_gpu_prep.py).

usage: python tests/golden/make_prep_golden.py
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "prep_ref.npz")
FULL_MAX = 8192   # outputs of at most this many values are stored in full

# (name, H, W, sizes or zoom factors, relative, the reference script whose preprocess runs, seed)
CASES = [
    ("tiny", 7, 9, (5, 13), False, "test-ms.py", 1),                     # down- and upsampling
    ("row", 1, 17, (5, 9), False, "test-ms.py", 2),                      # H = 1
    ("column", 23, 1, (4, 11), False, "generate_train_gt.py", 3),        # W = 1
    ("cval", 40, 51, (45,), False, "test-ms.py", 4),                     # 51 -> 45: scipy's 0 in the last column
    ("factors", 37, 53, (0.75, 1, 1.25), True, "test-ms-f.py", 5),       # odd sizes, zoom factors
    ("tie", 334, 47, (0.75, 1, 1.25), True, "test-ms-f.py", 6),          # 334 * 0.75 = 250.5 -> 250, * 1.25 -> 418
    ("up", 23, 31, (241,), False, "test-coco.py", 7),                    # strong upsampling
    ("voc_375x500", 375, 500, (241, 321, 401), False, "test-ms.py", 10),
    ("voc_500x375", 500, 375, (241, 321, 401), False, "test-ms.py", 11),
    ("voc_333x500", 333, 500, (241, 321, 401), False, "test-ms.py", 12),
    ("voc_500x334", 500, 334, (241, 321, 401), False, "test-ms.py", 13),
    ("voc_gt_375x500", 375, 500, (321,), False, "generate_train_gt.py", 14),
    ("coco_480x640", 480, 640, (481,), False, "test-coco.py", 20),
    ("coco_640x480", 640, 480, (481,), False, "test-coco.py", 21),
    ("coco_612x612", 612, 612, (481,), False, "test-coco.py", 22),
]


def case_image(H, W, seed):
    """uint8 (H, W, 3) noise image (synth.make_image): every value stays reproducible across numpy versions."""
    from dsrg_b200 import synth
    return synth.make_image(np.random.RandomState(7000 + seed), H, W, "noise")


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()


def main():
    from oracle import prep_oracle
    if not prep_oracle.available():
        sys.exit("the reference is not mounted")
    out = {}
    for name, H, W, sizes, relative, script, seed in CASES:
        im = case_image(H, W, seed)
        for k, size in enumerate(sizes):
            got = prep_oracle.reference(script, im, size)
            key = "%s_%d" % (name, k)
            out["shape_" + key] = np.array(got.shape, np.int64)
            if got.size <= FULL_MAX:
                out["full_" + key] = got
            else:
                out["sha_" + key] = np.array(digest(got))
    np.savez_compressed(OUT, **out)
    print("wrote %s (%d arrays, %d bytes)" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
