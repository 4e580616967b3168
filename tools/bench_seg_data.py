"""Time ImageSegDataLayer.forward, the stage-2 training input (pylayers/pylayers/layer.py:51-61), on the device and
with numpy.

The drop-in layer runs through the caffe shim at train-f.prototxt's settings (batch 10, crop 321, mirror, the VOC
mean) on pre-decoded VOC-sized arrays (500x375 and 375x500) fed through ``_imread``, so decoding is excluded from
both legs: what is timed is the mean, the padding, the crop, the mirror and the layout of one batch, plus the
layer's host work and the copies.  ``--cpu`` adds the same statements in numpy on one core
(oracle/seg_data_oracle.py, np.pad in cv2.copyMakeBorder's place).  Prints one JSON line with the card's name and
power limit next to the numbers.

usage: python tools/bench_seg_data.py [--batch 10] [--crop 321] [--steps 50] [--warmup 5] [--cpu]
"""
import argparse
import contextlib
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MEAN = (104.0, 117.0, 123.0)   # train-f.prototxt's param_str
SIZES = [(500, 375), (375, 500)]   # VOC-sized decoded images


def card():
    """Name and power limit of GPU 0 (a read-only nvidia-smi query; None where it is unavailable)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:
        return None, None


def dataset(n, seed=0):
    from dsrg_b200 import synth
    rng = np.random.RandomState(seed)
    files, lines = {}, []
    for i in range(n):
        H, W = SIZES[i % len(SIZES)]
        files["/d/im%d.jpg" % i] = synth.make_image(np.random.RandomState(seed + i), H, W, "noise")
        files["/d/lab%d.png" % i] = np.array([0, 3, 15, 255], np.uint8)[rng.randint(0, 4, (H, W))]
        lines.append("im%d.jpg lab%d.png\n" % (i, i))
    return files, lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=10)
    ap.add_argument("--crop", type=int, default=321)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cpu", action="store_true", help="also time the numpy statements on one core")
    args = ap.parse_args()

    from dsrg_b200.dropin import caffe_shim
    caffe_shim.install()
    from pylayers import layer as seg_layer
    from pylayers import pylayers as _pl

    B, S = args.batch, args.crop
    files, lines = dataset(2 * B)
    _pl._imread = lambda path, flag: files[path]
    params = {"root_folder": "/d/", "batch_size": B, "mean": MEAN, "mirror": True, "crop_size": (S, S)}
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "train.txt")
        with open(src, "w") as f:
            f.writelines(lines)
        layer = seg_layer.ImageSegDataLayer()
        layer.param_str = repr(dict(params, source=src))
        top = [caffe_shim.Blob() for _ in range(2)]
        with contextlib.redirect_stdout(sys.stderr):   # the layer's two lines; stdout carries the JSON line only
            layer.setup([], top)
    random.seed(0)
    np.random.seed(0)
    for _ in range(args.warmup):
        layer.forward([], top)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        layer.forward([], top)   # returns once the tops have landed in host memory
    dt = (time.perf_counter() - t0) / args.steps
    eng = _pl._engine(B, 1, 1, 1)
    eng.profile(True)
    layer.forward([], top)
    prof = eng.profile_read()
    eng.profile(False)
    name, limit = card()
    out_bytes = 4 * B * 4 * S * S
    res = {"metric": "image_seg_data_forward", "unit": "ms per batch", "batch": B, "crop": S,
           "gpu": name, "power_limit": limit, "device_ms": 1e3 * dt,
           "kernel_ms": sum(v[0] for v in prof.values()), "launches": sum(v[1] for v in prof.values()),
           "kernel_out_MB": out_bytes / 1e6, "engine_MB": eng.device_bytes / 1e6}
    if args.cpu:
        from oracle import seg_data_oracle
        if hasattr(os, "sched_setaffinity"):
            os.sched_setaffinity(0, {sorted(os.sched_getaffinity(0))[0]})
        indexlist = [ln.split() for ln in lines]
        reps = max(1, args.steps // 10)
        t0 = time.perf_counter()
        for _ in range(reps):
            seg_data_oracle.seg_data_forward(lambda p, f: files[p], indexlist, 0, "/d/", B, params)
        res["numpy_one_core_ms"] = 1e3 * (time.perf_counter() - t0) / reps
    print(json.dumps(res))


if __name__ == "__main__":
    main()
