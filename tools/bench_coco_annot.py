"""Time AnnotationLayerCOCO.forward, the COCO training input (pylayers.py:432-512), on the device and with scipy.

The drop-in layer runs through the caffe shim with pre-decoded arrays fed through ``_imread``, so decoding is
excluded from both legs: what is timed is the zoom, the mean, the mirror, the cue planes and the tags of one batch,
plus the layer's host work and the copies.  ``--cpu`` adds the same statements with scipy on one core
(oracle/annot_coco_oracle.py, the per-pixel cue loop included), the way the reference's layer runs them.  Prints one
JSON line with the card's name and power limit next to the numbers.

usage: python tools/bench_coco_annot.py [--batch 20] [--steps 20] [--warmup 3] [--cpu]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MEAN = (104.008, 116.669, 122.675)
SIZES = [(480, 640), (640, 480), (427, 640), (612, 612), (375, 500)]   # COCO-like decoded image sizes


def card():
    """Name and power limit of GPU 0 (a read-only nvidia-smi query; None where it is unavailable)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:
        return None, None


def dataset(n, h, w, seed=0):
    from dsrg_b200 import synth
    rng = np.random.RandomState(seed)
    files, lines = {}, []
    for i in range(n):
        H, W = SIZES[i % len(SIZES)]
        files["/d/im%d.jpg" % i] = synth.make_image(np.random.RandomState(seed + i), H, W, "noise")
        values = np.array([0, rng.randint(1, 81), rng.randint(1, 81), 255])
        files["/d/lab%d.png" % i] = values[rng.randint(0, 4, (h, w))].astype(np.uint8)
        lines.append("im%d.jpg lab%d.png\n" % (i, i))
    return files, lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=20)
    ap.add_argument("--new-size", type=int, default=321)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu", action="store_true", help="also time the scipy statements on one core")
    args = ap.parse_args()

    from dsrg_b200.dropin import caffe_shim
    caffe_shim.install()
    import pylayers
    from pylayers import pylayers as _pl

    B, S = args.batch, args.new_size
    h = w = S // 8 + 1
    files, lines = dataset(2 * B, h, w)
    _pl._imread = lambda path, flag: files[path]
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "list.txt")
        with open(src, "w") as f:
            f.writelines(lines)
        layer = pylayers.AnnotationLayerCOCO()
        layer.param_str = repr({"source": src, "root": "/d/", "batch_size": B, "mean": MEAN, "new_size": (S, S),
                                "mirror": True})
        top = [caffe_shim.Blob() for _ in range(3)]
        layer.setup([], top)
    np.random.seed(0)
    for _ in range(args.warmup):
        layer.forward([], top)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        layer.forward([], top)
    dt = (time.perf_counter() - t0) / args.steps
    eng = _pl._engine(B, 81, h, w)
    eng.profile(True)
    layer.forward([], top)
    prof = eng.profile_read()
    eng.profile(False)
    name, limit = card()
    res = {"metric": "annotation_coco_forward", "unit": "ms per batch", "batch": B, "new_size": S,
           "gpu": name, "power_limit": limit, "device_ms": 1e3 * dt,
           "kernel_ms": sum(v[0] for k, v in prof.items()), "launches": sum(v[1] for v in prof.values())}
    if args.cpu:
        from oracle import annot_coco_oracle
        if hasattr(os, "sched_setaffinity"):
            os.sched_setaffinity(0, {sorted(os.sched_getaffinity(0))[0]})
        paths = [ln.split() for ln in lines]
        t0 = time.perf_counter()
        for i in range(B):
            annot_coco_oracle.coco_preprocess(files["/d/" + paths[i][0]], files["/d/" + paths[i][1]], (S, S),
                                              MEAN, -1 if i % 2 else 1)
        res["scipy_one_core_ms"] = 1e3 * (time.perf_counter() - t0)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
