"""Latency of the inference post-processing (SURVEY.md 8f rank 3): predict_mask() tails of
training/tools/test-ms.py on VOC-sized images, one image per call, sizes changing from call to call --
through postprocess.predict_mask_ms (host numpy in, host label map out).  Not the headline metric
(that is bench.py); prints one JSON line.

With --labels 81 it times the COCO tool's post-processing instead (training/tools/test-coco.py:108-133: one
481-pixel scale, 81 labels, the mean field on the label-chunked path) on COCO-sized images.

With --preprocess it also times the step before the network, preprocess(image, size) of every scale of an image
(postprocess.preprocess, one launch), next to the same statements with scipy on one core.

usage: python tools/bench_infer.py [--images 40] [--cpu 2] [--labels 21|81] [--preprocess [--cpu-preprocess 8]]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZES = [(375, 500), (500, 375), (333, 500), (500, 334), (366, 500), (281, 500), (500, 500), (375, 500)]
COCO_SIZES = [(480, 640), (640, 480), (427, 640), (640, 427), (480, 640), (612, 612), (426, 640), (480, 640)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=40)
    ap.add_argument("--cpu", type=int, default=None, help="images timed through the CPU oracle (0 = skip; "
                                                          "default 2 at 21 labels, 0 at 81)")
    ap.add_argument("--labels", type=int, default=21, choices=(21, 81))
    ap.add_argument("--preprocess", action="store_true", help="also time the network input of every scale "
                                                              "(postprocess.preprocess) and its scipy statements")
    ap.add_argument("--cpu-preprocess", type=int, default=8, help="images whose preprocess is timed with scipy")
    args = ap.parse_args()
    if args.cpu is None:
        args.cpu = 2 if args.labels == 21 else 0
    import torch
    from dsrg_b200 import pool, postprocess, synth
    coco = args.labels == 81
    sizes = COCO_SIZES if coco else SIZES
    scales = (61,) if coco else (31, 41, 51)        # fc8 of the 481 input (test-coco.py:116) / of 241, 321, 401
    cases = [synth.make_score_blobs(100 + i, H, W, scales, C=args.labels) for i, (H, W) in enumerate(sizes)]
    for c in cases:                                   # warm-up: engine growth, lazy allocations
        postprocess.predict_mask_ms(c["image"], c["blobs"])
    eng = list(pool._ENGINES.values())[0]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(args.images):
        c = cases[i % len(cases)]
        postprocess.predict_mask_ms(c["image"], c["blobs"])
    dt = time.perf_counter() - t0
    eng.take_launch_count()
    eng.profile(True)
    for c in cases:
        postprocess.predict_mask_ms(c["image"], c["blobs"])
    prof = eng.profile_read()
    eng.profile(False)
    launches = eng.take_launch_count()
    gpu_ms = sum(v[0] for v in prof.values()) / len(cases)
    what = ("81 labels, 1 score scale -> zoom -> softmax -> CRF 10 it -> argmax), one COCO-sized image per call"
            if coco else "3 score scales -> zoom/sum -> softmax -> CRF 10 it -> argmax), one VOC-sized image per call")
    out = {"metric": "images/s, predict_mask post-processing (" + what + ", host in / host out",
           "labels": args.labels, "gpu": torch.cuda.get_device_name(0),
           "value": args.images / dt, "ms_per_image": 1e3 * dt / args.images, "images": args.images,
           "sizes": sizes, "engine_capacity": list(eng.capacity), "engine_device_MB": eng.device_bytes / 1e6,
           "kernel_ms_per_image": gpu_ms, "launches_per_image": launches / len(cases),
           "kernel_classes_ms_per_image": {k: v[0] / len(cases) for k, v in sorted(prof.items())}}
    if args.cpu:
        from oracle import post_oracle
        t0 = time.perf_counter()
        for c in cases[:args.cpu]:
            post_oracle.predict_mask_ms(c["image"], c["blobs"])
        cdt = (time.perf_counter() - t0) / args.cpu
        out["cpu_oracle"] = {"ms_per_image": 1e3 * cdt, "images": args.cpu, "cores": 1,
                             "kind": "port (scipy zoom + numpy + oracle/crf_oracle.c)"}
    if args.preprocess:
        out["preprocess"] = time_preprocess(args, cases, eng, coco)
    print(json.dumps(out), flush=True)


def time_preprocess(args, cases, eng, coco):
    """preprocess(image, size) of every scale of an image (test-ms.py:68-81 at 241/321/401, test-coco.py:92-105 at
    481) through postprocess.preprocess: host uint8 image in, host float32 blobs out; the kernel time from the
    profile; and the same statements with scipy (oracle/prep_oracle.py) on one core of this host."""
    import torch
    from dsrg_b200 import postprocess
    from oracle import prep_oracle
    sizes = (481,) if coco else (241, 321, 401)
    for c in cases:                                   # warm-up: staging growth
        postprocess.preprocess(c["image"], sizes, M=args.labels)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(args.images):
        c = cases[i % len(cases)]
        postprocess.preprocess(c["image"], sizes, M=args.labels)
    dt = (time.perf_counter() - t0) / args.images
    eng.take_launch_count()
    eng.profile(True)
    for c in cases:
        postprocess.preprocess(c["image"], sizes, M=args.labels)
    prof = eng.profile_read()
    eng.profile(False)
    launches = eng.take_launch_count()
    kms = prof["prepare_image"][0] / len(cases)
    nbytes = 0
    for c in cases:
        H, W = c["image"].shape[:2]
        nbytes += 3 * H * W + sum(12 * h * w for h, w in (postprocess.net_input_size(H, W, s) for s in sizes))
    nbytes /= len(cases)
    res = {"sizes": list(sizes), "ms_per_image": 1e3 * dt, "images": args.images, "kernel_ms_per_image": kms,
           "launches_per_image": launches / len(cases), "algorithmic_MB_per_image": nbytes / 1e6,
           "kernel_GB_per_s": nbytes / (kms * 1e6)}
    n = max(1, args.cpu_preprocess)
    t0 = time.perf_counter()
    for i in range(n):
        c = cases[i % len(cases)]
        for s in sizes:
            prep_oracle.preprocess(c["image"], s)
    res["cpu_scipy"] = {"ms_per_image": 1e3 * (time.perf_counter() - t0) / n, "images": n, "cores": 1,
                        "kind": "the reference's statements (scipy.ndimage.zoom + numpy)"}
    return res


if __name__ == "__main__":
    main()
