"""Milliseconds per image of the inference post-processing (predict_mask() of training/tools/test-ms.py) when many
images are processed per pass, on the mixed VOC sizes of tools/bench_infer.py (or, with --labels 81, the COCO tool's
81 labels on COCO sizes).  Compares, on the same images:
  per_image      postprocess.predict_mask_ms, one image per call (host numpy in, host label map out)
  host_batch_K   postprocess.predict_masks_ms(batch=K): images grouped by size, K per pass (host in / host out)
  device         postprocess.predict_mask_batch_dev on CUDA tensors already on the device, one pass per size group
                 of at most 16 images, label maps left on the device
Each row gives ms per image (host clock around work that ends in a device synchronise), kernel launches per image
(those inside replayed graphs counted) and, for the batched rows, the batch engine's device_bytes.  The card's name,
power limit and SM clock are read in the same run.  Not the headline metric (that is bench.py); prints one JSON line.

usage: python tools/bench_infer_batch.py [--images 64] [--labels 21|81] [--repeats 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZES = [(375, 500), (500, 375), (333, 500), (500, 334), (366, 500), (281, 500), (500, 500), (375, 500)]
COCO_SIZES = [(480, 640), (640, 480), (427, 640), (640, 427), (480, 640), (612, 612), (426, 640), (480, 640)]


def card():
    import torch
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock"], info["sm_clock_max"] = [v.strip() for v in q.split(",")]
    except Exception as exc:   # the query is informative only
        info["nvidia_smi"] = "unavailable: %s" % exc
    return info


def timed(fn, n_images, repeats):
    """Best of `repeats` windows of fn() (which ends in a device synchronise), in ms per image."""
    best = None
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return 1e3 * best / n_images


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--labels", type=int, default=21, choices=(21, 81))
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    from dsrg_b200 import pool, postprocess, synth
    coco = args.labels == 81
    sizes = COCO_SIZES if coco else SIZES
    scales = (61,) if coco else (31, 41, 51)
    uniq = [synth.make_score_blobs(100 + i, H, W, scales, C=args.labels) for i, (H, W) in enumerate(sizes)]
    cases = [uniq[i % len(uniq)] for i in range(args.images)]
    ims, blobs = [c["image"] for c in cases], [c["blobs"] for c in cases]
    n = len(cases)
    rows = {}

    def sync_after(f):
        def g():
            f()
            torch.cuda.synchronize()
        return g

    # one image per call
    def per_image():
        for im, b in zip(ims, blobs):
            postprocess.predict_mask_ms(im, b)
    per_image()
    per_image()
    eng1 = pool.engine_for(*sizes[0], args.labels)
    eng1.take_launch_count()
    ms = timed(sync_after(per_image), n, args.repeats)
    rows["per_image"] = {"ms_per_image": ms, "launches_per_image": eng1.take_launch_count() / (n * args.repeats)}
    want = [postprocess.predict_mask_ms(im, b, smooth=False) for im, b in zip(ims, blobs)]

    # grouped on the host, K images per pass
    for K in (1, 4, 16):
        def host_batch(K=K):
            return postprocess.predict_masks_ms(ims, blobs, batch=K)
        host_batch()
        host_batch()
        engb = pool.batch_engine_for(1, *sizes[0], args.labels)
        engb.take_launch_count()
        ms = timed(sync_after(host_batch), n, args.repeats)
        rows["host_batch_%d" % K] = {"ms_per_image": ms,
                                     "launches_per_image": engb.take_launch_count() / (n * args.repeats),
                                     "engine_max_batch": engb.max_batch, "device_bytes": engb.device_bytes}
    got = postprocess.predict_masks_ms(ims, blobs, smooth=False, batch=16)
    assert all(np.array_equal(a, b) for a, b in zip(got, want)), "batched result differs from the per-image one"

    # on the device: inputs already there, one pass per size group of at most 16, results stay there
    keys = [(im.shape[:2], tuple(b.shape for b in bl)) for im, bl in zip(ims, blobs)]
    groups = []
    for idx in postprocess._chunks(keys, 16):
        groups.append((torch.from_numpy(np.stack([ims[i] for i in idx])).cuda(),
                       [torch.from_numpy(np.stack([blobs[i][k] for i in idx])).cuda() for k in range(len(scales))],
                       torch.empty((len(idx),) + ims[idx[0]].shape[:2], dtype=torch.int32, device="cuda")))
    stream = torch.cuda.Stream()   # the engine replays its graphs on a non-default stream

    def device():
        with torch.cuda.stream(stream):
            for im, sc, out in groups:
                postprocess.predict_mask_batch_dev(im, sc, out=out)
    for _ in range(3):   # eager, captured, replayed
        sync_after(device)()
    engb = pool.batch_engine_for(1, *sizes[0], args.labels)
    engb.take_launch_count()
    ms = timed(sync_after(device), n, args.repeats)
    rows["device"] = {"ms_per_image": ms, "launches_per_image": engb.take_launch_count() / (n * args.repeats),
                      "passes_per_window": len(groups), "engine_max_batch": engb.max_batch,
                      "device_bytes": engb.device_bytes}
    base = rows["per_image"]["ms_per_image"]
    for r in rows.values():
        r["speedup_vs_per_image"] = base / r["ms_per_image"]
    what = ("81 labels, 1 score scale (test-coco.py), COCO sizes" if coco else
            "21 labels, 3 score scales (test-ms.py), mixed VOC sizes")
    out = {"metric": "ms per image, predict_mask post-processing (zoom/sum -> softmax -> CRF 10 it -> argmax), " + what,
           "labels": args.labels, "images": n, "sizes": sizes, "repeats": args.repeats, "rows": rows}
    out.update(card())
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
