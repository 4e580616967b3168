"""Throughput of segmentation scoring (csrc/eval.cu): the confusion matrix of a VOC-val-sized run -- 1449 label
maps at the VOC image sizes of tools/bench_infer.py, 21 classes -- as evaluate.py builds it
(training/tools/evaluate.py:133-153).  Prints one JSON line:

* kernel: the whole set device-resident, one dsrg_confusion_add_dev pass per repeat, CUDA events over many
  passes; pixels/s and bytes/s from the bytes the count has to read (1 B gt + 1 or 4 B pred per pixel), and that
  rate as a share of the H100 SXM data sheet's 3.35 TB/s;
* host: the same set from host numpy arrays through metrics.ConfusionMatrix.generateM_all (PCIe included);
* cpu_baseline: evaluate.py's generateM -- the reference's own code run in place when it is mounted, else the
  same per-pixel Python loop restated -- on a few images on one core;
* the card's name and power limit, read in the same run.

usage: python tools/bench_eval.py [--images 1449] [--repeats 20] [--cpu 2]
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
K = 21
PEAK_BPS = 3.35e12   # H100 SXM data sheet, HBM3


def make_set(n_images, seed=0):
    """Label maps like VOC's: background majority, a few object regions, 255 on object borders; predictions that
    agree on most pixels."""
    rng = np.random.RandomState(seed)
    gts, preds = [], []
    protos = []
    for i, (H, W) in enumerate(SIZES):
        gt = np.zeros((H, W), np.uint8)
        for _ in range(3):
            c = rng.randint(1, K)
            y, x = rng.randint(0, H // 2), rng.randint(0, W // 2)
            h, w = rng.randint(H // 8, H // 2), rng.randint(W // 8, W // 2)
            gt[y:y + h, x:x + w] = c
            gt[y:y + h, x:x + 3] = 255
        pred = gt.copy()
        pred[pred == 255] = 0
        flip = rng.rand(H, W) < 0.1
        pred[flip] = rng.randint(0, K, int(flip.sum()))
        protos.append((gt.ravel(), pred.ravel()))
    for i in range(n_images):
        gts.append(protos[i % len(protos)][0])
        preds.append(protos[i % len(protos)][1])
    return gts, preds


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as ex:   # noqa: BLE001
        return "unknown (%s)" % ex


def generateM_loop(gt, pred, nclass):
    """evaluate.py:61-68's per-pixel loop, restated (used only when the reference is not mounted)."""
    m = np.zeros((nclass, nclass))
    for i in range(len(gt)):
        if gt[i] < nclass:
            m[gt[i], pred[i]] += 1.0
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=1449)
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--cpu", type=int, default=2, help="images through the per-pixel Python loop (0 = skip)")
    args = ap.parse_args()
    import torch
    from dsrg_b200 import api, metrics
    gts, preds = make_set(args.images)
    gt_all, pred_all = np.concatenate(gts), np.concatenate(preds)
    n = gt_all.size
    want = np.bincount(gt_all[gt_all < K].astype(np.int64) * K + pred_all[gt_all < K], minlength=K * K).reshape(K, K)
    out = {"metric": "confusion matrix of a VOC-val-sized run (%d label maps, %d pixels, K = %d)" % (args.images, n, K),
           "gpu": card(), "pixels": int(n)}
    d_gt = torch.from_numpy(gt_all).cuda()
    conf = api.Confusion(K)
    stream = torch.cuda.current_stream()
    for name, pred in (("u8", torch.from_numpy(pred_all).cuda()),
                       ("i32", torch.from_numpy(pred_all.astype(np.int32)).cuda())):
        conf.reset()
        conf.add_dev(d_gt, pred)                 # warm-up, and the result check
        M, inv = conf.read()
        assert np.array_equal(M, want.astype(np.uint64)) and not inv.any(), "device matrix differs from bincount"
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        for _ in range(args.repeats):
            conf.add_dev(d_gt, pred)
        b.record(stream)
        b.synchronize()
        ms = a.elapsed_time(b) / args.repeats
        nbytes = n * (1 + pred.element_size())
        out["kernel_" + name] = {"ms_per_pass": ms, "pixels_per_s": n / ms * 1e3, "bytes_per_s": nbytes / ms * 1e3,
                                 "share_of_3.35TB/s": nbytes / ms * 1e3 / PEAK_BPS, "repeats": args.repeats}
        del pred
    cm = metrics.ConfusionMatrix(K)
    items = list(zip(gts, preds))
    cm.generateM_all(items)                      # warm-up: staging allocation
    t0 = time.perf_counter()
    m = cm.generateM_all(items)
    dt = time.perf_counter() - t0
    assert np.array_equal(m, want)
    out["host_generateM_all"] = {"ms": dt * 1e3, "pixels_per_s": n / dt, "ms_per_image": dt * 1e3 / args.images,
                                 "pred": "uint8 numpy"}
    if args.cpu:
        from oracle import eval_oracle
        live = eval_oracle.available()
        f = eval_oracle.evaluate_cm()(K).generateM if live else (lambda it: generateM_loop(it[0], it[1], K))
        t0 = time.perf_counter()
        for i in range(args.cpu):
            f([gts[i], preds[i]])
        cdt = (time.perf_counter() - t0) / args.cpu
        out["cpu_baseline"] = {"ms_per_image": cdt * 1e3, "images": args.cpu, "cores": 1,
                               "kind": "reference generateM in place" if live else "generateM loop restated"}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
