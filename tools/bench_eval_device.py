"""Images per second of an evaluation run (test-ms.py / test-coco.py: preprocess -> network -> predict_mask ->
confusion matrix) with a stand-in network, two ways on the same seeded images:
  host     the tools' per-image loop: postprocess.preprocess -> net on a (1, 3, h, w) batch -> fc8 to the host ->
           postprocess.predict_mask_ms -> Confusion.add_host
  device   per chunk of --batch images: postprocess.preprocess_batch_dev (one launch for every scale) -> one network
           batch per scale -> postprocess.predict_masks_dev (grouped by size) -> Confusion.add_dev; images and ground
           truth already on the device, as a loader's .cuda() leaves them
The stand-in network is avg_pool2d(8, ceil_mode=True) and a fixed 1x1 convolution (41 x 41 scores at 321), so the
figure is the library's share of an evaluation run, not a real network's.  Both legs are warmed up on every shape
they time, then alternated --repeats times; each row reports the best window (host clock around work that ends in a
device synchronise) and the library's kernel launches per image (torch's own launches not counted).  The card's
name, power limit and SM clock are read in the same run.  Prints one JSON line per workload:
  voc: --images mixed VOC sizes, 21 labels, scales 241 / 321 / 401 (test-ms.py)
  coco: --images // 2 COCO sizes, 81 labels, scale 481 (test-coco.py)

usage: python tools/bench_eval_device.py [--images 32] [--batch 16] [--coco-batch 4] [--repeats 3]
                                      [--only voc|coco]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_infer_batch import COCO_SIZES, SIZES, card   # noqa: E402


def stand_in_net(torch, M, seed=0):
    g = torch.Generator().manual_seed(seed)
    conv = torch.nn.Conv2d(3, M, 1).cuda()
    with torch.no_grad():
        conv.weight.copy_(torch.randn(M, 3, 1, 1, generator=g) * 0.05)
        conv.bias.copy_(torch.randn(M, generator=g) * 0.5)

    def net(x):
        with torch.no_grad():
            return conv(torch.nn.functional.avg_pool2d(x, 8, 8, ceil_mode=True)).contiguous()
    return net


def workload(name, M, shapes, scales, batch, repeats):
    import torch
    from dsrg_b200 import api, pool, postprocess, synth
    rng = np.random.RandomState(7)
    ims = [synth.make_image(rng, H, W, "photo") for H, W in shapes]
    gts = [rng.randint(0, M, (H, W)).astype(np.uint8) for H, W in shapes]
    d_ims = [torch.from_numpy(im).cuda() for im in ims]
    d_gts = [torch.from_numpy(gt).cuda() for gt in gts]
    net = stand_in_net(torch, M)
    n = len(ims)
    cms = {"host": api.Confusion(M), "device": api.Confusion(M)}

    def host():
        cm = cms["host"]
        for im, gt in zip(ims, gts):
            blobs = postprocess.preprocess(im, scales, M=M)
            fc8 = [net(torch.from_numpy(b).cuda())[0].cpu().numpy() for b in blobs]
            cm.add_host(gt, postprocess.predict_mask_ms(im, fc8))
        torch.cuda.synchronize()

    def device():
        cm = cms["device"]
        for a in range(0, n, batch):
            x = postprocess.preprocess_batch_dev(d_ims[a:a + batch], scales, M=M)
            preds = postprocess.predict_masks_dev(d_ims[a:a + batch], [net(t) for t in x])
            for gt, p in zip(d_gts[a:a + batch], preds):
                cm.add_dev(gt, p)
        torch.cuda.synchronize()

    dev = torch.cuda.current_device()
    # the pooled engines the legs ran on, looked up without re-shaping them
    engines = {"host": lambda: [pool._ENGINES[(M, dev)]],
               "device": lambda: [pool._PREP_ENGINES[dev], pool._BATCH_ENGINES[(M, dev)]]}
    legs = {"host": host, "device": device}
    for _ in range(2):   # warm-up: every engine, image size, graph and torch kernel the windows use
        for f in legs.values():
            f()
    best = {k: None for k in legs}
    launches = {k: 0 for k in legs}
    for _ in range(repeats):
        for k, f in legs.items():
            for e in engines[k]():
                e.take_launch_count()
            t0 = time.perf_counter()
            f()
            dt = time.perf_counter() - t0
            launches[k] += sum(e.take_launch_count() for e in engines[k]())
            best[k] = dt if best[k] is None else min(best[k], dt)
    rows = {k: {"images_per_s": round(n / best[k], 1), "ms_per_image": round(1e3 * best[k] / n, 3),
                "library_launches_per_image": round(launches[k] / (n * repeats), 2)} for k in legs}
    m = {k: cm.read()[0] for k, cm in cms.items()}
    out = {"bench": "eval_device", "workload": name, "labels": M, "images": n, "scales": list(scales),
           "batch": batch, "repeats": repeats, "rows": rows,
           "device_vs_host": round(best["host"] / best["device"], 3),
           # both legs counted the same images (2 + repeats) times; the CRF's float atomics may flip near-ties
           "confusion_mismatch_share": float(np.abs(m["host"].astype(np.int64) - m["device"].astype(np.int64)).sum()
                                             / max(1, int(m["host"].sum())))}
    out.update(card())
    for cm in cms.values():
        cm.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--coco-batch", type=int, default=4,
                    help="81 labels: the batch engine holds about 4.7 GB per 640x640 image")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--only", choices=("voc", "coco"))
    args = ap.parse_args()
    rng = np.random.RandomState(3)
    voc = [SIZES[i] for i in rng.randint(0, len(SIZES), args.images)]
    coco = [COCO_SIZES[i] for i in rng.randint(0, len(COCO_SIZES), max(1, args.images // 2))]
    for name, M, shapes, scales, batch in (("voc", 21, voc, (241, 321, 401), args.batch),
                                           ("coco", 81, coco, (481,), args.coco_batch)):
        if args.only in (None, name):
            print(json.dumps(workload(name, M, shapes, scales, batch, args.repeats)), flush=True)


if __name__ == "__main__":
    main()
