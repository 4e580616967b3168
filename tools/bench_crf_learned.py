"""Time the learned CRF at inference against the Potts inference and the training forward, per call:

  potts     dsrg_crf_batch_dev: CRF()'s mean field (the inference every evaluation tool runs)
  matrix    dsrg_crf_batch_learned_dev with a compatibility matrix per kernel (random, not symmetric)
  features  dsrg_crf_batch_learned_dev on caller-given bilateral features (the image's own float32(x)/theta_alpha,
            ..., so the lattice is the image path's)
  train     dsrg_crf_forward_train_compat_dev (dsrg_crf_forward_train_wide_dev above 32 labels) with the same
            matrices, then the copy of Q_T out of the history: what nn.dense_crf(compat_bi=..., compat_sp=...)'s
            forward runs (it returns q_hist[T].clone()), as the inference legs copy Q_T into their output

on batch 64 at 321 x 321 with 21 labels on smooth and photo-like images, train-s's shape (batch 20 at 41 x 41, scale
factor 12) and COCO's 81 labels at batch 8 @ 321 x 321 on photo-like images; 10 mean-field iterations.  The matrix
inference skips the T stores of B·M·N floats the training forward makes, so it should be no slower than it.  Each line
also gives the engine's device bytes before and after the first matrix call.

--chain also times postprocess.predict_masks_dev on 32 images of mixed VOC sizes (one batched forward of 41 x 41
score maps, "ms"), with CRF()'s CRF and with the learned one (matrices -w I and the images' own features, so the two
compute the same function), and checks that their label maps agree.

The legs run on a side stream (the engine's CUDA graphs need one), are warmed up, and alternate in rounds within one
session; each window is timed with CUDA events.  One JSON line per workload with the median ms per call of each leg,
the spread, and the card's name, power limit and SM clocks read in the same run.

usage: python tools/bench_crf_learned.py [--steps 10] [--warmup 3] [--rounds 5] [--workloads ...] [--chain]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_crf_grad import _image_features  # noqa: E402
from bench_torch_step import card  # noqa: E402

WORKLOADS = {   # name -> (B, H, W, M, scale factor, image)
    "b64_smooth": (64, 321, 321, 21, 1.0, "smooth"),
    "b64_photo": (64, 321, 321, 21, 1.0, "photo"),
    "train_s": (20, 41, 41, 21, 12.0, "smooth"),
    "coco_b8_photo": (8, 321, 321, 81, 1.0, "photo"),
}
T = 10


def _timed(torch, s, legs, steps, warmup, rounds):
    times = {k: [] for k in legs}
    with torch.cuda.stream(s):
        for fn in legs.values():
            for _ in range(warmup):
                fn()
        torch.cuda.synchronize()
        for _ in range(rounds):
            for k, fn in legs.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(s)
                for _ in range(steps):
                    fn()
                b.record(s)
                b.synchronize()
                times[k].append(a.elapsed_time(b) / steps)
    return times


def run(name, steps, warmup, rounds):
    import torch
    from dsrg_b200 import api, synth
    B, H, W, M, sf, img = WORKLOADS[name]
    batch = synth.make_batch(B, H, W, C=M, image=img, start=3, unique=8)
    unary = torch.from_numpy(np.log(np.maximum(batch["probs"], 1e-5)).astype(np.float32)).cuda()
    image = torch.from_numpy(batch["image"]).cuda()
    p = api.crf_params(sf, 13, T)
    eng = api.Engine(B, H, W, M)
    s = torch.cuda.Stream()
    mu = (torch.randn((2, M, M), generator=torch.Generator().manual_seed(5)) - 2 * torch.eye(M)).cuda()
    feat = _image_features(torch, image, p)
    outs = {k: torch.empty_like(unary) for k in ("potts", "matrix", "features", "train")}
    q_hist = torch.empty((T + 1,) + tuple(unary.shape), device="cuda")
    nchw = dict(unary_layout=api.LAYOUT_NCHW, out_layout=api.LAYOUT_NCHW, stream=s.cuda_stream)
    legs = {
        "potts": lambda: eng.crf_dev(unary, image, p, outs["potts"], **nchw),
        "matrix": lambda: eng.crf_learned_dev(unary, image, p, outs["matrix"], compat=mu, **nchw),
        "features": lambda: eng.crf_learned_dev(unary, None, p, outs["features"], features=feat, **nchw),
    }
    if M > 32:
        fwd = lambda: eng.crf_forward_train_wide_dev(unary, image, p, q_hist, compat=mu, stream=s.cuda_stream)  # noqa: E731
    else:
        fwd = lambda: eng.crf_forward_train_compat_dev(unary, image, p, mu, q_hist, stream=s.cuda_stream)  # noqa: E731
    legs["train"] = lambda: (fwd(), outs["train"].copy_(q_hist[T]))   # the legs run on s (_timed)
    b0 = eng.device_bytes
    with torch.cuda.stream(s):
        legs["potts"]()
        legs["features"]()
        b1 = eng.device_bytes
        legs["matrix"]()
    torch.cuda.synchronize()
    b2 = eng.device_bytes
    times = _timed(torch, s, legs, steps, warmup, rounds)
    torch.cuda.synchronize()
    checks = dict(matrix_vs_train=float((outs["matrix"] - q_hist[T]).abs().max()),
                  features_vs_potts=float((outs["features"] - outs["potts"]).abs().max()))
    eng.close()
    med = {k: float(np.median(v)) for k, v in times.items()}
    return dict(workload=name, B=B, H=H, W=W, M=M, scale_factor=sf, image=img, n_iters=T,
                ms_per_call={k: round(v, 3) for k, v in med.items()},
                spread_ms={k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
                matrix_over_train=round(med["matrix"] / med["train"], 3),
                matrix_over_potts=round(med["matrix"] / med["potts"], 3),
                features_over_potts=round(med["features"] / med["potts"], 3),
                max_abs=checks, engine_bytes=int(b0), feature_scratch_bytes=int(b1 - b0),
                matrix_scratch_bytes=int(b2 - b1), q_hist_bytes=(T + 1) * B * M * H * W * 4)


def chain(steps, warmup, rounds, n=32, M=21):
    import torch
    from dsrg_b200 import api, postprocess, synth
    rng = np.random.RandomState(4)
    sizes = [(375, 500), (500, 375), (333, 500), (500, 333), (375, 500), (281, 500), (500, 500), (366, 500)]
    ims = []
    for i in range(n):
        h, w = sizes[i % len(sizes)]
        ims.append(torch.from_numpy(synth.make_image(rng, h, w, "photo")).cuda())
    scores = [torch.from_numpy(rng.randn(n, M, 41, 41).astype(np.float32) * 3).cuda()]
    p = api.crf_params(1.0)
    feats = [_image_features(torch, im[None], p)[0] for im in ims]
    eye = torch.eye(M, device="cuda")
    learned = dict(compat_bi=-p.w1 * eye, compat_sp=-p.w2 * eye, features_bi=feats)
    res = {}
    legs = {"crf": lambda: res.__setitem__("crf", postprocess.predict_masks_dev(ims, scores, mode="ms")),
            "learned": lambda: res.__setitem__("learned", postprocess.predict_masks_dev(ims, scores, mode="ms",
                                                                                        **learned))}
    s = torch.cuda.Stream()
    times = _timed(torch, s, legs, steps, warmup, rounds)
    torch.cuda.synchronize()
    differ = sum(int((a != b).sum()) for a, b in zip(res["crf"], res["learned"]))
    total = sum(int(a.numel()) for a in res["crf"])
    med = {k: float(np.median(v)) for k, v in times.items()}
    return dict(workload="predict_masks_dev_voc32", images=n, M=M, n_scales=1,
                ms_per_call={k: round(v, 3) for k, v in med.items()},
                spread_ms={k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
                learned_over_crf=round(med["learned"] / med["crf"], 3), label_pixels_differing=differ,
                label_pixels=total)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--chain", action="store_true", help="also time predict_masks_dev on 32 mixed VOC sizes")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_crf_learned.py needs a CUDA device")
    info = card()
    for name in [w for w in a.workloads.split(",") if w]:
        r = run(name, a.steps, a.warmup, a.rounds)
        r.update(info)
        print(json.dumps(r), flush=True)
    if a.chain:
        r = chain(max(1, a.steps // 5), 1, a.rounds)
        r.update(info)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
