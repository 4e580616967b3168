"""Time the differentiable CRF against the plain forward, per step:

  forward   dsrg_crf_batch_dev: the mean field alone (inference)
  train     dsrg_crf_forward_train_dev + dsrg_crf_backward_dev: the forward that keeps Q_0..Q_T, then the exact
            backward to the unaries and the Potts weights (what nn.dense_crf runs per training step)
  compat    (--compat) dsrg_crf_forward_train_compat_dev + dsrg_crf_backward_compat_dev: the same step with a
            compatibility matrix per kernel (random, not symmetric) and its gradient
  train_theta, compat_theta
            (--kernel) the train (and with --compat the compat) step with the backward that also gives the gradient
            to the seven kernel bandwidths (dsrg_crf_backward_theta_dev, dsrg_crf_backward_compat_theta_dev); the
            line also reports the device memory the first such backward allocates (kgrad_bytes)
  train_feat
            (--features) the Potts step on caller-given bilateral features (dsrg_crf_forward_train_feat_dev +
            dsrg_crf_backward_feat_dev with grad_theta_sp): the image's own float32(x)/theta_alpha, ..., so the
            lattice is the image path's; timed beside train_theta (implied) and train

  wide_potts, wide_compat
            (--wide, on its own workloads at COCO's 81 labels) dsrg_crf_forward_train_wide_dev +
            dsrg_crf_backward_wide_dev, the label-chunked step with device Potts weights and with a matrix per kernel,
            timed beside the label-chunked inference forward; the line also reports the device memory the first
            backwards allocate (wide_bytes) and the FLOPs of the matrices' outer products (outer_flops)
  wide_theta, wide_feat
            (--wide --kernel, --wide --features) the label-chunked Potts step whose backward also gives the seven
            kernel bandwidths' gradient (dsrg_crf_backward_wide_theta_dev), and the one on the image's own features
            (dsrg_crf_forward_train_wide_feat_dev + dsrg_crf_backward_wide_feat_dev with grad_theta_sp), timed beside
            wide_potts; the line also reports what the first of them allocates (wide_kgrad_bytes)

on three workloads: train-s's shape (batch 20, 41 x 41 maps, 21 labels, scale_factor 12, smooth images) and batch 64
at 321 x 321 with scale_factor 1 on smooth and on photo-like images; 10 mean-field iterations.  The legs run on a side
stream (the engine's CUDA graphs need one), are warmed up, and are alternated in rounds within one session; each
window is timed with CUDA events.  Prints one JSON line per workload with the median ms per step of each leg, and the
card's name, power limit and SM clocks read in the same run.

usage: python tools/bench_crf_grad.py [--steps 20] [--warmup 3] [--rounds 5] [--workloads train_s,b64_smooth,b64_photo]
                                     [--compat] [--kernel] [--features] [--wide]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_torch_step import card  # noqa: E402

WORKLOADS = {   # name -> (B, H, W, M, scale factor, image)
    "train_s": (20, 41, 41, 21, 12.0, "smooth"),
    "b64_smooth": (64, 321, 321, 21, 1.0, "smooth"),
    "b64_photo": (64, 321, 321, 21, 1.0, "photo"),
}
WIDE_WORKLOADS = {   # --wide: COCO's training shape, and large photo-like images
    "coco_train": (20, 41, 41, 81, 12.0, "photo"),
    "b8_photo": (8, 321, 321, 81, 1.0, "photo"),
}
T = 10


def _image_features(torch, image, p):
    """The image's own bilateral features float32(x)/theta_alpha, ... (B, 5, H, W): the lattice is the image path's."""
    B, H, W = image.shape[:3]
    sig = torch.tensor([p.theta_alpha_x, p.theta_alpha_y, p.theta_beta_r, p.theta_beta_g, p.theta_beta_b],
                       device="cuda").view(1, 5, 1, 1)
    yy, xx = torch.meshgrid(torch.arange(H, device="cuda"), torch.arange(W, device="cuda"), indexing="ij")
    raw = torch.cat([xx.expand(B, 1, H, W).float(), yy.expand(B, 1, H, W).float(),
                     image.permute(0, 3, 1, 2).float()], 1)
    return (raw / sig).contiguous()


def run(name, steps, warmup, rounds, compat=False, kernel=False, features=False, wide=False):
    import torch
    from dsrg_b200 import api, synth
    B, H, W, M, sf, img = (WIDE_WORKLOADS if wide else WORKLOADS)[name]
    batch = synth.make_batch(B, H, W, C=M, image=img, start=3, unique=8)
    unary = torch.from_numpy(np.log(np.maximum(batch["probs"], 1e-5)).astype(np.float32)).cuda()
    image = torch.from_numpy(batch["image"]).cuda()
    G = torch.randn_like(unary)
    p = api.crf_params(sf, 13, T)
    eng = api.Engine(B, H, W, M)
    out = torch.empty_like(unary)
    q_hist = torch.empty((T + 1,) + tuple(unary.shape), device="cuda")
    gu, gw = torch.empty_like(unary), torch.empty((B, 2), device="cuda")
    s = torch.cuda.Stream()
    if compat:
        mu = (torch.randn((2, M, M), generator=torch.Generator().manual_seed(5)) - 2 * torch.eye(M)).cuda()
        gmu = torch.empty((B, 2, M, M), device="cuda")
    legs = {
        "forward": lambda: eng.crf_dev(unary, image, p, out, unary_layout=api.LAYOUT_NCHW,
                                       out_layout=api.LAYOUT_NCHW, stream=s.cuda_stream),
        "train": lambda: (eng.crf_forward_train_dev(unary, image, p, q_hist, stream=s.cuda_stream),
                          eng.crf_backward_dev(q_hist, image, p, G, gu, grad_potts=gw, stream=s.cuda_stream)),
    }
    extra = {}
    if wide:
        from dsrg_b200 import _lib
        del legs["train"]
        potts = torch.tensor([10.0, 3.0], device="cuda")
        mu = (torch.randn((2, M, M), generator=torch.Generator().manual_seed(5)) - 2 * torch.eye(M)).cuda()
        gmu = torch.empty((B, 2, M, M), device="cuda")
        legs["wide_potts"] = lambda: (
            eng.crf_forward_train_wide_dev(unary, image, p, q_hist, potts=potts, stream=s.cuda_stream),
            eng.crf_backward_wide_dev(q_hist, image, p, G, gu, potts=potts, grad_potts=gw, stream=s.cuda_stream))
        legs["wide_compat"] = lambda: (
            eng.crf_forward_train_wide_dev(unary, image, p, q_hist, compat=mu, stream=s.cuda_stream),
            eng.crf_backward_wide_dev(q_hist, image, p, G, gu, compat=mu, grad_compat=gmu, stream=s.cuda_stream))
        before = _lib.lib().dsrg_engine_device_bytes(eng.h)
        with torch.cuda.stream(s):
            legs["wide_potts"]()
            extra["wide_bytes_potts"] = int(_lib.lib().dsrg_engine_device_bytes(eng.h) - before)
            legs["wide_compat"]()
        torch.cuda.synchronize()
        extra["wide_bytes"] = int(_lib.lib().dsrg_engine_device_bytes(eng.h) - before)
        extra["outer_flops"] = 2 * 2 * M * M * H * W * B * T   # two lattices, a multiply-add per (l, l', pixel, t)
        if kernel or features:
            gt = torch.empty((B, 7), device="cuda")
            before = _lib.lib().dsrg_engine_device_bytes(eng.h)
            legs["wide_theta"] = lambda: (
                eng.crf_forward_train_wide_dev(unary, image, p, q_hist, potts=potts, stream=s.cuda_stream),
                eng.crf_backward_wide_theta_dev(q_hist, image, p, G, gu, gt, potts=potts, grad_potts=gw,
                                                stream=s.cuda_stream))
            with torch.cuda.stream(s):
                legs["wide_theta"]()
            torch.cuda.synchronize()
            extra["wide_kgrad_bytes"] = int(_lib.lib().dsrg_engine_device_bytes(eng.h) - before)
            if not kernel:
                del legs["wide_theta"]
        if features:
            feat = _image_features(torch, image, p)
            gf, gsp = torch.empty_like(feat), torch.empty((B, 2), device="cuda")
            legs["wide_feat"] = lambda: (
                eng.crf_forward_train_wide_feat_dev(unary, feat, p, q_hist, potts=potts, stream=s.cuda_stream),
                eng.crf_backward_wide_feat_dev(q_hist, feat, p, G, gu, gf, potts=potts, grad_potts=gw,
                                               grad_theta_sp=gsp, stream=s.cuda_stream))
    if compat and not wide:
        legs["compat"] = lambda: (eng.crf_forward_train_compat_dev(unary, image, p, mu, q_hist, stream=s.cuda_stream),
                                  eng.crf_backward_compat_dev(q_hist, image, p, mu, G, gu, grad_compat=gmu,
                                                              stream=s.cuda_stream))
    if kernel and not wide:
        from dsrg_b200 import _lib
        gt = torch.empty((B, 7), device="cuda")
        before = _lib.lib().dsrg_engine_device_bytes(eng.h)
        legs["train_theta"] = lambda: (eng.crf_forward_train_dev(unary, image, p, q_hist, stream=s.cuda_stream),
                                       eng.crf_backward_theta_dev(q_hist, image, p, G, gu, gt, grad_potts=gw,
                                                                  stream=s.cuda_stream))
        if compat:
            legs["compat_theta"] = lambda: (
                eng.crf_forward_train_compat_dev(unary, image, p, mu, q_hist, stream=s.cuda_stream),
                eng.crf_backward_compat_theta_dev(q_hist, image, p, mu, G, gu, gt, grad_compat=gmu,
                                                  stream=s.cuda_stream))
        with torch.cuda.stream(s):
            legs["train_theta"]()
        torch.cuda.synchronize()
        extra["kgrad_bytes"] = int(_lib.lib().dsrg_engine_device_bytes(eng.h) - before)
    if features and not wide:
        feat = _image_features(torch, image, p)
        gf, gsp = torch.empty_like(feat), torch.empty((B, 2), device="cuda")
        legs["train_feat"] = lambda: (
            eng.crf_forward_train_feat_dev(unary, feat, p, q_hist, stream=s.cuda_stream),
            eng.crf_backward_feat_dev(q_hist, feat, p, G, gu, gf, grad_potts=gw, grad_theta_sp=gsp,
                                      stream=s.cuda_stream))
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
    eng.close()
    med = {k: float(np.median(v)) for k, v in times.items()}
    if compat:
        extra["compat_over_train"] = round(med["compat"] / med["train"], 2)
    if features and not wide:
        extra["train_feat_over_train"] = round(med["train_feat"] / med["train"], 2)
    if wide:
        extra["wide_potts_over_forward"] = round(med["wide_potts"] / med["forward"], 2)
        extra["wide_compat_over_forward"] = round(med["wide_compat"] / med["forward"], 2)
        for k in ("wide_theta", "wide_feat"):
            if k in med:
                extra[k + "_over_wide_potts"] = round(med[k] / med["wide_potts"], 2)
    elif kernel:
        extra["train_theta_over_train"] = round(med["train_theta"] / med["train"], 2)
        if compat:
            extra["compat_theta_over_compat"] = round(med["compat_theta"] / med["compat"], 2)
    return dict(**extra, workload=name, B=B, H=H, W=W, M=M, scale_factor=sf, image=img, n_iters=T,
                ms_per_step={k: round(v, 3) for k, v in med.items()},
                spread_ms={k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
                **({} if wide else dict(train_over_forward=round(med["train"] / med["forward"], 2))),
                q_hist_bytes=(T + 1) * B * M * H * W * 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--compat", action="store_true", help="also time the compatibility-matrix step")
    ap.add_argument("--kernel", action="store_true", help="also time the steps with the kernel-bandwidth gradient")
    ap.add_argument("--features", action="store_true",
                    help="also time the step with caller-given bilateral features (implies --kernel without --wide)")
    ap.add_argument("--wide", action="store_true",
                    help="time the label-chunked steps at 81 labels instead, on their own workloads")
    a = ap.parse_args()
    a.kernel = a.kernel or (a.features and not a.wide)
    if a.wide and a.workloads == ",".join(WORKLOADS):
        a.workloads = ",".join(WIDE_WORKLOADS)
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_crf_grad.py needs a CUDA device")
    info = card()
    for name in a.workloads.split(","):
        # --compat times a fused-path leg; --kernel and --features the fused or the label-chunked ones (--wide)
        r = run(name, a.steps, a.warmup, a.rounds, a.compat and not a.wide, a.kernel, a.features, a.wide)
        r.update(info)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
