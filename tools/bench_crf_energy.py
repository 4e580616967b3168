"""Time the CRF energy (dsrg_crf_energy_dev) and its gradient (dsrg_crf_energy_backward_dev) against one mean-field
inference, per call:

  inference  dsrg_crf_batch_dev with 10 iterations, NCHW in and out (CRF()'s mean field)
  energy     dsrg_crf_energy_dev of the inference's marginals with the unary: the lattice build, one splat, the
             forward blur and the per-pixel pass
  energy_bwd dsrg_crf_energy_dev then dsrg_crf_energy_backward_dev (the backward rebuilds the lattices and adds the
             transposed blur of the same splat), what a training step with nn.dense_crf_energy runs

on train-s's shape (batch 20 at 41 x 41, scale factor 12) and batch 64 at 321 x 321 with 21 labels on smooth and
photo-like images.  --wide times the label-chunked pair (dsrg_crf_energy_wide_dev, dsrg_crf_energy_backward_wide_dev)
at COCO's 81 labels instead, against the label-chunked inference: batch 20 at 41 x 41 (scale factor 12) on smooth
images and batch 8 at 321 x 321 on photo-like ones.  A mean-field call is one lattice build and 10 iterations, so energy / inference near 1/10 means the
energy costs about one iteration beyond the lattice build.  The per-kernel split of one energy_bwd call (the engine's
event profile) is printed with each line.

The legs run on a side stream (the engine's CUDA graphs need one), are warmed up, and alternate in rounds within one
session; each window is timed with CUDA events.  One JSON line per workload with the median ms per call of each leg,
the spread, and the card's name, power limit and SM clocks read in the same run.

usage: python tools/bench_crf_energy.py [--wide] [--steps 10] [--warmup 3] [--rounds 5] [--workloads ...]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_crf_learned import _timed  # noqa: E402
from bench_torch_step import card  # noqa: E402

WORKLOADS = {   # name -> (B, H, W, M, scale factor, image)
    "train_s": (20, 41, 41, 21, 12.0, "smooth"),
    "b64_smooth": (64, 321, 321, 21, 1.0, "smooth"),
    "b64_photo": (64, 321, 321, 21, 1.0, "photo"),
}
WIDE_WORKLOADS = {   # the label-chunked path at COCO's 81 labels
    "coco_train": (20, 41, 41, 81, 12.0, "smooth"),
    "coco_b8_photo": (8, 321, 321, 81, 1.0, "photo"),
}
T = 10


def run(name, steps, warmup, rounds, wide=False):
    import torch
    from dsrg_b200 import api, synth
    B, H, W, M, sf, img = (WIDE_WORKLOADS if wide else WORKLOADS)[name]
    batch = synth.make_batch(B, H, W, C=M, image=img, start=3, unique=8)
    unary = torch.from_numpy(np.log(np.maximum(batch["probs"], 1e-5)).astype(np.float32)).cuda()
    image = torch.from_numpy(batch["image"]).cuda()
    p = api.crf_params(sf, 13, T)
    eng = api.Engine(B, H, W, M)
    s = torch.cuda.Stream()
    q = torch.empty_like(unary)
    terms = torch.empty((B, 4), device="cuda")
    g = torch.ones((B, 4), device="cuda")
    grad_q = torch.empty_like(unary)
    ss = s.cuda_stream
    energy, energy_bwd = ((eng.crf_energy_wide_dev, eng.crf_energy_backward_wide_dev) if wide
                          else (eng.crf_energy_dev, eng.crf_energy_backward_dev))
    legs = {
        "inference": lambda: eng.crf_dev(unary, image, p, q, api.LAYOUT_NCHW, api.LAYOUT_NCHW, stream=ss),
        "energy": lambda: energy(q, unary, image, p, terms, stream=ss),
        "energy_bwd": lambda: (energy(q, unary, image, p, terms, stream=ss),
                               energy_bwd(q, unary, image, p, g, grad_q, stream=ss)),
    }
    b0 = eng.device_bytes
    with torch.cuda.stream(s):
        legs["inference"]()
        legs["energy_bwd"]()
    torch.cuda.synchronize()
    b1 = eng.device_bytes
    times = _timed(torch, s, legs, steps, warmup, rounds)
    torch.cuda.synchronize()
    eng.profile(True)   # one call per leg outside the timed windows: the per-kernel split (graphs are off meanwhile)
    with torch.cuda.stream(s):
        legs["energy_bwd"]()
    prof = eng.profile_read()
    eng.profile(False)
    ok = bool(torch.isfinite(terms).all() and torch.isfinite(grad_q).all())
    eng.close()
    med = {k: float(np.median(v)) for k, v in times.items()}
    return dict(workload=name, B=B, H=H, W=W, M=M, scale_factor=sf, image=img, n_iters=T,
                ms_per_call={k: round(v, 3) for k, v in med.items()},
                spread_ms={k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
                energy_over_inference=round(med["energy"] / med["inference"], 3),
                energy_bwd_over_inference=round(med["energy_bwd"] / med["inference"], 3),
                energy_bwd_profile_ms={k: round(v[0], 3) for k, v in sorted(prof.items())},
                first_energy_call_bytes=int(b1 - b0), finite=ok)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--workloads", default=None, help="comma-separated; default: every workload of the mode")
    ap.add_argument("--wide", action="store_true",
                    help="time the label-chunked energy at 81 labels instead, on its own workloads")
    a = ap.parse_args()
    if a.workloads is None:
        a.workloads = ",".join(WIDE_WORKLOADS if a.wide else WORKLOADS)
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_crf_energy.py needs a CUDA device")
    info = card()
    for name in [w for w in a.workloads.split(",") if w]:
        r = run(name, a.steps, a.warmup, a.rounds, a.wide)
        r.update(info)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
