"""Time one training step of train-s's stage-1 head (Softmax -> CRF -> DSRG -> BalancedSeedLoss + ConstrainLoss,
train-s.prototxt:746-812), forward plus backward, three ways:

  head      dsrg_b200.nn.DSRGHead: one mean-field pass shared by the CRF and DSRG layers
  composed  the same layers composed from the dsrg_b200.nn functions (crf_layer + dsrg_seeds): two passes
  dropin    the drop-in Caffe layers (dsrg_b200/dropin/pylayers) through caffe_shim on host numpy blobs, the
            diffs of the shared blobs summed the way Caffe's split layers do

at train-s's shape: 21 labels, 41 x 41 score maps, 321 x 321 images, batch 20 by default.  The torch legs run on a
side stream, as a training loop that wants the engine's own CUDA graphs does (they need a real stream).  Each leg is
warmed up, then timed with CUDA events around the window (the drop-in leg's host calls end in a synchronisation,
so its window covers the host work and the copies too).  Prints one JSON line with the card's name, power limit and
SM clocks read in the same run.

usage: python tools/bench_torch_step.py [--batch 20] [--steps 50] [--warmup 10] [--legs head,composed,dropin]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

M, H, W, HI = 21, 41, 41, 321


def card():
    """Name, power limit and SM clocks of GPU 0 (a read-only nvidia-smi query; None where it is unavailable)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, limit, sm, sm_max = [s.strip() for s in out.stdout.strip().split(",")]
        return dict(gpu=name, power_limit=limit, sm_clock=sm, max_sm_clock=sm_max)
    except Exception:
        return dict(gpu=None, power_limit=None, sm_clock=None, max_sm_clock=None)


def inputs(B, seed=0):
    from dsrg_b200 import synth
    batch = synth.make_batch(B, H, W, C=M, cues="cam", image="smooth", start=seed)
    rng = np.random.RandomState(seed)
    fc8 = (np.log(batch["probs"]) + 0.3 * rng.randn(B, M, H, W)).astype(np.float32)
    images = rng.rand(B, 3, HI, HI) * 255.0 - np.array([104.0, 117.0, 123.0])[None, :, None, None]
    images = ((images + np.roll(images, 1, 2) + np.roll(images, 1, 3)) / 3).astype(np.float32)
    return dict(fc8=fc8, images=images, labels=batch["labels"].reshape(B, 1, 1, M).astype(np.float32),
                cues=batch["cues"].astype(np.float32))


def torch_step(inp, composed):
    import torch
    from dsrg_b200 import nn
    d = {k: torch.from_numpy(v).cuda() for k, v in inp.items()}
    fc8 = d["fc8"].requires_grad_()
    head = nn.DSRGHead()

    def step():
        fc8.grad = None
        if composed:
            probs = nn.softmax(fc8)
            log_crf, probs_c = nn.crf_layer(probs, d["images"])
            seeds = nn.dsrg_seeds(d["labels"], probs_c, d["cues"], d["images"])
            ls, lc = nn.balanced_seed_loss(probs_c, seeds), nn.constrain_loss(probs_c, log_crf)
        else:
            ls, lc, _ = head(fc8, d["images"], d["labels"], d["cues"])
        (ls + lc).backward()
    return step


def dropin_step(inp):
    from dsrg_b200.dropin import caffe_shim
    caffe_shim.install()
    import pylayers
    Blob = caffe_shim.Blob

    def view(blob):   # a second top of a split blob: the same data, a diff of its own
        b = Blob()
        b.data, b.diff = blob.data, np.zeros_like(blob.data)
        return b
    fc8, images, labels, cues = Blob(inp["fc8"]), Blob(inp["images"]), Blob(inp["labels"]), Blob(inp["cues"])
    probs, log_crf, seeds, l_seed, l_con = Blob(), Blob(), Blob(), Blob(), Blob()
    layers = [(pylayers.SoftmaxLayer(), "", [fc8], [probs]),
              (pylayers.CRFLayer(), "", [probs, images], [log_crf]),
              (pylayers.DSRGLayer(), "{'th1': 0.99, 'th2': 0.85}", [labels, probs, cues, images], [seeds]),
              (pylayers.BalancedSeedLossLayer(), "", [probs, seeds], [l_seed]),
              (pylayers.ConstrainLossLayer(), "", [probs, log_crf], [l_con])]
    for layer, param_str, bottom, top in layers:
        layer.param_str = param_str
        layer.setup(bottom, top)
        layer.reshape(bottom, top)
    sm, crf, dsrg, bsl, con = (layer for layer, _, _, _ in layers)
    p_seed, p_con, p_crf = view(probs), view(probs), view(probs)
    log_con = view(log_crf)

    def step():
        fc8.data[...] = inp["fc8"]
        sm.forward([fc8], [probs])
        crf.forward([probs, images], [log_crf])
        dsrg.forward([labels, probs, cues, images], [seeds])
        bsl.forward([probs, seeds], [l_seed])
        con.forward([probs, log_crf], [l_con])
        bsl.backward([l_seed], [True, False], [p_seed, seeds])
        con.backward([l_con], [True, True], [p_con, log_con])
        log_crf.diff[...] = log_con.diff
        crf.backward([log_crf], [True, False], [p_crf, images])
        probs.diff[...] = p_seed.diff + p_con.diff + p_crf.diff   # Caffe's split layer sums the diffs
        sm.backward([probs], [True], [fc8])
    return step


def time_leg(step, steps, warmup):
    import torch
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        for _ in range(warmup):
            step()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            step()
        b.record()
    b.synchronize()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=20)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--legs", default="head,composed,dropin")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_torch_step.py needs a CUDA device")
    inp = inputs(args.batch)
    res = dict(bench="torch_step", batch=args.batch, labels=M, maps=[H, W], images=[HI, HI], steps=args.steps,
               warmup=args.warmup)
    legs = args.legs.split(",")
    for leg in legs:
        step = dropin_step(inp) if leg == "dropin" else torch_step(inp, composed=(leg == "composed"))
        ms = time_leg(step, args.steps, args.warmup)
        res[leg + "_ms"] = round(ms, 4)
        res[leg + "_images_per_s"] = round(1e3 * args.batch / ms, 1)
    if "head" in legs and "composed" in legs:
        res["head_vs_composed"] = round(res["composed_ms"] / res["head_ms"], 3)
    res.update(card())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
