"""tests/golden/make_sec_golden.py -- regenerates tests/golden/sec_layers_ref.npz.

Runs only where the reference is mounted: the reference's own SeedLossLayer and ExpandLossLayer class bodies
(pylayers/pylayers/pylayers.py:95-118, :183-233) are executed in place (oracle/sec_layers.py, Theano stand-in),
in float64 and in float32, on the seeded inputs below.  The file pins oracle/sec_oracle.py
(tests/test_sec_losses_cpu.py) and the device layers (tests/test_gpu_sec_losses.py).

usage: python tests/golden/make_sec_golden.py
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import loss_oracle  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))

SEED_CASES = {"s0": (3, 21, 9, 7, False), "s1": (3, 21, 9, 7, True), "s2": (2, 5, 13, 4, False)}  # N, C, H, W, empty
EXPAND_CASES = {"e0": (3, 101), "e1": (2, 102)}   # N, seed; the reference's graph fixes (21, 41, 41)


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def softmax_probs(logits):
    """SoftmaxLayer's output (pylayers.py:33-36) in float32."""
    return loss_oracle.softmax_layer_forward(logits).astype(np.float32)


def seed_inputs(name):
    """probs and seed masks; `empty` gives image 1 no seeds at all (the loss is then NaN)."""
    N, C, H, W, empty = SEED_CASES[name]
    rng = np.random.RandomState(7000 + int(name[1:]))
    probs = softmax_probs(3 * rng.randn(N, C, H, W))
    lab = (rng.rand(N, C, H, W) < 0.1).astype(np.float32)
    lab[0, 0, 0, 0] = 1.0
    if empty:
        lab[1] = 0
    return probs, lab


def expand_inputs(name, saturate=True):
    """probs (N, 21, 41, 41) from SoftmaxLayer on random logits and labels (N, 1, 1, 21).  Image 0 has saturated
    logits (planes of identical floored values, a tie group at a plane max), image 1 no present foreground class
    (P = 0) when N > 2, image N-1 every foreground class present (A = 0) when N > 2."""
    N, seed = EXPAND_CASES[name]
    rng = np.random.RandomState(seed)
    logits = 2 * rng.randn(N, 21, 41, 41)
    if saturate:
        logits[0, 7, :20] = 40.0     # class 7 wins the top rows outright: a tie group at its max
        logits[0, 5] = -40.0         # class 5 loses everywhere: its values are the floor, up to normalisation
        logits[0, 0, :, 30:] = 40.0  # background, too
    probs = softmax_probs(logits)
    if saturate:
        probs[0, 9] = probs[0, 9].min()   # one exactly constant plane: every element ties with the max
    labels = np.zeros((N, 1, 1, 21), np.float32)
    labels[:, 0, 0, 0] = 1.0
    for b in range(N):
        labels[b, 0, 0, rng.choice(np.arange(1, 21), size=rng.randint(1, 4), replace=False)] = 1.0
    labels[0, 0, 0, [7, 9]] = 1.0
    if N > 2:
        labels[1, 0, 0, 1:] = 0.0
        labels[N - 1, 0, 0, 1:] = 1.0
    return probs, labels


def main():
    from oracle import sec_layers
    assert sec_layers.available(), "needs the reference's pylayers.py"
    rec = {}
    for name in SEED_CASES:
        probs, lab = seed_inputs(name)
        rec[name + "_sha256"] = digest(probs, lab)
        for dt in ("float64", "float32"):
            rec["%s_%s_loss" % (name, dt)], rec["%s_%s_grad" % (name, dt)] = sec_layers.seed_loss_layer(probs, lab, dt)
        print("seed", name, float(rec[name + "_float64_loss"]))
    for name in EXPAND_CASES:
        probs, labels = expand_inputs(name)
        rec[name + "_sha256"] = digest(probs, labels)
        for dt in ("float64", "float32"):
            rec["%s_%s_loss" % (name, dt)], rec["%s_%s_grad" % (name, dt)] = \
                sec_layers.expand_loss_layer(probs, labels, dt)
        print("expand", name, float(rec[name + "_float64_loss"]))
    np.savez_compressed(os.path.join(OUT, "sec_layers_ref.npz"), **rec)


if __name__ == "__main__":
    main()
