"""tests/golden/make_eval_golden.py -- regenerates tests/golden/eval_ref.npz.

Runs only where the reference is mounted: the reference's own ConfusionMatrix classes (training/tools/evaluate.py,
ap.py) and get_confusion_matrix (test-coco.py) are executed in place (oracle/eval_oracle.py) on the seeded label maps
below.  The file pins dsrg_b200/metrics.py: tests/test_eval_cpu.py (the formulas, on the frozen matrices) and
tests/test_gpu_eval.py (the device-counted matrices).

usage: python tests/golden/make_eval_golden.py
"""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "eval_ref.npz")
KS = (2, 21, 22, 81, 82)
SIZES = ((23, 31), (40, 17), (9, 64))   # one image per size; image 1's prediction is int64 (np.argmax), the others uint8


def eval_inputs(K, index):
    """A ground-truth map (uint8) with a background majority, blocky class regions, an ignore (255) rectangle and
    a few labels >= K other than 255, and a prediction that agrees on ~70 % of the pixels.  Where gt >= K the
    prediction holds values >= K too: generateM skips those pixels."""
    H, W = SIZES[index]
    rng = np.random.RandomState(9000 + 10 * K + index)
    coarse = rng.randint(0, K, ((H + 3) // 4, (W + 3) // 4))
    gt = np.repeat(np.repeat(coarse, 4, 0), 4, 1)[:H, :W]
    gt[rng.rand(H, W) < 0.5] = 0
    y, x = rng.randint(0, H - 3), rng.randint(0, W - 5)
    gt[y:y + 3, x:x + 5] = 255
    odd = rng.rand(H, W) < 0.03
    gt[odd] = rng.randint(K, 255, odd.sum()) if K < 255 else 255
    gt = gt.astype(np.uint8)
    pred = np.where(rng.rand(H, W) < 0.7, gt, rng.randint(0, K, (H, W)))
    pred[gt >= K] = rng.randint(0, 256, int((gt >= K).sum()))
    return gt, pred.astype(np.int64 if index == 1 else np.uint8)


def add_inputs(gt, pred, K):
    """What ConfusionMatrix.add accepts (evaluate.py:24-29): no gt >= K other than 255, every pred <= K."""
    bad = gt >= K
    return np.where(bad, 255, gt).astype(np.uint8), np.where(bad, 0, pred).astype(pred.dtype)


def main():
    from oracle import eval_oracle
    if not eval_oracle.available():
        sys.exit("the reference is not mounted")
    EvCM, ApCM = eval_oracle.evaluate_cm(), eval_oracle.ap_cm()
    out = {}
    warnings.simplefilter("ignore", RuntimeWarning)   # 0/0 of classes that never occur: NaN, as the reference gives
    for K in KS:
        ev, ap, ev_add = EvCM(K), ApCM(K), EvCM(K)
        for i in range(len(SIZES)):
            gt, pred = eval_inputs(K, i)
            out["gt_%d_%d" % (K, i)], out["pred_%d_%d" % (K, i)] = gt, pred
            m = ev.generateM([gt.flatten(), pred.flatten()])
            ev.addM(m)
            ap.addM(ap.generateM([gt.flatten(), pred.flatten()]))
            ev_add.add(*[a.flatten() for a in add_inputs(gt, pred, K)])
            keep = gt != 255                                           # test-coco.py:165-167
            out["coco_%d_%d" % (K, i)] = eval_oracle.get_confusion_matrix(gt[keep], pred[keep].astype(np.int64), K)
        assert np.array_equal(ev.M, ap.M)
        out["M_%d" % K], out["M_add_%d" % K] = ev.M, ev_add.M
        out["ev_recall_%d" % K] = np.float64(ev.recall())
        out["ev_accuracy_%d" % K] = np.float64(ev.accuracy())
        j, per, _ = ev.jaccard()
        out["ev_jaccard_%d" % K], out["ev_jaccard_per_%d" % K] = np.float64(j), np.asarray(per, np.float64)
        for name in ("recall", "accuracy"):
            mean, per = getattr(ap, name)()
            out["ap_%s_%d" % (name, K)], out["ap_%s_per_%d" % (name, K)] = np.float64(mean), np.asarray(per, np.float64)
        j, per, _ = ap.jaccard()
        out["ap_jaccard_%d" % K], out["ap_jaccard_per_%d" % K] = np.float64(j), np.asarray(per, np.float64)
    # the wrap itself: K = 81, gt = 4, pred = 4 lands in row 0, column 72
    out["wrap_gt"], out["wrap_pred"] = np.array([4, 4, 0, 1], np.uint8), np.array([4, 4, 0, 2], np.int64)
    out["wrap_ref"] = eval_oracle.get_confusion_matrix(out["wrap_gt"], out["wrap_pred"], 81)
    np.savez_compressed(OUT, **out)
    print("wrote %s (%d arrays)" % (OUT, len(out)))


if __name__ == "__main__":
    main()
