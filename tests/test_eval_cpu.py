"""CPU tests of the scoring module (dsrg_b200/metrics.py): the metric formulas against the reference's own
ConfusionMatrix classes (training/tools/evaluate.py, ap.py) -- frozen in tests/golden/eval_ref.npz and, when the
reference is mounted, run live -- the uint8 wrap of test-coco.py's get_confusion_matrix, and that counting has no
CPU fallback."""
import warnings

import numpy as np
import pytest

from conftest import load_golden
from dsrg_b200 import _lib, api, metrics

KS = (2, 21, 22, 81, 82)


def same(a, b):
    """== on float64, NaN where the other is NaN."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


def ours(cls, M):
    cm = cls(M.shape[0])
    cm.M = M
    return cm


@pytest.mark.parametrize("K", KS)
def test_formulas_equal_frozen_reference(K):
    g = load_golden("eval_ref.npz")
    M = g["M_%d" % K]
    ev, ap = ours(metrics.ConfusionMatrix, M), ours(metrics.APConfusionMatrix, M)
    with warnings.catch_warnings():
        warnings.simplefilter("error")       # the formulas keep numpy quiet where the reference warns
        assert same(ev.recall(), g["ev_recall_%d" % K])
        assert same(ev.accuracy(), g["ev_accuracy_%d" % K])
        j, per, m = ev.jaccard()
        assert same(j, g["ev_jaccard_%d" % K]) and same(per, g["ev_jaccard_per_%d" % K]) and m is ev.M
        for name in ("recall", "accuracy"):
            mean, per = getattr(ap, name)()
            assert same(mean, g["ap_%s_%d" % (name, K)]) and same(per, g["ap_%s_per_%d" % (name, K)])
        j, per, _ = ap.jaccard()
        assert same(j, g["ap_jaccard_%d" % K]) and same(per, g["ap_jaccard_per_%d" % K])


def test_frozen_reference_has_nan_cases():
    """The goldens exercise the reference's NaN (a class never predicted or never present)."""
    g = load_golden("eval_ref.npz")
    assert any(np.isnan(g["ev_accuracy_%d" % K]) for K in KS)


def _random_matrices():
    rng = np.random.RandomState(5)
    for K in (1, 2, 21, 81, 255):
        M = rng.randint(0, 1000, (K, K)).astype(np.float64)
        M[:, rng.rand(K) < 0.2] = 0           # never predicted: evaluate.py's recall is NaN
        M[rng.rand(K) < 0.2] = 0              # never present
        yield M
    yield np.zeros((21, 21))                  # nothing at all: the mean IoU of no classes
    yield rng.rand(21, 21) * 1e6              # addM of non-integer matrices: the order of the sums matters


@pytest.mark.parametrize("i", range(7))
def test_formulas_equal_reference_live(i):
    from oracle import eval_oracle
    if not eval_oracle.available():
        pytest.skip("reference not mounted")
    M = list(_random_matrices())[i]
    for ref_cls, cls in ((eval_oracle.evaluate_cm(), metrics.ConfusionMatrix),
                         (eval_oracle.ap_cm(), metrics.APConfusionMatrix)):
        ref = ref_cls(M.shape[0])
        ref.M = M.copy()
        cm = ours(cls, M)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            for name in ("recall", "accuracy"):
                want, got = getattr(ref, name)(), getattr(cm, name)()
                if isinstance(want, tuple):
                    assert same(got[0], want[0]) and same(got[1], want[1])
                else:
                    assert same(got, want)
            want, got = ref.jaccard(), cm.jaccard()
        assert same(got[0], want[0]) and same(got[1], want[1]) and np.array_equal(got[2], want[2])


def test_reference_get_confusion_matrix_wraps_and_ours_is_intended():
    """test-coco.py forms gt * 81 in uint8: gt = 4, pred = 4 is counted in row 0, column 72.  The intended matrix
    (an int64 bincount restatement, which is what the device counts) has it at (4, 4)."""
    g = load_golden("eval_ref.npz")
    ref = g["wrap_ref"]
    from oracle import eval_oracle
    if eval_oracle.available():
        assert np.array_equal(eval_oracle.get_confusion_matrix(g["wrap_gt"], g["wrap_pred"], 81), ref)
    assert ref[0, 72] == 2 and ref[4, 4] == 0
    gt, pred = g["wrap_gt"].astype(np.int64), g["wrap_pred"]
    intended = np.bincount(gt * 81 + pred, minlength=81 * 81).reshape(81, 81)
    assert intended[4, 4] == 2 and intended[0, 72] == 0
    # VOC's 21 classes wrap as well: 20 * 21 = 420 > 255
    K = 21
    differs = 0
    for i in range(3):
        gt, pred = g["gt_%d_%d" % (K, i)], g["pred_%d_%d" % (K, i)]
        keep = gt != 255
        gt64, p64 = gt[keep].astype(np.int64), pred[keep].astype(np.int64)
        ok = gt64 < K
        want = np.bincount(gt64[ok] * K + p64[ok], minlength=K * K).reshape(K, K)
        differs += not np.array_equal(want, g["coco_%d_%d" % (K, i)])
    assert differs == 3


def test_mean_iu_restates_test_coco():
    g = load_golden("eval_ref.npz")
    for K in KS:
        M = g["M_%d" % K]
        mean, iu = metrics.mean_iu(M)
        tp = np.diag(M)
        want = tp / np.maximum(1.0, M.sum(1) + M.sum(0) - tp)
        assert np.array_equal(iu, want) and mean == want.mean()


def test_int64_predictions_are_narrowed_never_wrapped():
    pred = np.array([0, 3, 2 ** 32 + 1, -2 ** 32 + 2, -1, 2 ** 40, 20, 21], np.int64)
    got = api._pred_host(pred, 21)
    assert got.dtype == np.int32
    assert got.tolist() == [0, 3, -1, -1, -1, -1, 20, -1]
    assert api._pred_host(np.array([5, 300], np.uint16), 21).tolist() == [5, -1]
    u8 = np.array([1, 250], np.uint8)
    assert np.array_equal(api._pred_host(u8, 21), u8)   # uint8 and int32 go to the device as they are


def test_add_rejects_what_the_reference_rejects_before_counting():
    cm = metrics.ConfusionMatrix(21)
    with pytest.raises(IndexError):
        cm.add(np.array([3, 21], np.uint8), np.array([1, 1]))       # gt >= nclass, not 255
    with pytest.raises(IndexError):
        cm.add(np.array([3, 255], np.uint8), np.array([21, 1]))     # pred == nclass passes the reference's assert
    with pytest.raises(ValueError):
        cm.add(np.array([3], np.uint8), np.array([1, 1]))
    assert cm._conf is None and not cm.M.any()                      # nothing reached the device


def test_addM_and_assigned_M():
    cm = metrics.ConfusionMatrix(3)
    cm.addM(np.eye(3))
    cm.addM(2 * np.eye(3))
    assert np.array_equal(cm.M, 3 * np.eye(3)) and cm.M.dtype == np.float64
    with pytest.raises(ValueError):
        cm.addM(np.eye(4))


def test_no_cpu_fallback_for_counting():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.DsrgError):
        api.Confusion(21)
    with pytest.raises(_lib.DsrgError):
        metrics.ConfusionMatrix(21).generateM((np.zeros(4, np.uint8), np.zeros(4, np.uint8)))
    with pytest.raises(_lib.DsrgError):
        metrics.get_confusion_matrix(np.zeros(4, np.uint8), np.zeros(4, np.int64), 81)


def test_confusion_symbols_are_bound():
    names = ("dsrg_confusion_create", "dsrg_confusion_destroy", "dsrg_confusion_reset", "dsrg_confusion_add_dev",
             "dsrg_confusion_add_host", "dsrg_confusion_read")
    L = _lib.lib()
    for n in names:
        assert n in _lib.SIGNATURES and hasattr(L, n)
