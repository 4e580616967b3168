"""Scoring of segmentation results: the confusion matrix and the metrics of the reference's evaluation tools, with
the matrix counted on the device (csrc/eval.cu, dsrg_confusion_*).

* ``ConfusionMatrix``    -- training/tools/evaluate.py:17-68 (column sums for recall, row sums for accuracy)
* ``APConfusionMatrix``  -- training/tools/ap.py:19-72 (row sums for recall, column sums for accuracy, ``max(., 1)``
  denominators, per-class lists)
* ``get_confusion_matrix`` and ``mean_iu`` -- training/tools/test-coco.py:62-81 and :151-156

The metric formulas are restated in float64 in the reference's order of operations, so they give the reference's
values bit for bit, NaN included.  The matrix differs from the reference's in one case, by design: test-coco.py
forms ``gt * class_num`` on uint8 ground truth, which wraps mod 256 (K = 81: gt = 4, pred = 4 is counted in row 0,
column 72); here every pair lands in its own bin.

Counting needs the CUDA library and a GPU: there is no CPU fallback.  The formulas work on any matrix.
"""
import numpy as np

from . import api as _api

_GROUP_PIXELS = 1 << 24   # generateM_all: items are concatenated into groups of about this many pixels


def _flat_gt(gt):
    gt = np.ascontiguousarray(gt).reshape(-1)
    if gt.dtype == np.uint8:
        return gt
    if gt.dtype.kind not in "iu":
        raise TypeError("gt must be an integer label map, not %s" % gt.dtype)
    if gt.size and (gt.min() < 0 or gt.max() > 255):
        raise ValueError("gt labels must be 8-bit (0..255), as a label PNG holds them")
    return gt.astype(np.uint8)


class ConfusionMatrix(object):
    """The surface of evaluate.py's ConfusionMatrix: ``nclass``, ``classes``, ``M`` (float64, rows = ground truth,
    columns = prediction), ``add``, ``addM``, ``generateM``, ``recall``, ``accuracy``, ``jaccard``, plus
    ``generateM_all`` for a whole list of images in one device pass."""

    def __init__(self, nclass, classes=None, device=None):
        self.nclass = int(nclass)
        self.classes = classes
        self._device = device
        self._conf = None        # dsrg_confusion of add(): created on first use
        self._scratch = None     # dsrg_confusion of generateM / generateM_all
        self._host = np.zeros((self.nclass, self.nclass))   # what addM() and assignments to M contributed
        self._cache = None

    def _obj(self, name):
        if getattr(self, name) is None:
            setattr(self, name, _api.Confusion(self.nclass, self._device))
        return getattr(self, name)

    @property
    def M(self):
        if self._cache is None:
            m = self._host
            if self._conf is not None:
                m = m + self._conf.read()[0].astype(np.float64)
            self._cache = m
        return self._cache

    @M.setter
    def M(self, value):
        value = np.array(value, dtype=np.float64)
        if value.shape != (self.nclass, self.nclass):
            raise ValueError("M must be %d x %d" % (self.nclass, self.nclass))
        if self._conf is not None:
            self._conf.reset()
        self._host = value
        self._cache = None

    def add(self, gt, pred):
        """evaluate.py:24-29: count every pixel whose gt is not 255.  Any other gt or pred outside [0, nclass)
        raises IndexError before anything is counted (the reference raises at the first such pixel; a negative
        pred, which the reference would count in the last column, raises too)."""
        gt = np.asarray(gt).reshape(-1)
        pred = np.asarray(pred).reshape(-1)
        if gt.size != pred.size:
            raise ValueError("gt and pred differ in size (%d vs %d)" % (gt.size, pred.size))
        keep = gt != 255
        if np.any(keep & ((gt < 0) | (gt >= self.nclass))):
            raise IndexError("gt label outside [0, %d) and not 255" % self.nclass)
        if np.any(keep & ((pred < 0) | (pred >= self.nclass))):
            raise IndexError("pred label outside [0, %d)" % self.nclass)
        self._obj("_conf").add_host(_flat_gt(gt), pred)
        self._cache = None

    def addM(self, matrix):
        matrix = np.asarray(matrix)
        if matrix.shape != (self.nclass, self.nclass):
            raise ValueError("matrix must be %d x %d" % (self.nclass, self.nclass))
        self._host = self._host + matrix
        self._cache = None

    def _count(self, items):
        conf = self._obj("_scratch")
        conf.reset()
        for gt, pred in items:
            conf.add_host(gt, pred)
        m, inv = conf.read()
        if inv[1]:
            raise IndexError("%d pixels with gt < %d have a pred outside [0, %d)" % (inv[1], self.nclass, self.nclass))
        return m.astype(np.float64)

    def generateM(self, item):
        """evaluate.py:61-68: the matrix of one (gt, pred) pair of flat label maps; pixels with gt >= nclass are
        skipped.  A pred outside [0, nclass) where gt < nclass raises IndexError."""
        gt, pred = item
        if np.size(gt) != np.size(pred):
            raise ValueError("gt and pred differ in size (%d vs %d)" % (np.size(gt), np.size(pred)))
        return self._count([(_flat_gt(gt), pred)])

    def generateM_all(self, items):
        """The sum of generateM over `items`, as one device pass: replaces
        ``m_list = Pool().map(ConfM.generateM, data_list); for m in m_list: ConfM.addM(m)`` (evaluate.py:148-156)
        with ``ConfM.addM(ConfM.generateM_all(data_list))``.  Items are concatenated into large host chunks, which
        the device counts while the next chunk is copied."""
        def groups():
            gts, preds, n = [], [], 0
            for gt, pred in items:
                gt, pred = _flat_gt(gt), _api._pred_host(pred, self.nclass)
                if gt.size != pred.size:
                    raise ValueError("gt and pred differ in size (%d vs %d)" % (gt.size, pred.size))
                if preds and pred.dtype != preds[0].dtype:
                    pred = pred.astype(np.int32)
                    preds = [p.astype(np.int32) for p in preds]
                gts.append(gt)
                preds.append(pred)
                n += gt.size
                if n >= _GROUP_PIXELS:
                    yield np.concatenate(gts), np.concatenate(preds)
                    gts, preds, n = [], [], 0
            if gts:
                yield np.concatenate(gts), np.concatenate(preds)
        return self._count(groups())

    # ---- metrics (evaluate.py:40-59), float64, in the reference's order of operations ----
    def recall(self):
        M, r = self.M, 0.0
        with np.errstate(divide="ignore", invalid="ignore"):
            for i in range(self.nclass):
                r += M[i, i] / np.sum(M[:, i])
        return r / self.nclass

    def accuracy(self):
        M, a = self.M, 0.0
        with np.errstate(divide="ignore", invalid="ignore"):
            for i in range(self.nclass):
                a += M[i, i] / np.sum(M[i, :])
        return a / self.nclass

    def jaccard(self):
        """(mean IoU over the classes with a true positive, their IoUs, M)."""
        M = self.M
        per = [M[i, i] / (np.sum(M[i, :]) + np.sum(M[:, i]) - M[i, i]) for i in range(self.nclass) if M[i, i] != 0]
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.sum(per) / len(per), per, M


class APConfusionMatrix(ConfusionMatrix):
    """ap.py's ConfusionMatrix: recall and accuracy return (mean, per-class list) with the sums the other way
    round from evaluate.py's and ``max(sum, 1)`` as the denominator (ap.py:40-54)."""

    def recall(self):
        M = self.M
        per = [M[i, i] / max(np.sum(M[i, :]), 1) for i in range(self.nclass)]
        return np.sum(per) / self.nclass, per

    def accuracy(self):
        M = self.M
        per = [M[i, i] / max(np.sum(M[:, i]), 1) for i in range(self.nclass)]
        return np.sum(per) / self.nclass, per


def get_confusion_matrix(gt_label, pred_label, class_num, device=None):
    """test-coco.py:62-81, counted on the device: the (class_num, class_num) float64 matrix of the (gt, pred) pairs.
    Pixels with gt >= class_num (255 among them) are skipped; a pred outside [0, class_num) where gt < class_num
    raises ValueError.  Every pair lands in its own bin: the reference's uint8 ``gt * class_num`` wraps, this does
    not."""
    conf = _api.Confusion(class_num, device)
    try:
        conf.add_host(_flat_gt(gt_label), pred_label)
        m, inv = conf.read()
    finally:
        conf.close()
    if inv[1]:
        raise ValueError("%d pixels with gt < %d have a pred outside [0, %d)" % (inv[1], class_num, class_num))
    return m.astype(np.float64)


def mean_iu(confusion_matrix):
    """test-coco.py:151-156: (mean IU, per-class IU) with IU = tp / max(1, pos + res - tp)."""
    M = np.asarray(confusion_matrix, dtype=np.float64)
    pos, res, tp = M.sum(1), M.sum(0), np.diag(M)
    iu = tp / np.maximum(1.0, pos + res - tp)
    return iu.mean(), iu
