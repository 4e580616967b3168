"""oracle/eval_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE (dev container only).

Runs the reference's OWN scoring code in place: the ``ConfusionMatrix`` classes of
/root/reference/training/tools/evaluate.py and ap.py, and ``get_confusion_matrix`` of test-coco.py.  The scripts
cannot be imported (they import cv2, copy_reg, caffe and pylab at top level), so their ``ClassDef`` /
``FunctionDef`` nodes are pulled out with ``ast`` and executed in a namespace that supplies ``np`` and
``xrange = range``; nothing is copied.  tests/golden/make_eval_golden.py freezes the outputs in
tests/golden/eval_ref.npz, and tests/test_eval_cpu.py compares live when the reference is mounted.
"""
import ast
import os

import numpy as np

TOOLS = "/root/reference/training/tools"
_NS = {}


def available():
    return all(os.path.exists(os.path.join(TOOLS, f)) for f in ("evaluate.py", "ap.py", "test-coco.py"))


def _load(script, names):
    if script not in _NS:
        path = os.path.join(TOOLS, script)
        with open(path) as fh:
            tree = ast.parse(fh.read())
        keep = [n for n in tree.body if isinstance(n, (ast.ClassDef, ast.FunctionDef)) and n.name in names]
        ns = {"np": np, "xrange": range}
        exec(compile(ast.Module(body=keep, type_ignores=[]), path, "exec"), ns)
        _NS[script] = ns
    return _NS[script]


def evaluate_cm():
    """evaluate.py's ConfusionMatrix class."""
    return _load("evaluate.py", ("ConfusionMatrix",))["ConfusionMatrix"]


def ap_cm():
    """ap.py's ConfusionMatrix class."""
    return _load("ap.py", ("ConfusionMatrix",))["ConfusionMatrix"]


def get_confusion_matrix(gt_label, pred_label, class_num):
    """test-coco.py's get_confusion_matrix, as it runs (uint8 gt_label * class_num wraps mod 256)."""
    return _load("test-coco.py", ("get_confusion_matrix",))["get_confusion_matrix"](gt_label, pred_label, class_num)
