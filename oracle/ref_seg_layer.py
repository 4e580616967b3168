"""oracle/ref_seg_layer.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE (dev container only).

Runs the reference's OWN pylayers/pylayers/layer.py classes (ImageSegDataLayer, BatchLoader, SimpleTransformer,
print_info) in place.  That module does not parse on Python 3 and imports caffe, cv2, PIL, skimage and scipy.misc at
the top, so its text is read, not imported, and nothing is copied:
  1. the ``if __name__ == '__main__':`` block is cut off;
  2. its two Python 2 print statements become ``pass`` (exactly two are replaced);
  3. after ``ast.parse`` every ``/`` becomes ``//`` (all six divide ints: the crop offsets, Python 2's integer
     division);
  4. the ``ClassDef`` / ``FunctionDef`` nodes are executed in a namespace of their own with numpy, Python's
     ``random`` (and its ``shuffle``), a stub ``caffe.Layer`` and a ``cv2`` whose ``copyMakeBorder`` is the real one
     and whose ``imread`` is replaced per call by in-memory arrays.
The outputs pin ``oracle/seg_data_oracle.py``: tests/golden/make_seg_data_golden.py freezes them in
tests/golden/seg_data_ref.npz, and tests/test_seg_data_cpu.py compares live when the reference and cv2 are present.
"""
import ast
import os
import random
import re
import types

import numpy as np

from .ref_layers import REF_FILE, Blob

LAYER_FILE = os.path.join(os.path.dirname(REF_FILE), "layer.py")
_NS = None


def available():
    if not os.path.exists(LAYER_FILE):
        return False
    try:
        import cv2  # noqa: F401
    except ImportError:
        return False
    return True


class _FloorDiv(ast.NodeTransformer):
    def visit_BinOp(self, node):
        self.generic_visit(node)
        if isinstance(node.op, ast.Div):
            node.op = ast.FloorDiv()
        return node


def namespace():
    """The reference's classes, defined by executing their own (Python 3-parsable) source in place."""
    global _NS
    if _NS is None:
        import cv2 as real_cv2
        with open(LAYER_FILE) as fh:
            src = fh.read()
        src = src.split("\nif __name__ == '__main__':")[0]
        src, n = re.subn(r'^([ \t]*)print (.*?\n(?:\1[ \t]+.*\n)*)', r'\1pass\n', src, flags=re.M)
        assert n == 2, "expected the reference's two print statements, replaced %d" % n
        tree = ast.parse(src, LAYER_FILE)
        keep = [_FloorDiv().visit(node) for node in tree.body if isinstance(node, (ast.ClassDef, ast.FunctionDef))]
        caffe = types.ModuleType("caffe")
        caffe.Layer = type("Layer", (object,), {"param_str": ""})
        cv2 = types.ModuleType("cv2")
        cv2.IMREAD_COLOR, cv2.IMREAD_GRAYSCALE = real_cv2.IMREAD_COLOR, real_cv2.IMREAD_GRAYSCALE
        cv2.BORDER_CONSTANT, cv2.copyMakeBorder = real_cv2.BORDER_CONSTANT, real_cv2.copyMakeBorder
        ns = {"np": np, "random": random, "shuffle": random.shuffle, "caffe": caffe, "cv2": cv2, "osp": os.path}
        exec(compile(ast.Module(body=keep, type_ignores=[]), LAYER_FILE, "exec"), ns)
        _NS = ns
    return _NS


def transformer(params):
    """The reference's SimpleTransformer(params); check_params fills in the caller's dict."""
    return namespace()["SimpleTransformer"](params)


def seg_layer_forward(files, indexlist, cur, root, batch_size, params):
    """The reference's own ImageSegDataLayer.forward (layer.py:51-61), reading `files` (path -> decoded array)
    through the cv2 stand-in.  setup() and BatchLoader.__init__ open the list file, so their attributes are set
    directly.  Shuffles `indexlist` in place like the reference; returns (top0, top1, the new _cur)."""
    ns = namespace()
    ns["cv2"].imread = lambda path, flag: np.array(files[path])
    params = dict(params, batch_size=batch_size, root_folder=root)
    loader = ns["BatchLoader"].__new__(ns["BatchLoader"])
    loader.batch_size = batch_size
    loader.root_folder = root
    loader.indexlist = indexlist
    loader._cur = cur
    loader.transformer = ns["SimpleTransformer"](params)
    layer = ns["ImageSegDataLayer"]()
    layer.batch_size = batch_size
    layer.input_shape = params["crop_size"]
    layer.batch_loader = loader
    top = [Blob(), Blob()]
    top[0].reshape(batch_size, 3, *params["crop_size"])
    top[1].reshape(batch_size, 1, *params["crop_size"])
    layer.forward([], top)
    return top[0].data, top[1].data, loader._cur
