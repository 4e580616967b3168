"""oracle/ref_coco_layer.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE (dev container only).

Runs the reference's OWN AnnotationLayerCOCO (pylayers/pylayers/pylayers.py:389-512) in place, the way
oracle/ref_layers.py runs the other layers: its ``ClassDef`` node is pulled out with ``ast`` (the module itself cannot
be imported: it needs caffe, theano and cPickle at import time; nothing is copied) and executed in a namespace of its
own.  The outputs pin ``oracle/annot_coco_oracle.py``: tests/golden/make_annot_coco_golden.py freezes them in
tests/golden/annot_coco_ref.npz, and tests/test_annot_coco_cpu.py compares live when the reference is mounted.
"""
import ast
import os
import types

import numpy as np

from .ref_layers import REF_FILE, Blob, available  # noqa: F401
_COCO_NS = None


def _coco_namespace():
    """AnnotationLayerCOCO in a namespace of its own: the module-level names its methods use are supplied --
    ``zoom``, numpy.random's ``shuffle`` (pylayers.py:4, :14), ``xrange = range`` and a ``cv2`` whose imread is
    replaced per call (see annotation_coco_layer_forward)."""
    global _COCO_NS
    if _COCO_NS is None:
        from scipy.ndimage import zoom
        with open(REF_FILE) as fh:
            tree = ast.parse(fh.read())
        keep = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "AnnotationLayerCOCO"]
        caffe = types.ModuleType("caffe")
        caffe.Layer = type("Layer", (object,), {"param_str": ""})
        cv2 = types.ModuleType("cv2")
        cv2.IMREAD_COLOR, cv2.IMREAD_GRAYSCALE = 1, 0
        ns = {"np": np, "caffe": caffe, "zoom": zoom, "shuffle": np.random.shuffle, "xrange": range, "cv2": cv2,
              "osp": os.path}
        exec(compile(ast.Module(body=keep, type_ignores=[]), REF_FILE, "exec"), ns)
        _COCO_NS = ns
    return _COCO_NS


def annotation_coco_layer_forward(files, indexlist, cur, root, batch_size, mean, new_size, is_mirror=False,
                                  ignore_label=255):
    """The reference's own AnnotationLayerCOCO.forward (pylayers.py:432-512), reading `files` (path -> decoded
    array) through the cv2 stand-in.  setup() is skipped -- it divides with Python 2's `/` and opens a
    multiprocessing.Queue (:391-417) -- and its attributes are set directly.  Shuffles `indexlist` in place like the
    reference; returns (top0, top1, top2, the new _cur)."""
    ns = _coco_namespace()
    ns["cv2"].imread = lambda path, flag: np.array(files[path])
    layer = ns["AnnotationLayerCOCO"]()
    layer.root_folder = root
    layer.batch_size = batch_size
    layer.is_mirror = is_mirror
    layer.mean = mean
    layer.new_h, layer.new_w = new_size
    layer.ignore_label = ignore_label
    layer.indexlist = indexlist
    layer._cur = cur
    new_h, new_w = new_size
    top = [Blob(), Blob(), Blob()]
    top[0].reshape(batch_size, 1, 1, 81)
    top[1].reshape(batch_size, 81, new_h // 8 + 1, new_w // 8 + 1)
    top[2].reshape(batch_size, 3, new_h, new_w)
    layer.forward([], top)
    return top[0].data, top[1].data, top[2].data, layer._cur
