"""oracle/prep_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The network input of the reference's evaluation tools, ``preprocess(image, size)``, two ways:

* ``reference(script, image, size)`` runs the reference's OWN ``preprocess`` of training/tools/test-ms.py,
  test-ms-f.py, test-coco.py or generate_train_gt.py in place (dev container only).  The scripts cannot be imported
  (they import caffe, cv2 and pylab at top level), so the script's ``mean_pixel = ...`` assignment and its
  ``preprocess`` ``FunctionDef`` are pulled out with ``ast`` and executed in a namespace that supplies ``np`` and
  ``nd``, the way oracle/eval_oracle.py does it; nothing is copied.
* ``preprocess(image, size, relative)`` restates the same four statements in order on top of
  ``scipy.ndimage.zoom``.

Both return what the tools store into the float32 ``images`` blob: a (3, h, w) float32 array.
tests/golden/make_prep_golden.py freezes the in-place outputs in tests/golden/prep_ref.npz.

Parity status: like oracle/post_oracle.py, UNPINNED against the scipy the reference pins (0.18,
python-dependencies.txt:15); scipy is 1.18 here -- the same corner-aligned order-1 mapping (grid_mode=False).
"""
import ast
import os

import numpy as np
from scipy import ndimage as nd

TOOLS = "/root/reference/training/tools"
SCRIPTS = ("test-ms.py", "test-ms-f.py", "test-coco.py", "generate_train_gt.py")
RELATIVE = ("test-ms-f.py",)          # preprocess(image, size) takes a zoom factor there
MEAN_PIXEL = np.array([104.0, 117.0, 123.0])   # test-ms.py:48 and the other tools
_NS = {}


def available():
    return all(os.path.exists(os.path.join(TOOLS, f)) for f in SCRIPTS)


def _top_level_source(lines, first):
    """The lines of the top-level statement that starts at lines[first]: up to the next unindented line."""
    end = first + 1
    while end < len(lines) and (not lines[end].strip() or lines[end][0] in " \t"):
        end += 1
    return lines[first:end]


def _load(script):
    if script not in _NS:
        path = os.path.join(TOOLS, script)
        with open(path) as fh:
            lines = fh.read().splitlines(True)
        # the scripts are Python 2 (print statements elsewhere): only the two statements wanted are parsed, each in
        # full and at its own line numbers
        src = [""] * len(lines)
        for i, line in enumerate(lines):
            if line.startswith(("mean_pixel", "def preprocess(")):
                src[i:i + len(_top_level_source(lines, i))] = _top_level_source(lines, i)
        tree = ast.parse("".join(s if s else "\n" for s in src), path)

        def wanted(n):
            if isinstance(n, ast.FunctionDef):
                return n.name == "preprocess"
            return isinstance(n, ast.Assign) and [getattr(t, "id", None) for t in n.targets] == ["mean_pixel"]
        keep = [n for n in tree.body if wanted(n)]
        assert [type(n) for n in keep] == [ast.Assign, ast.FunctionDef], script
        ns = {"np": np, "nd": nd}
        exec(compile(ast.Module(body=keep, type_ignores=[]), path, "exec"), ns)
        _NS[script] = ns
    return _NS[script]


def reference(script, image, size):
    """The script's own preprocess(image, size), stored into a float32 blob: (3, h, w) float32."""
    out = _load(script)["preprocess"](image, size)
    out = np.asarray(out)
    return out.reshape(out.shape[-3:]).astype(np.float32)


def preprocess(image, size, relative=False, mean_pixel=MEAN_PIXEL):
    """The four statements of preprocess() in order, then the blob's float32 store: (3, h, w) float32."""
    image = np.array(image)
    if relative:
        zoom = (size, size, 1.0)                                             # test-ms-f.py:104-106
    else:
        zoom = (size / float(image.shape[0]), size / float(image.shape[1]), 1.0)   # test-ms.py:72-75
    image = nd.zoom(image.astype('float32'), zoom, order=1)
    image = image[:, :, [2, 1, 0]]                                           # :77
    image = image - mean_pixel                                               # :78 (float64)
    image = image.transpose([2, 0, 1])                                       # :80
    return image.astype(np.float32)                                          # net.blobs['images'].data[...] = ...


def output_shape(H, W, size, relative=False):
    """The (h, w) scipy gives the zoom above: int(round(in * factor)) with Python's round."""
    fy, fx = (size, size) if relative else (size / float(H), size / float(W))
    return int(round(H * fy)), int(round(W * fx))


def hits_cval(H, W, h, w):
    """True when scipy's mode='constant' makes the last output row or column 0 (o * ((in-1)/(out-1)) rounds to
    just above in-1, DESIGN.md section 1.1)."""
    def axis(i, o):
        z = (i - 1) / float(o - 1) if o > 1 else 0.0
        return float(o - 1) * z > i - 1
    return axis(H, h) or axis(W, w)
