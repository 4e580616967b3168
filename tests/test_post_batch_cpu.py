"""CPU tests of the batched inference post-processing: the header and the binding table agree on the two entry
points, the host-side grouping keeps the input order, and the Python wrappers refuse bad arguments before they
touch the library or a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from dsrg_b200 import _lib, postprocess

NAMES = ("dsrg_predict_mask_batch_dev", "dsrg_predict_mask_batch_host")


def _declaration(name):
    src = open(os.path.join(ROOT, "include", "dsrg_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    m = re.search(r"\bint\s+%s\s*\(([^)]*)\)\s*;" % name, src)
    assert m, name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


def _ctype(param):
    if "*" in param:
        return "dsrg_crf_params" in param and _lib._pp or _lib._vp
    kind = param.rsplit(" ", 1)[0]
    return {"int": _lib._i, "float": _lib._f}[kind]


@pytest.mark.parametrize("name", NAMES)
def test_header_and_signatures_agree(name):
    params = _declaration(name)
    res, args = _lib.SIGNATURES[name]
    assert res is _lib._i
    assert [_ctype(p) for p in params] == args
    # the batch size is not the second parameter: the prologue tests of the B-first entry points do not apply
    assert args[1] is not C.c_int
    assert params[5].endswith(" B")
    assert name.endswith("_host") or params[-1] == "void *stream"


def test_chunks_group_by_key_in_input_order():
    keys = ["a", "b", "a", "c", "a", "b", "a", "a"]
    got = postprocess._chunks(keys, 2)
    assert got == [[0, 2], [4, 6], [7], [1, 5], [3]]
    assert sorted(i for c in got for i in c) == list(range(len(keys)))
    for c in postprocess._chunks(keys, 1):
        assert len(c) == 1
    assert postprocess._chunks(keys, 100) == [[0, 2, 4, 6, 7], [1, 5], [3]]


def test_host_wrappers_refuse_bad_arguments_before_any_call():
    im = np.zeros((8, 10, 3), np.uint8)
    blob = np.zeros((21, 4, 5), np.float32)
    with pytest.raises(ValueError):
        postprocess.predict_masks_ms([im, im], [[blob]])              # one set of blobs per image
    with pytest.raises(ValueError):
        postprocess.predict_masks_ms([im], [[blob]], batch=0)
    with pytest.raises(ValueError):
        postprocess.predict_masks_ms([im[:, :, :2]], [[blob]])        # not (H, W, 3)
    with pytest.raises(ValueError):
        postprocess.predict_masks_ms([im], [[blob, np.zeros((20, 4, 5), np.float32)]])   # label counts differ
    with pytest.raises(ValueError):
        postprocess.predict_masks_ms([im], [[]])
    with pytest.raises(ValueError):
        postprocess.predict_masks_gt([im], [blob], [[3, 21]])          # label id outside [0, 21)
    with pytest.raises(ValueError):
        postprocess.predict_masks_gt([im], [blob], [[-2]])
    with pytest.raises(ValueError):
        postprocess.predict_masks_gt([im, im], [blob, blob], [[3]])    # one tag list per image


def test_device_wrapper_refuses_host_tensors():
    torch = pytest.importorskip("torch")
    images = torch.zeros((2, 8, 10, 3), dtype=torch.uint8)
    scores = [torch.zeros((2, 21, 4, 5))]
    with pytest.raises(ValueError):
        postprocess.predict_mask_batch_dev(images, scores)
    with pytest.raises(ValueError):
        postprocess.predict_mask_batch_dev(images, scores, mode="other")


def test_library_version_has_the_batched_pass():
    assert _lib.lib().dsrg_version() >= 108
