"""CPU tests of the batched network input: the header and the binding table agree on the two entry points, the
network input shapes of a mixed-size list, the launch split, and the Python wrappers' refusals before they touch the
library or a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from dsrg_b200 import _lib, postprocess

NAMES = ("dsrg_prepare_net_input_batch_dev", "dsrg_prepare_net_input_batch_host")


def _header():
    src = open(os.path.join(ROOT, "include", "dsrg_b200.h")).read()
    return re.sub(r"/\*.*?\*/", "", src, flags=re.S)


def _declaration(name):
    m = re.search(r"\bint\s+%s\s*\(([^)]*)\)\s*;" % name, _header())
    assert m, name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


@pytest.mark.parametrize("name", NAMES)
def test_header_and_signatures_agree(name):
    params = _declaration(name)
    res, args = _lib.SIGNATURES[name]
    assert res is _lib._i
    assert [_lib._vp if "*" in p else _lib._i for p in params] == args
    assert all(p.rsplit(" ", 1)[0] == "int" for p in params if "*" not in p)
    # the batch size is not the second parameter: the prologue tests of the B-first entry points do not apply
    assert args[1] is not C.c_int
    assert params[1].startswith("const uint8_t *const *")
    assert params[4] == "int B" and params[5] == "int n_scales"
    assert name.endswith("_host") or params[-1] == "void *stream"


def test_images_per_launch_matches_the_header():
    m = re.search(r"#define\s+DSRG_PREP_IMAGES_PER_LAUNCH\s+(\d+)", _header())
    assert m and int(m.group(1)) == _lib.PREP_IMAGES_PER_LAUNCH == 64


@pytest.mark.parametrize("B,launches", [(1, 1), (2, 1), (63, 1), (64, 1), (65, 2), (128, 2), (129, 3), (1000, 16)])
def test_launch_split(B, launches):
    assert postprocess.prep_launches(B) == launches
    # the images of launch j are [64 j, min(64 (j + 1), B)): every image once, none of them in two launches
    per = _lib.PREP_IMAGES_PER_LAUNCH
    spans = [range(b0, min(b0 + per, B)) for b0 in range(0, B, per)]
    assert len(spans) == launches and [i for r in spans for i in r] == list(range(B))


def test_absolute_sizes_give_one_shape_across_mixed_sizes():
    voc = [(500, 375), (375, 500), (333, 500), (500, 334), (1, 17), (481, 481)]
    assert postprocess.net_input_shapes(voc, (241, 321, 401)) == [(241, 241), (321, 321), (401, 401)]
    assert postprocess.net_input_shapes([(640, 427), (427, 640)], [481]) == [(481, 481)]
    for H in range(1, 700, 7):
        for W in (1, 333, 375, 500, 640):
            assert postprocess.net_input_size(H, W, 321) == (321, 321)


def test_relative_sizes_are_refused_across_sizes():
    assert postprocess.net_input_shapes([(334, 47)] * 3, (0.75, 1, 1.25), relative=True) == \
        [(250, 35), (334, 47), (418, 59)]
    with pytest.raises(ValueError):
        postprocess.net_input_shapes([(334, 47), (335, 47)], (0.75,), relative=True)
    with pytest.raises(ValueError):
        postprocess.net_input_shapes([(334, 47), (47, 334)], (1,), relative=True)
    for bad in (([], [321]), ([(20, 30)], []), ([(20, 30)], [0.01])):
        with pytest.raises(ValueError):
            postprocess.net_input_shapes(bad[0], bad[1], relative=True)


@pytest.mark.parametrize("image_sizes,sizes,relative", [
    ([(20, 30)], list(range(1, 18)), False),          # 17 scales: the library takes at most 16
    ([(20, 30), (0, 30)], [321], False),              # an image of no rows (size / H would divide by zero)
    ([(20, 0)], [321], False),
    ([(20, 30)], [1 << 16], True),                    # a 1310720 x 1966080 plane: 2^31 pixels and more
    ([(1 << 16, 1 << 15)], [5], False),               # an image of 2^31 pixels
])
def test_shapes_the_library_would_refuse_are_value_errors(image_sizes, sizes, relative):
    with pytest.raises(ValueError):
        postprocess.net_input_shapes(image_sizes, sizes, relative)
    assert len(postprocess.net_input_shapes([(20, 30)], list(range(1, 17)))) == 16


def test_grouping_restores_input_order():
    sizes = [(375, 500), (500, 375), (375, 500), (333, 500), (500, 375), (375, 500)]
    groups = postprocess._chunks(sizes, len(sizes))
    assert groups == [[0, 2, 5], [1, 4], [3]]
    out = [None] * len(sizes)
    for idx in groups:
        assert len({sizes[i] for i in idx}) == 1
        for i in idx:
            out[i] = sizes[i]
    assert out == sizes


def test_host_wrapper_refuses_bad_arguments_before_any_call():
    im = np.zeros((20, 30, 3), np.uint8)
    for bad in ([im.astype(np.float32)], [im[:, :, :2]], [im, im[:, :, 0]], [im.tolist()], []):
        with pytest.raises(ValueError):
            postprocess.preprocess_batch(bad, [241])
    with pytest.raises(ValueError):
        postprocess.preprocess_batch([im], [241], mean_pixel=(104.0, 117.0))
    with pytest.raises(ValueError):
        postprocess.preprocess_batch([im], [241], M=256)
    with pytest.raises(ValueError):
        postprocess.preprocess_batch([im, np.zeros((21, 30, 3), np.uint8)], [0.75], relative=True)


def test_device_wrappers_refuse_host_tensors():
    torch = pytest.importorskip("torch")
    images = torch.zeros((2, 8, 10, 3), dtype=torch.uint8)
    with pytest.raises(ValueError):
        postprocess.preprocess_batch_dev(images, [41])
    with pytest.raises(ValueError):
        postprocess.preprocess_batch_dev(list(images), [41])
    with pytest.raises(ValueError):
        postprocess.preprocess_batch_dev([], [41])
    with pytest.raises(ValueError):
        postprocess.predict_masks_dev(list(images), [torch.zeros((2, 21, 4, 5))])
    with pytest.raises(ValueError):
        postprocess.predict_masks_dev([], [torch.zeros((0, 21, 4, 5))])


def test_library_version_has_the_batched_network_input():
    assert _lib.lib().dsrg_version() >= 109
