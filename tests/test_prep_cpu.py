"""CPU tests of the evaluation tools' network input (preprocess(image, size), training/tools/test-ms.py:68-81 and its
siblings): the numpy restatement in oracle/prep_oracle.py against the reference's own preprocess functions -- run
in place when the reference is mounted, frozen in tests/golden/prep_ref.npz -- and the output shapes, which the
library computes on the host exactly as scipy does."""
import importlib.util
import os

import numpy as np
import pytest

from conftest import GOLDEN, load_golden
from dsrg_b200 import postprocess
from oracle import prep_oracle

_spec = importlib.util.spec_from_file_location("make_prep_golden", os.path.join(GOLDEN, "make_prep_golden.py"))
make_prep_golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(make_prep_golden)
CASES = make_prep_golden.CASES


def frozen_matches(g, key, got):
    assert tuple(g["shape_" + key]) == got.shape, key
    if "full_" + key in g:
        return np.array_equal(g["full_" + key], got)
    return str(g["sha_" + key]) == make_prep_golden.digest(got)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_restatement_equals_frozen_reference(case):
    name, H, W, sizes, relative, _, seed = case
    g = load_golden("prep_ref.npz")
    im = make_prep_golden.case_image(H, W, seed)
    for k, size in enumerate(sizes):
        assert frozen_matches(g, "%s_%d" % (name, k), prep_oracle.preprocess(im, size, relative)), (name, size)


@pytest.mark.parametrize("case", CASES[:7], ids=[c[0] for c in CASES[:7]])
def test_restatement_equals_reference_live(case):
    """Every script of the same kind (absolute sizes or zoom factors) gives the same array, and so does ours."""
    if not prep_oracle.available():
        pytest.skip("reference not mounted")
    name, H, W, sizes, relative, _, seed = case
    im = make_prep_golden.case_image(H, W, seed)
    scripts = [s for s in prep_oracle.SCRIPTS if (s in prep_oracle.RELATIVE) == relative]
    assert scripts
    for size in sizes:
        want = prep_oracle.preprocess(im, size, relative)
        for script in scripts:
            assert np.array_equal(prep_oracle.reference(script, im, size), want), (name, script, size)


def test_golden_file_is_small_and_covers_scipys_zero_column():
    assert os.path.getsize(os.path.join(GOLDEN, "prep_ref.npz")) < 1 << 20
    g = load_golden("prep_ref.npz")
    assert prep_oracle.hits_cval(40, 51, 45, 45)
    out = g["full_cval_0"]
    # the last column is scipy's cval: 0 - mean_pixel of the channel
    assert np.array_equal(out[:, :, -1], np.broadcast_to(-prep_oracle.MEAN_PIXEL[:, None], (3, 45)).astype(np.float32))


@pytest.mark.parametrize("H,W,size,relative,want", [
    (334, 47, 1.25, True, (418, 59)),      # 417.5: Python's round goes to the even neighbour
    (334, 47, 0.75, True, (250, 35)),      # 250.5 -> 250, 35.25 -> 35
    (37, 53, 0.75, True, (28, 40)),
    (375, 500, 321, False, (321, 321)),
    (500, 334, 401, False, (401, 401)),
    (1, 17, 5, False, (5, 5)),
    (7, 9, 1, True, (7, 9)),
])
def test_output_shapes_follow_scipy(H, W, size, relative, want):
    assert postprocess.net_input_size(H, W, size, relative) == want
    assert prep_oracle.output_shape(H, W, size, relative) == want
    im = np.zeros((H, W, 3), np.uint8)
    assert prep_oracle.preprocess(im, size, relative).shape == (3,) + want


def test_preprocess_refuses_what_the_tools_never_pass():
    """JPEGs are read as uint8 (H, W, 3): float images, other shapes and means that are not 3 values are refused
    before anything reaches the device."""
    im = np.zeros((20, 30, 3), np.uint8)
    for bad in (im.astype(np.float32), im[:, :, :2], im[:, :, 0], im.tolist()):
        with pytest.raises(ValueError):
            postprocess.preprocess(bad, [241])
    with pytest.raises(ValueError):
        postprocess.preprocess(im, [241], mean_pixel=(104.0, 117.0))
    with pytest.raises(ValueError):
        postprocess.preprocess(im, [0.01], relative=True)   # rounds to no rows
    with pytest.raises(ValueError):
        postprocess.preprocess(im, [])
