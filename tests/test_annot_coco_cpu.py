"""CPU tests of AnnotationLayerCOCO (pylayers.py:389-512), the COCO training input: the numpy restatement in
oracle/annot_coco_oracle.py against the reference's own class -- run in place when the reference is mounted, frozen in
tests/golden/annot_coco_ref.npz -- and the drop-in layer's setup / reshape surface, which needs no device."""
import importlib.util
import os

import numpy as np
import pytest

import fake_caffe
from conftest import GOLDEN, load_golden
from oracle import annot_coco_oracle, prep_oracle, ref_coco_layer

fake_caffe.install()
import pylayers  # noqa: E402

_spec = importlib.util.spec_from_file_location("make_annot_coco_golden",
                                               os.path.join(GOLDEN, "make_annot_coco_golden.py"))
make_golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(make_golden)
CASES = make_golden.CASES
IDS = [c[0] for c in CASES]


def restated(case):
    name, sizes, shapes, B, new_size, mirror, ignore, seed = case
    files, indexlist, root = make_golden.case_files(case)
    original = [list(e) for e in indexlist]
    np.random.seed(seed)
    t0, t1, t2, cur = annot_coco_oracle.annotation_coco_forward(lambda p, f: np.array(files[p]), indexlist, 0,
                                                                root, B, make_golden.MEAN, new_size, mirror,
                                                                ignore)
    return t0, t1, t2, cur, make_golden.order_of(indexlist, original)


def matches_golden(g, name, t0, t1, t2, cur, order):
    assert np.array_equal(g["labels_" + name], t0), name
    assert np.array_equal(g["cues_" + name], t1), name
    assert tuple(g["shape_" + name]) == t2.shape, name
    if "full_" + name in g:
        assert np.array_equal(g["full_" + name], t2), name
    else:
        assert str(g["sha_" + name]) == make_golden.digest(t2), name
    assert int(g["cur_" + name]) == cur and np.array_equal(g["order_" + name], order), name


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_restatement_equals_frozen_reference(case):
    matches_golden(load_golden("annot_coco_ref.npz"), case[0], *restated(case))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_restatement_equals_reference_live(case):
    if not ref_coco_layer.available():
        pytest.skip("reference not mounted")
    name, sizes, shapes, B, new_size, mirror, ignore, seed = case
    files, indexlist, root = make_golden.case_files(case)
    np.random.seed(seed)
    want = ref_coco_layer.annotation_coco_layer_forward(files, indexlist, 0, root, B, make_golden.MEAN, new_size,
                                                        mirror, ignore)
    got = restated(case)
    for a, b in zip(want[:3], got[:3]):
        assert a.shape == b.shape and np.array_equal(a, b), name
    assert want[3] == got[3]


def test_cases_cover_the_corners():
    """Epoch wraps with a shuffle, mirrored and unmirrored images, ignore pixels, a non-default ignore_label,
    scipy's zero column, broadcast label maps and a batch above 16 images."""
    g = load_golden("annot_coco_ref.npz")
    assert not np.array_equal(g["order_wrap"], np.arange(3)) and not np.array_equal(g["order_batch18"], np.arange(5))
    assert max(c[3] for c in CASES) > 16
    assert {c[5] for c in CASES} == {False, True} and {c[6] for c in CASES} == {7, 255}
    assert prep_oracle.hits_cval(40, 51, 45, 45)
    for case in CASES:
        files, _, _ = make_golden.case_files(case)
        labels = [a for p, a in files.items() if p.endswith(".png")]
        assert any((lab == case[6]).any() for lab in labels), case[0]


def test_out_of_range_label_raises_numpys_index_error():
    label = np.zeros((3, 3), np.uint8)
    label[1, 2] = 90
    with pytest.raises(IndexError, match="^index 90 is out of bounds for axis 0 with size 81$"):
        annot_coco_oracle.coco_preprocess(np.zeros((5, 5, 3), np.uint8), label, (17, 17), make_golden.MEAN, 1)
    label[1, 2] = 255   # ignored
    _, cues, tags = annot_coco_oracle.coco_preprocess(np.zeros((5, 5, 3), np.uint8), label, (17, 17),
                                                      make_golden.MEAN, 1)
    assert cues.sum() == 8 and tags.sum() == 1


def _setup(tmp_path, params, n_top=3):
    src = tmp_path / "list.txt"
    src.write_text("a.jpg a.png\nb.jpg b.png\n")
    layer = pylayers.AnnotationLayerCOCO()
    layer.param_str = params.replace("SRC", str(src))
    top = [fake_caffe.Blob() for _ in range(n_top)]
    layer.setup([], top)
    return layer, top


def test_layer_setup_and_reshape(tmp_path):
    layer, top = _setup(tmp_path, "{'source': 'SRC', 'root': '/r/', 'batch_size': 5, "
                                  "'mean': (104.008, 116.669, 122.675), 'new_size': (321, 305)}")
    assert [t.data.shape for t in top] == [(5, 1, 1, 81), (5, 81, 41, 39), (5, 3, 321, 305)]
    assert all(t.data.dtype == np.float32 for t in top)
    assert layer.is_mirror is False and layer.ignore_label == 255
    assert layer.indexlist == [["a.jpg", "a.png"], ["b.jpg", "b.png"]] and layer._cur == 0
    assert layer.root_folder == "/r/" and layer.batch_size == 5 and (layer.new_h, layer.new_w) == (321, 305)
    layer.reshape([], top)
    layer.backward(top, [], [])
    assert [t.data.shape for t in top] == [(5, 1, 1, 81), (5, 81, 41, 39), (5, 3, 321, 305)]
    layer, top = _setup(tmp_path, "{'source': 'SRC', 'root': '', 'batch_size': 1, 'mean': [1, 2, 3], "
                                  "'new_size': [8, 8], 'mirror': True, 'ignore_label': 0}")
    assert layer.is_mirror is True and layer.ignore_label == 0
    assert [t.data.shape for t in top] == [(1, 1, 1, 81), (1, 81, 2, 2), (1, 3, 8, 8)]


@pytest.mark.parametrize("missing", ["source", "root", "batch_size", "mean", "new_size"])
def test_layer_setup_requires_the_reference_keys(tmp_path, missing):
    params = {"source": "SRC", "root": "/r/", "batch_size": 2, "mean": (1.0, 2.0, 3.0), "new_size": (17, 17)}
    del params[missing]
    with pytest.raises(KeyError, match=missing):
        _setup(tmp_path, repr(params))


@pytest.mark.parametrize("mean", ["104.0", "(104.0, 117.0)", "[[1, 2, 3]]", "(1, 2, 3, 4)"])
def test_layer_refuses_a_mean_that_is_not_three_values(tmp_path, mean):
    with pytest.raises(ValueError):
        _setup(tmp_path, "{'source': 'SRC', 'root': '', 'batch_size': 1, 'mean': %s, 'new_size': (17, 17)}" % mean)


def test_layer_parses_literals_only(tmp_path):
    with pytest.raises(ValueError):
        _setup(tmp_path, "{'source': 'SRC', 'root': '', 'batch_size': __import__('os').getpid(), "
                         "'mean': (1, 2, 3), 'new_size': (17, 17)}")
