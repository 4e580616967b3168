"""CPU tests of ImageSegDataLayer (pylayers/pylayers/layer.py), the stage-2 training input: the numpy restatement in
oracle/seg_data_oracle.py against the reference's own classes -- run in place when the reference and cv2 are
present, frozen in tests/golden/seg_data_ref.npz -- its padding against cv2.copyMakeBorder, and the drop-in's setup
surface and host-side draws, which need no device."""
import importlib.util
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import fake_caffe
from conftest import GOLDEN, ROOT, load_golden
from oracle import ref_seg_layer, seg_data_oracle

fake_caffe.install()
from pylayers import layer as seg_layer  # noqa: E402

_spec = importlib.util.spec_from_file_location("make_seg_data_golden", os.path.join(GOLDEN, "make_seg_data_golden.py"))
make_golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(make_golden)
CASES = make_golden.CASES
IDS = [c[0] for c in CASES]


def restated(case):
    """The restatement's outputs of a case, seeded like the golden run: (top0, top1, _cur, order), the last three
    None for the image-only kinds."""
    name, kind, sizes, label_sizes, B, params, seed = case
    files, indexlist, root = make_golden.case_files(case)
    original = [list(e) for e in indexlist]
    random.seed(seed)
    np.random.seed(seed)
    if kind == "layer":
        t0, t1, cur = seg_data_oracle.seg_data_forward(lambda p, f: np.array(files[p]), indexlist, 0, root, B, params)
        return t0, t1, cur, make_golden.order_of(indexlist, original)
    images = [files[root + im] for im, _ in indexlist]
    if kind == "preprocess":
        out = [seg_data_oracle.preprocess(im, None, params) for im in images]
    else:
        out = [seg_data_oracle.pre_test_image(im, params) for im in images]
    return np.stack(out), None, None, None


def matches_key(g, key, a):
    assert tuple(g["shape" + key]) == a.shape, key
    if "full" + key in g:
        assert np.array_equal(g["full" + key], a), key
    else:
        assert str(g["sha" + key]) == make_golden.digest(a), key


def matches_golden(g, name, t0, t1=None, cur=None, order=None):
    matches_key(g, "0_" + name, t0)
    if "shape1_" + name in g:
        matches_key(g, "1_" + name, t1)
        assert int(g["cur_" + name]) == cur and np.array_equal(g["order_" + name], order), name


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_restatement_equals_frozen_reference(case):
    matches_golden(load_golden("seg_data_ref.npz"), case[0], *restated(case))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_restatement_equals_reference_live(case):
    if not ref_seg_layer.available():
        pytest.skip("reference or cv2 not available")
    want = make_golden.run_reference(case)
    states = random.getstate(), np.random.get_state()
    got = restated(case)
    assert random.getstate() == states[0]
    assert all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), states[1]))
    for w, g in zip(want, got):
        if w is None:
            assert g is None
        else:
            assert np.shape(w) == np.shape(g) and np.array_equal(w, g), case[0]


def test_cases_cover_the_corners():
    """Padding on one axis and on both, an image larger than its label, a window drawn in a larger label in Train
    and centred with odd differences in Test, mirror on and off, an epoch wrap, the ignore_label values 255, 300, -5
    and 254.5, scale 0.017 with the int default mean, both image-only paths, H or W of 1 and a batch of 18."""
    g = load_golden("seg_data_ref.npz")
    layer_cases = [c for c in CASES if c[1] == "layer"]
    crop = lambda c: c[5]["crop_size"]  # noqa: E731
    labels = lambda c: c[3] or c[2]  # noqa: E731
    assert any(all(h < crop(c)[0] and w >= crop(c)[1] for h, w in labels(c)) for c in layer_cases)
    assert any(any(h < crop(c)[0] and w < crop(c)[1] for h, w in labels(c)) for c in layer_cases)
    assert any(c[3] and any(a[0] > b[0] or a[1] > b[1] for a, b in zip(c[2], c[3])) for c in layer_cases)
    assert any(c[5].get("phase", "Train") == "Train" and all(h > crop(c)[0] for h, w in labels(c))
               for c in layer_cases)
    assert any(c[5].get("phase") == "Test" and all((h - crop(c)[0]) % 2 or (w - crop(c)[1]) % 2 for h, w in labels(c))
               for c in layer_cases)
    assert {bool(c[5].get("mirror")) for c in layer_cases} == {False, True}
    assert not np.array_equal(g["order_wrap"], np.arange(3)) and int(g["cur_wrap"]) == 2
    assert {c[5].get("ignore_label", 255) for c in layer_cases} == {255, 300, -5, 254.5}
    assert any(c[5].get("scale") == 0.017 and "mean" not in c[5] for c in layer_cases)
    assert {c[1] for c in CASES} == {"layer", "preprocess", "pre_test"}
    assert any(1 in s for c in CASES for s in c[2])
    assert max(c[4] for c in CASES) > 16
    for name in ("ignore300", "ignore_m5", "ignore_half"):
        assert {255.0, 0.0, 254.0} & set(np.unique(g["full1_" + name]))   # the pad byte is in the label top


@pytest.mark.parametrize("ignore_label", [255, 300, -5, 254.5, 253.5, 0.5, 1.5, 0, 17])
def test_padding_matches_cv2(ignore_label):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.RandomState(3)
    label = rng.randint(0, 256, (7, 5)).astype(np.uint8)
    image = (rng.rand(7, 5, 3) * 200 - 100).astype(np.float32)
    for ph, pw in ((3, 0), (0, 4), (2, 6)):
        want = cv2.copyMakeBorder(label, 0, ph, 0, pw, cv2.BORDER_CONSTANT, value=(ignore_label,))
        got = seg_data_oracle.pad_bottom_right(label, ph, pw, seg_data_oracle.pad_byte(ignore_label))
        assert got.dtype == want.dtype and np.array_equal(got, want), (ignore_label, ph, pw)
        want = cv2.copyMakeBorder(image, 0, ph, 0, pw, cv2.BORDER_CONSTANT, value=(0.0, 0.0, 0.0))
        assert np.array_equal(seg_data_oracle.pad_bottom_right(image, ph, pw, 0.0), want)
    assert seg_layer._pad_byte(ignore_label) == seg_data_oracle.pad_byte(ignore_label)


def test_pad_byte_saturates_and_rounds_half_to_even():
    assert [seg_layer._pad_byte(v) for v in (300, -5, 254.5, 253.5, 255, 0.5, 1.5)] == [255, 0, 254, 254, 255, 0, 2]


def _setup(tmp_path, params, lines="a.jpg a.png\nb.jpg b.png\n"):
    src = tmp_path / "train.txt"
    src.write_text(lines)
    layer = seg_layer.ImageSegDataLayer()
    layer.param_str = params.replace("SRC", str(src))
    top = [fake_caffe.Blob() for _ in range(2)]
    layer.setup([], top)
    return layer, top, str(src)


def test_layer_setup_surface(tmp_path, capsys):
    """train-f.prototxt's param_str: the defaults are filled in, the reference's two lines are printed, and the
    tops are shaped once."""
    layer, top, src = _setup(tmp_path, "{'batch_size': 10, 'root_folder': '/voc/', 'mean': (104.0, 117.0, 123.0), "
                                       "'source': 'SRC', 'mirror': True, 'crop_size': (321, 321)}")
    assert capsys.readouterr().out.splitlines() == [
        "BatchLoader initialized with 2 images",
        "ImageSegDataLayer initialized for split: %s, with bs: 10, im_shape: (321, 321)." % src]
    assert [t.data.shape for t in top] == [(10, 3, 321, 321), (10, 1, 321, 321)]
    assert all(t.data.dtype == np.float32 for t in top)
    assert layer.top_names == ["data", "label"] and layer.batch_size == 10 and layer.input_shape == (321, 321)
    bl = layer.batch_loader
    assert bl.indexlist == [["a.jpg", "a.png"], ["b.jpg", "b.png"]] and bl._cur == 0
    assert bl.root_folder == "/voc/" and bl.source == src and bl.batch_size == 10
    t = bl.transformer
    assert (t.mean, t.is_mirror, t.crop_h, t.crop_w, t.scale, t.phase, t.ignore_label) == (
        (104.0, 117.0, 123.0), True, 321, 321, 1.0, "Train", 255)
    layer.reshape([], top)
    layer.backward(top, [], [])
    layer, top, _ = _setup(tmp_path, "{'batch_size': 1, 'root_folder': '', 'source': 'SRC'}", "x y\n")
    assert [t.data.shape for t in top] == [(1, 3, 505, 505), (1, 1, 505, 505)]
    t = layer.batch_loader.transformer
    assert (t.mean, t.is_mirror, t.scale, t.phase, t.ignore_label) == ([128, 128, 128], False, 1.0, "Train", 255)


def test_check_params_fills_the_callers_dict():
    p = {"mean": (1.0, 2.0, 3.0), "phase": "Test"}
    seg_layer.SimpleTransformer.check_params(p)
    assert p == {"mean": (1.0, 2.0, 3.0), "phase": "Test", "crop_size": (505, 505), "scale": 1.0, "mirror": False,
                 "ignore_label": 255}
    q = {}
    seg_layer.SimpleTransformer.check_params(q)
    q["mean"].append(4)   # a list of its own per call
    r = {}
    seg_layer.SimpleTransformer.check_params(r)
    assert r["mean"] == [128, 128, 128]
    t = seg_layer.SimpleTransformer({"crop_size": (5, 7)})
    t.set_scale(0.5)
    t.set_mean((1, 2, 3))
    assert (t.scale, t.mean, t.crop_h, t.crop_w) == (0.5, (1, 2, 3), 5, 7)
    with pytest.raises(ValueError):
        t.set_mean(7.0)


@pytest.mark.parametrize("mean", ["104.0", "(104.0, 117.0)", "[[1, 2, 3]]", "(1, 2, 3, 4)"])
def test_layer_refuses_a_mean_that_is_not_three_values(tmp_path, mean):
    with pytest.raises(ValueError):
        _setup(tmp_path, "{'batch_size': 1, 'root_folder': '', 'source': 'SRC', 'mean': %s}" % mean)


def test_layer_parses_literals_only(tmp_path):
    with pytest.raises(ValueError):
        _setup(tmp_path, "{'batch_size': __import__('os').getpid(), 'root_folder': '', 'source': 'SRC'}")


def test_layer_requires_the_reference_keys(tmp_path):
    for missing in ("batch_size", "root_folder", "source"):
        params = {"batch_size": 2, "root_folder": "", "source": "SRC"}
        del params[missing]
        with pytest.raises(KeyError, match=missing):
            _setup(tmp_path, repr(params))


@pytest.mark.parametrize("phase,mirror", [("Train", True), ("Train", False), ("Test", True), ("Val", False)])
def test_draws_follow_the_restatement(phase, mirror):
    """The drop-in's crop windows and mirror flags, and what they leave of both random states."""
    t = seg_layer.SimpleTransformer({"crop_size": (21, 17), "phase": phase, "mirror": mirror})
    shapes = [(30, 40), (21, 17), (5, 50), (60, 3), (22, 18), (1, 1)]
    for seed in range(3):
        random.seed(seed)
        np.random.seed(seed)
        want = [seg_data_oracle.draw(s, (21, 17), phase, mirror) for s in shapes]
        states = random.getstate(), np.random.get_state()
        random.seed(seed)
        np.random.seed(seed)
        got = [t._draw(s, s) for s in shapes]
        assert got == want
        assert random.getstate() == states[0]
        assert all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), states[1]))


def test_window_that_leaves_the_image_raises_numpys_error_after_the_draws():
    """An image shorter than its label: the reference's slice comes back short and the store into the top fails."""
    t = seg_layer.SimpleTransformer({"crop_size": (321, 321), "mirror": True})
    im = np.zeros((200, 400, 3), np.uint8)
    lab = np.zeros((400, 400), np.uint8)
    random.seed(5)
    np.random.seed(5)
    with pytest.raises(ValueError) as want:
        seg_data_oracle.seg_data_forward(lambda p, f: im if f else lab, [["a", "b"]], 0, "", 1,
                                         {"crop_size": (321, 321), "mirror": True})
    states = random.getstate(), np.random.get_state()
    assert "could not broadcast input array from shape (3," in str(want.value)
    random.seed(5)
    np.random.seed(5)
    with pytest.raises(ValueError) as got:
        t._draw(im.shape, lab.shape)
    assert str(got.value) == str(want.value)
    assert random.getstate() == states[0]
    assert all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), states[1]))
    # one row left: numpy would broadcast it over the window; the drop-in refuses
    t = seg_layer.SimpleTransformer({"crop_size": (4, 4), "phase": "Test"})
    with pytest.raises(ValueError, match="not supported"):
        t._draw((5, 4), (12, 4))


def test_import_loads_no_image_library():
    code = ("import sys; from dsrg_b200.dropin import caffe_shim; caffe_shim.install(); import pylayers.layer; "
            "bad = [m for m in ('cv2', 'PIL', 'skimage', 'scipy.misc') if m in sys.modules]; "
            "assert not bad, bad; print('ok')")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], cwd=ROOT, capture_output=True, text=True,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr
