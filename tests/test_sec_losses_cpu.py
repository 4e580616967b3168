"""CPU tests of SEC's seeding and expansion losses (SeedLossLayer, ExpandLossLayer; pylayers.py:95-118, :183-233):
the numpy restatements against the reference's own class bodies (frozen in tests/golden/sec_layers_ref.npz, live
when the reference is mounted), the Theano stand-in's sort / max gradients, and the drop-in's surface.  No GPU."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import fake_caffe
from conftest import GOLDEN, load_golden
from dsrg_b200 import _lib
from helpers import digest
from oracle import sec_layers, sec_oracle

fake_caffe.install()
import pylayers  # noqa: E402

_spec = importlib.util.spec_from_file_location("make_sec_golden", os.path.join(GOLDEN, "make_sec_golden.py"))
make_sec_golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(make_sec_golden)

TIGHT = dict(rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("name", sorted(make_sec_golden.SEED_CASES))
def test_seed_loss_restatement_matches_reference_golden(name):
    g = load_golden("sec_layers_ref.npz")
    probs, lab = make_sec_golden.seed_inputs(name)
    assert digest(probs, lab) == str(g[name + "_sha256"]), "input generator drifted"
    np.testing.assert_allclose(sec_oracle.seed_loss(probs, lab), g[name + "_float64_loss"], **TIGHT)
    np.testing.assert_allclose(sec_oracle.seed_loss_grad(probs, lab), g[name + "_float64_grad"], **TIGHT)
    np.testing.assert_allclose(g[name + "_float32_grad"], g[name + "_float64_grad"], rtol=2e-5, atol=1e-7)
    assert np.isnan(g[name + "_float64_loss"]) == make_sec_golden.SEED_CASES[name][4]   # no seeds: NaN, no floor


@pytest.mark.parametrize("name", sorted(make_sec_golden.EXPAND_CASES))
def test_expand_loss_restatement_matches_reference_golden(name):
    g = load_golden("sec_layers_ref.npz")
    probs, labels = make_sec_golden.expand_inputs(name)
    assert digest(probs, labels) == str(g[name + "_sha256"]), "input generator drifted"
    np.testing.assert_allclose(sec_oracle.expand_loss(probs, labels), g[name + "_float64_loss"], **TIGHT)
    want = sec_oracle.tie_canonical(g[name + "_float64_grad"], probs)
    got = sec_oracle.tie_canonical(sec_oracle.expand_loss_grad(probs, labels), probs)
    np.testing.assert_allclose(got, want, **TIGHT)     # NaN exactly where the reference's is (equal_nan)
    f32 = sec_oracle.tie_canonical(g[name + "_float32_grad"], probs)
    np.testing.assert_allclose(f32, want, rtol=2e-5, atol=1e-9)
    if name == "e0":   # image 1 has no present, image 2 no absent foreground class: their fg gradient is all NaN
        G = g[name + "_float64_grad"]
        assert np.isnan(G[1:, 1:]).all() and not np.isnan(G[0]).any() and not np.isnan(G[:, 0]).any()


@pytest.mark.skipif(not sec_layers.available(), reason="the reference is not mounted")
def test_reference_classes_in_place_match_the_golden():
    g = load_golden("sec_layers_ref.npz")
    for name in make_sec_golden.SEED_CASES:
        loss, grad = sec_layers.seed_loss_layer(*make_sec_golden.seed_inputs(name))
        np.testing.assert_allclose(loss, g[name + "_float64_loss"], **TIGHT)
        np.testing.assert_allclose(grad, g[name + "_float64_grad"], **TIGHT)
    for name in make_sec_golden.EXPAND_CASES:
        probs, labels = make_sec_golden.expand_inputs(name)
        loss, grad = sec_layers.expand_loss_layer(probs, labels)
        np.testing.assert_allclose(loss, g[name + "_float64_loss"], **TIGHT)
        np.testing.assert_allclose(sec_oracle.tie_canonical(grad, probs),
                                   sec_oracle.tie_canonical(g[name + "_float64_grad"], probs), **TIGHT)


def test_shim_max_gives_every_tied_maximum_the_full_gradient():
    x = torch.tensor([[1.0, 3.0, 3.0, 2.0, 3.0], [0.5, 0.25, 0.5, 0.5, 0.0]], dtype=torch.float64, requires_grad=True)
    m = sec_layers.tie_max(x, 1)
    (g,) = torch.autograd.grad((m * torch.tensor([2.0, -1.0], dtype=torch.float64)).sum(), x)
    assert g.tolist() == [[0, 2, 2, 0, 2], [-1, 0, -1, -1, 0]]
    # without ties it agrees exactly with torch.amax
    y = torch.tensor([[1.0, 4.0, 3.0]], dtype=torch.float64, requires_grad=True)
    (ga,) = torch.autograd.grad(torch.amax(y, 1).sum(), y)
    (gt,) = torch.autograd.grad(sec_layers.tie_max(y, 1).sum(), y)
    assert torch.equal(ga, gt)
    # eq(xmax, x) * g_max: a NaN max gradient reaches every element
    (gn,) = torch.autograd.grad((sec_layers.tie_max(x, 1) * torch.tensor([float("nan"), 1.0],
                                                                        dtype=torch.float64)).sum(), x)
    assert torch.isnan(gn[0]).all() and not torch.isnan(gn[1]).any()


def test_shim_sort_gradient_is_a_permutation_of_the_rank_weights():
    rng = np.random.RandomState(3)
    n, q, coef = 37, 0.9, -2.5
    w, Z = sec_oracle.gwrp_weights(q, n)
    xv = rng.rand(n)
    xv[[3, 8, 20]] = xv[5]                      # a tie group
    x = torch.tensor(xv, requires_grad=True)
    theano, T = sec_layers.install()
    p = sec_layers.Placeholder()
    G = T.sum((T.sort(p, axis=0) * theano.shared(w)) / Z)
    (g,) = torch.autograd.grad(coef * G.ev({id(p): x}), x)
    np.testing.assert_allclose(np.sort(g.numpy()), np.sort(coef * w / Z), rtol=1e-15)
    order = np.argsort(xv, kind="stable")
    untied = np.setdiff1d(np.arange(n), [3, 5, 8, 20])
    want = np.empty(n)
    want[order] = coef * w / Z
    np.testing.assert_allclose(g.numpy()[untied], want[untied], rtol=1e-15)


def test_shim_comparison_and_integer_counts_follow_theano_dtypes():
    T = sec_layers.install()[1]
    s = sec_layers.Placeholder()
    env = {id(s): torch.tensor([[0.2, 0.7, 0.9]], dtype=torch.float32)}
    mask = s > 0.5
    assert mask.ev(env).dtype == torch.int8
    assert (1 - mask).ev(env).tolist() == [[1, 0, 0]]
    cnt = T.sum(mask, axis=1, keepdims=True)
    assert cnt.ev(env).dtype == torch.int64
    assert (T.log(s) / cnt).ev(env).dtype == torch.float64      # float32 / int64 upcasts like Theano


def _num_grad(f, x, idx, eps):
    xp, xm = x.copy(), x.copy()
    xp[idx] += eps
    xm[idx] -= eps
    return (f(xp) - f(xm)) / (2 * eps)


def test_generic_restatements_are_self_consistent():
    """M, H, W and q other than the reference's: analytic gradients == central differences (no ties)."""
    rng = np.random.RandomState(5)
    N, M, H, W = 3, 6, 5, 7
    probs = rng.uniform(0.05, 0.9, (N, M, H, W))
    labels = np.zeros((N, 1, 1, M))
    labels[:, 0, 0, 0] = 1
    labels[0, 0, 0, [1, 3]] = 1
    labels[1, 0, 0, 2] = 1
    labels[2, 0, 0, [1, 4, 5]] = 1
    q = (0.9, 0.97)
    g = sec_oracle.expand_loss_grad(probs, labels, *q)
    for idx in [(0, 0, 1, 2), (0, 1, 4, 6), (1, 3, 0, 0), (2, 2, 2, 3)] + \
            [tuple([b, k]) + np.unravel_index(np.argmax(probs[b, k]), (H, W)) for b, k in ((0, 2), (1, 5))]:
        num = _num_grad(lambda p: sec_oracle.expand_loss(p, labels, *q), probs, idx, 1e-7)
        assert abs(num - g[idx]) <= 1e-6 * max(1.0, abs(g[idx])), (idx, num, g[idx])
    seeds = (rng.rand(N, M, H, W) < 0.2).astype(np.float64)
    gs = sec_oracle.seed_loss_grad(probs, seeds)
    for idx in [(0, 0, 0, 0), (2, 5, 4, 6)] + [tuple(np.argwhere(seeds > 0)[3])]:
        num = _num_grad(lambda p: sec_oracle.seed_loss(p, seeds), probs, idx, 1e-7)
        assert abs(num - gs[idx]) <= 1e-6 * max(1.0, abs(gs[idx]))


def test_dropin_exposes_the_sec_layers_and_refuses_bad_bottoms():
    for cls in (pylayers.SeedLossLayer, pylayers.ExpandLossLayer):
        for m in ("setup", "reshape", "forward", "backward"):
            assert callable(getattr(cls, m))
        layer = cls()
        with pytest.raises(Exception):                       # "The layer needs two inputs!"
            layer.setup([fake_caffe.Blob()] * 3, [fake_caffe.Blob()])
        with pytest.raises(Exception):
            layer.setup([fake_caffe.Blob()], [fake_caffe.Blob()])
        bottom = [fake_caffe.Blob(np.zeros((2, 21, 41, 41))), fake_caffe.Blob(np.zeros((2, 1, 1, 21)))]
        top = [fake_caffe.Blob()]
        layer.setup(bottom, top)
        layer.reshape(bottom, top)
        assert top[0].data.shape == (1,)


@pytest.mark.parametrize("shape", [(2, 21, 40, 41), (2, 20, 41, 41), (2, 21, 65, 65), (1, 81, 41, 41)])
def test_expand_loss_layer_refuses_shapes_the_reference_graph_cannot_mean(shape):
    layer = pylayers.ExpandLossLayer()
    bottom = [fake_caffe.Blob(np.full(shape, 0.05)), fake_caffe.Blob(np.zeros((shape[0], 1, 1, shape[1])))]
    top = [fake_caffe.Blob()]
    layer.setup(bottom, top)
    layer.reshape(bottom, top)
    with pytest.raises(Exception, match="41"):
        layer.forward(bottom, top)
    with pytest.raises(Exception, match="41"):
        layer.backward(top, [True, False], bottom)


def test_sec_abi_symbols_are_declared_and_exported():
    names = ["dsrg_%s_%s_%s" % (k, d, s) for k in ("seedloss_plain", "expandloss")
             for d in ("forward", "backward") for s in ("dev", "host")]
    src = open(os.path.join(os.path.dirname(GOLDEN), "..", "include", "dsrg_b200.h")).read()
    L = _lib.lib()
    for n in names:
        assert n in _lib.SIGNATURES and (n + "(") in src and hasattr(L, n), n
    assert "#define DSRG_GWRP_MAX_PLANE 8192" in src
