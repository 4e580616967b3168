"""GPU parity of SEC's seeding and expansion losses (dsrg_seedloss_plain_*, dsrg_expandloss_*; pylayers.py:95-118,
:183-233) against the float64 restatements of oracle/sec_oracle.py and the reference's own classes
(tests/golden/sec_layers_ref.npz).  The device may rank tied values differently from numpy, so gradients are
compared with the values of every tie group sorted (sec_oracle.tie_canonical)."""
import importlib.util
import os

import numpy as np
import pytest

import fake_caffe
from conftest import GOLDEN, load_golden
from dsrg_b200 import _lib, api
from oracle import sec_oracle

pytestmark = pytest.mark.gpu

fake_caffe.install()
import pylayers  # noqa: E402

_spec = importlib.util.spec_from_file_location("make_sec_golden", os.path.join(GOLDEN, "make_sec_golden.py"))
make_sec_golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(make_sec_golden)


def _inputs(B, special, seed):
    """probs from the device SoftmaxLayer on random logits with saturated planes, labels (B, 1, 1, 21)."""
    rng = np.random.RandomState(seed)
    logits = (2 * rng.randn(B, 21, 41, 41)).astype(np.float32)
    logits[:, 7, :20] = 40.0      # exact-tie groups at the plane max
    logits[:, 5] = -40.0          # planes of floored values
    eng = api.Engine(B, 41, 41, 21)
    probs = eng.softmax_forward_host(logits)
    eng.close()
    probs[0, 12] = probs[0, 12].max()   # one constant plane: every element is the max
    labels = np.zeros((B, 1, 1, 21), np.float32)
    labels[:, 0, 0, 0] = 1.0
    for b in range(B):
        labels[b, 0, 0, rng.choice(np.arange(1, 21), size=rng.randint(1, 4), replace=False)] = 1.0
    labels[0, 0, 0, 12] = 0.0
    labels[0, 0, 0, 7] = 0.0
    if special and B >= 2:
        labels[1, 0, 0, 1:] = 0.0            # P = 0
        labels[B - 1, 0, 0, 1:] = 1.0        # A = 0
    return probs, labels


def _check_grad(got, want, probs):
    g, w = sec_oracle.tie_canonical(got, probs), sec_oracle.tie_canonical(want, probs)
    assert np.array_equal(np.isnan(g), np.isnan(w))
    np.testing.assert_allclose(g, w, rtol=1e-5, atol=1e-12)


@pytest.mark.parametrize("B,special", [(1, False), (5, False), (5, True), (20, False), (20, True)])
def test_expandloss_matches_the_float64_oracle(torch_cuda, B, special):
    torch = torch_cuda
    probs, labels = _inputs(B, special, 10 + B)
    eng = api.Engine(B, 41, 41, 21)
    d_p, d_l = torch.from_numpy(probs).cuda(), torch.from_numpy(labels).cuda()
    terms = torch.zeros(3, device="cuda")
    eng.expandloss_forward_dev(d_p, d_l, terms)
    t = terms.cpu().numpy().astype(np.float64)
    want = sec_oracle.expand_loss_terms(probs, labels)
    for got_k, want_k in zip(-t / B, want):
        assert np.isnan(got_k) == np.isnan(want_k)
        if not np.isnan(want_k):
            assert abs(got_k - want_k) <= 1e-6 * abs(want_k), (got_k, want_k)
    loss, want_loss = float(-t.sum() / B), sec_oracle.expand_loss(probs, labels)
    assert np.isnan(loss) == np.isnan(want_loss) and (np.isnan(loss) or abs(loss - want_loss) <= 1e-6 * abs(want_loss))
    grad = torch.empty_like(d_p)
    eng.expandloss_backward_dev(d_p, d_l, grad)
    g = grad.cpu().numpy()
    wg = sec_oracle.expand_loss_grad(probs, labels)
    _check_grad(g, wg, probs)
    untied = np.ones(probs.shape, bool)
    for b in range(B):
        for k in range(21):
            _, inv, cnt = np.unique(probs[b, k], return_inverse=True, return_counts=True)
            untied[b, k] = (cnt[inv] == 1).reshape(41, 41)
    ok = untied & ~np.isnan(wg)
    np.testing.assert_allclose(g[ok], wg[ok], rtol=1e-5, atol=1e-12)
    # image 0, class 12 is absent and constant: every element is the max and carries the full max term, which is
    # all its gradient (the rank term of an absent class is 0)
    cm = (1.0 / B) / (20 - (labels[0, 0, 0, 1:] > 0.5).sum()) / (1.0 - np.float64(probs[0, 12].max()))
    np.testing.assert_allclose(g[0, 12], cm, rtol=1e-5)
    # class 7 of image 0 (absent) ties at its max over the saturated rows: each of those elements gets cm7 in full
    m7 = probs[0, 7] == probs[0, 7].max()
    assert m7.sum() > 1
    cm7 = (1.0 / B) / (20 - (labels[0, 0, 0, 1:] > 0.5).sum()) / (1.0 - np.float64(probs[0, 7].max()))
    np.testing.assert_allclose(g[0, 7][m7], cm7, rtol=1e-5)
    if special and B >= 2:
        assert np.isnan(g[1, 1:]).all() and np.isnan(g[B - 1, 1:]).all() and not np.isnan(g[:, 0]).any()
    eng.close()


def test_expandloss_generic_shape_and_q(torch_cuda):
    torch = torch_cuda
    B, M, H, W, q = 3, 81, 33, 57, (0.99, 0.9995)
    rng = np.random.RandomState(4)
    x = rng.randn(B, M, H, W) * 2
    e = np.exp(x - x.max(1, keepdims=True))
    probs = ((e / e.sum(1, keepdims=True)) + 1e-4).astype(np.float32)
    labels = (rng.rand(B, 1, 1, M) < 0.1).astype(np.float32)
    labels[:, 0, 0, 1] = 1.0
    eng = api.Engine(B, H, W, M)
    d_p, d_l = torch.from_numpy(probs).cuda(), torch.from_numpy(labels).cuda()
    terms = torch.zeros(3, device="cuda")
    eng.expandloss_forward_dev(d_p, d_l, terms, q_fg=q[0], q_bg=q[1])
    loss, want = -float(terms.sum().item()) / B, sec_oracle.expand_loss(probs, labels, *q)
    assert abs(loss - want) <= 1e-6 * abs(want)
    grad = torch.empty_like(d_p)
    eng.expandloss_backward_dev(d_p, d_l, grad, q_fg=q[0], q_bg=q[1])
    _check_grad(grad.cpu().numpy(), sec_oracle.expand_loss_grad(probs, labels, *q), probs)
    eng.close()


def test_expandloss_refuses_planes_above_the_limit(torch_cuda):
    eng = api.Engine(1, 91, 91, 21)      # 8281 > DSRG_GWRP_MAX_PLANE
    probs = np.full((1, 21, 91, 91), 1.0 / 21, np.float32)
    labels = np.ones((1, 1, 1, 21), np.float32)
    with pytest.raises(_lib.DsrgError) as ei:
        eng.expandloss_forward_host(probs, labels)
    assert ei.value.code == _lib.E_INVALID and "8192" in str(ei.value)
    with pytest.raises(_lib.DsrgError):
        eng.expandloss_backward_host(probs, labels)
    eng.close()
    eng = api.Engine(1, 128, 64, 3)      # exactly at the limit
    rng = np.random.RandomState(1)
    p = rng.uniform(0.01, 0.99, (1, 3, 128, 64)).astype(np.float32)
    lab = np.array([1, 1, 0], np.float32).reshape(1, 1, 1, 3)
    lab0 = np.array([1, 0, 0], np.float32).reshape(1, 1, 1, 3)     # P = 0: NaN
    for lb in (lab, lab0):
        t = eng.expandloss_forward_host(p, lb)
        want = sec_oracle.expand_loss_terms(p, lb)
        for a, w in zip(-t.astype(np.float64), want):
            assert np.isnan(a) == np.isnan(w) and (np.isnan(w) or abs(a - w) <= 1e-6 * abs(w))
        _check_grad(eng.expandloss_backward_host(p, lb), sec_oracle.expand_loss_grad(p, lb), p)
    eng.close()


def test_sec_losses_dev_host_and_repeat_are_bit_identical(torch_cuda):
    torch = torch_cuda
    B = 20
    probs, labels = _inputs(B, True, 77)
    seeds = (np.random.RandomState(2).rand(*probs.shape) < 0.05).astype(np.float32)
    eng = api.Engine(B, 41, 41, 21)
    d_p, d_l, d_s = (torch.from_numpy(a).cuda() for a in (probs, labels, seeds))
    outs = []
    for _ in range(2):
        terms, grad = torch.zeros(3, device="cuda"), torch.empty_like(d_p)
        eng.expandloss_forward_dev(d_p, d_l, terms)
        eng.expandloss_backward_dev(d_p, d_l, grad)
        st, sg = torch.zeros(1, device="cuda"), torch.empty_like(d_p)
        eng.seedloss_plain_forward_dev(d_p, d_s, st)
        eng.seedloss_plain_backward_dev(d_p, d_s, sg)
        outs.append([a.cpu().numpy() for a in (terms, grad, st, sg)])
    host = [eng.expandloss_forward_host(probs, labels), eng.expandloss_backward_host(probs, labels),
            eng.seedloss_plain_forward_host(probs, seeds), eng.seedloss_plain_backward_host(probs, seeds)]
    for a, b, h in zip(outs[0], outs[1], host):
        assert a.tobytes() == b.tobytes() and a.tobytes() == h.tobytes()
    eng.close()


@pytest.mark.parametrize("B,empty", [(1, False), (5, True), (20, False)])
def test_seedloss_plain_matches_the_float64_oracle(torch_cuda, B, empty):
    torch = torch_cuda
    probs, _ = _inputs(B, False, 200 + B)
    rng = np.random.RandomState(B)
    seeds = (rng.rand(*probs.shape) < 0.05).astype(np.float32)
    if empty:
        seeds[2] = 0.0
    eng = api.Engine(B, 41, 41, 21)
    d_p, d_s = torch.from_numpy(probs).cuda(), torch.from_numpy(seeds).cuda()
    terms = torch.zeros(1, device="cuda")
    eng.seedloss_plain_forward_dev(d_p, d_s, terms)
    loss, want = -float(terms.item()) / B, sec_oracle.seed_loss(probs, seeds)
    assert np.isnan(loss) == np.isnan(want) == empty
    if not empty:
        assert abs(loss - want) <= 1e-6 * abs(want)
    grad = torch.empty_like(d_p)
    eng.seedloss_plain_backward_dev(d_p, d_s, grad)
    g, wg = grad.cpu().numpy(), sec_oracle.seed_loss_grad(probs, seeds)
    assert np.array_equal(np.isnan(g), np.isnan(wg))
    np.testing.assert_allclose(g, wg, rtol=1e-5, atol=1e-12)
    eng.close()


def test_dropin_sec_layers_match_the_reference_golden(torch_cuda):
    g = load_golden("sec_layers_ref.npz")
    for name in make_sec_golden.SEED_CASES:
        probs, lab = make_sec_golden.seed_inputs(name)
        layer, bottom, top = fake_caffe.run_layer(pylayers.SeedLossLayer, [probs, lab])
        want = float(g[name + "_float64_loss"])
        assert top[0].data.shape == (1,)
        got = float(top[0].data[0])
        assert np.isnan(got) == np.isnan(want) and (np.isnan(want) or abs(got - want) <= 1e-6 * abs(want))
        top[0].diff[...] = 7.0                     # ignored, like the reference
        layer.backward(top, [True, False], bottom)
        wg = g[name + "_float64_grad"]
        assert np.array_equal(np.isnan(bottom[0].diff), np.isnan(wg))
        np.testing.assert_allclose(bottom[0].diff, wg, rtol=1e-5, atol=1e-12)
    for name in make_sec_golden.EXPAND_CASES:
        probs, labels = make_sec_golden.expand_inputs(name)
        layer, bottom, top = fake_caffe.run_layer(pylayers.ExpandLossLayer, [probs, labels])
        want = float(g[name + "_float64_loss"])
        got = float(top[0].data[0])
        assert np.isnan(got) == np.isnan(want) and (np.isnan(want) or abs(got - want) <= 1e-6 * abs(want))
        layer.backward(top, [True, False], bottom)
        _check_grad(bottom[0].diff, g[name + "_float64_grad"], probs)
