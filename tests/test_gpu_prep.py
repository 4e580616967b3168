"""GPU tests of the evaluation tools' network input on the device (dsrg_prepare_net_input_*, postprocess.preprocess):
bit-exact against the numpy restatement of preprocess() and the frozen outputs of the reference's own functions,
one launch for every scale, the entry-point contract, and the device-resident chain preprocess -> net ->
predict_mask -> confusion matrix on one stream."""
import ctypes as C

import numpy as np
import pytest

from conftest import load_golden
from dsrg_b200 import _lib, api, pool, postprocess, synth
from oracle import prep_oracle
from test_prep_cpu import CASES, frozen_matches, make_prep_golden

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_device_equals_restatement_and_frozen_reference(torch_cuda, case):
    name, H, W, sizes, relative, _, seed = case
    g = load_golden("prep_ref.npz")
    im = make_prep_golden.case_image(H, W, seed)
    got = postprocess.preprocess(im, sizes, relative=relative)
    assert len(got) == len(sizes)
    hit = False
    for k, size in enumerate(sizes):
        want = prep_oracle.preprocess(im, size, relative)
        assert got[k].shape == (1,) + want.shape and got[k].dtype == np.float32
        assert np.array_equal(got[k][0], want), (name, size)
        assert frozen_matches(g, "%s_%d" % (name, k), got[k][0]), (name, size)
        hit |= prep_oracle.hits_cval(H, W, want.shape[1], want.shape[2])
    if name == "cval":
        assert hit      # the case really has scipy's 0 in its last column


def test_one_call_equals_single_scale_calls_and_dev_equals_host(torch_cuda):
    torch = torch_cuda
    im = synth.make_image(np.random.RandomState(5), 333, 500, "photo")
    shapes = [postprocess.net_input_size(333, 500, s) for s in (241, 321, 401)] + [(17, 900), (1, 1)]
    eng = pool.engine_for(333, 500, 21)
    eng.take_launch_count()
    many = eng.prepare_net_input_host(im, shapes)
    assert eng.take_launch_count() == 1
    for k, hw in enumerate(shapes):
        assert np.array_equal(eng.prepare_net_input_host(im, [hw])[0], many[k])
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_im = torch.from_numpy(im).cuda()
        outs = [torch.full((1, 3, h, w), float("nan"), device="cuda") for h, w in shapes]
        eng.prepare_net_input_dev(d_im, outs, stream=s.cuda_stream)
    s.synchronize()
    for k in range(len(shapes)):
        assert np.array_equal(outs[k].cpu().numpy(), many[k])
    # another mean, as a list
    other = eng.prepare_net_input_host(im, shapes[:1], mean_pixel=[1.5, -2.0, 0.0])
    want = prep_oracle.preprocess(im, 241, mean_pixel=np.array([1.5, -2.0, 0.0]))
    assert np.array_equal(other[0][0], want)


def test_engine_size_is_neither_read_nor_changed(torch_cuda):
    eng = api.Engine(1, 64, 64, 21)
    eng.set_size(20, 30)
    im = synth.make_image(np.random.RandomState(6), 375, 500, "noise")
    got = eng.prepare_net_input_host(im, [(401, 401)])
    assert np.array_equal(got[0][0], prep_oracle.preprocess(im, 401))
    H, W = C.c_int(), C.c_int()
    _lib.check(_lib.lib().dsrg_engine_get_size(C.c_void_p(eng.h), C.byref(H), C.byref(W), None, None))
    assert (H.value, W.value) == (20, 30) and eng.capacity == (64, 64)
    eng.close()


def test_bad_arguments_are_refused_before_any_launch(torch_cuda):
    torch = torch_cuda
    dev = torch.cuda.current_device()
    L = _lib.lib()
    eng = api.Engine(1, 32, 32, 21)
    e = C.c_void_p(eng.h)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    H, W = 24, 40
    him = np.zeros((H, W, 3), np.uint8)
    dim = torch.zeros((H, W, 3), dtype=torch.uint8, device="cuda")
    mean = np.array([104.0, 117.0, 123.0])
    hout = [np.zeros((3, 8, 9), np.float32), np.zeros((3, 5, 5), np.float32)]
    dout = [torch.zeros((3, 8, 9), device="cuda"), torch.zeros((3, 5, 5), device="cuda")]

    def args(dev_variant, **kw):
        a = dict(image=C.c_void_p(dim.data_ptr() if dev_variant else him.ctypes.data), H=H, W=W, n=2,
                 hs=[8, 5], ws=[9, 5], mean=C.c_void_p(mean.ctypes.data),
                 outs=[o.data_ptr() for o in dout] if dev_variant else [o.ctypes.data for o in hout])
        a.update(kw)
        hs = None if a["hs"] is None else (C.c_int * len(a["hs"]))(*a["hs"])
        ws = None if a["ws"] is None else (C.c_int * len(a["ws"]))(*a["ws"])
        outs = None if a["outs"] is None else (C.c_void_p * len(a["outs"]))(*a["outs"])
        r = [e, a["image"], a["H"], a["W"], a["n"], hs, ws, a["mean"], outs]
        return r + [s] if dev_variant else r

    bad = [dict(image=None), dict(hs=None), dict(ws=None), dict(mean=None), dict(outs=None), dict(outs=[None, None]),
           dict(n=0), dict(n=-1), dict(n=17, hs=[8] * 17, ws=[9] * 17), dict(hs=[0, 5]), dict(ws=[9, 0]),
           dict(hs=[8, -5]), dict(H=0), dict(W=0), dict(H=-3)]
    eng.take_launch_count()
    for dev_variant, fn in ((True, L.dsrg_prepare_net_input_dev), (False, L.dsrg_prepare_net_input_host)):
        for kw in bad:
            rc = fn(*args(dev_variant, **kw))
            assert rc == _lib.E_INVALID, (dev_variant, kw, rc)
            assert eng.take_launch_count() == 0, (dev_variant, kw)
            assert torch.cuda.current_device() == dev
        assert fn(*args(dev_variant)) == _lib.OK
        assert eng.take_launch_count() == 1
    assert L.dsrg_prepare_net_input_host(None, *args(False)[1:]) == _lib.E_INVALID
    assert L.dsrg_last_error().decode() == "engine is NULL"
    torch.cuda.synchronize()
    assert np.array_equal(dout[0].cpu().numpy(), hout[0]) and np.array_equal(dout[1].cpu().numpy(), hout[1])
    eng.close()


def test_preprocess_then_predict_mask_keeps_replaying_graphs(torch_cuda):
    """test-ms.py's loop over images of alternating sizes: preprocess on the pooled engine before each
    predict_mask_ms re-shapes it no more often than predict_mask_ms alone, and the post-processing graphs are
    replayed as often."""
    cases = [synth.make_score_blobs(60 + i, H, W, (31, 41, 51)) for i, (H, W) in enumerate([(375, 500), (500, 375)])]
    rounds = 4

    def run(with_preprocess):
        pool.clear()
        eng = pool.engine_for(500, 500, 21)
        resizes = []
        orig = api.Engine.set_size

        def counting(self, H, W):
            if (int(H), int(W)) != (self.H, self.W):
                resizes.append((H, W))
            return orig(self, H, W)
        api.Engine.set_size = counting
        try:
            r0 = eng.graph_replays
            for _ in range(rounds):
                for c in cases:
                    if with_preprocess:
                        blobs = postprocess.preprocess(c["image"], (241, 321, 401))
                        assert [b.shape for b in blobs] == [(1, 3, s, s) for s in (241, 321, 401)]
                    postprocess.predict_mask_ms(c["image"], c["blobs"])
            assert pool.engine_for(500, 500, 21) is eng
            return eng.graph_replays - r0, len(resizes)
        finally:
            api.Engine.set_size = orig

    alone = run(False)
    assert alone[0] >= len(cases) * (rounds - 2)
    assert run(True) == alone


def _net(torch, M, seed):
    """A fixed stand-in for the network: 8x8 average pooling, then a 1x1 convolution to M channels (a matmul)."""
    g = torch.Generator().manual_seed(seed)
    wt = (torch.randn(M, 3, generator=g) * 0.05).cuda()
    b = (torch.randn(M, generator=g) * 0.5).cuda()

    def net(x):   # x (1, 3, h, w) -> (M, h', w')
        p = torch.nn.functional.avg_pool2d(x, 8, 8, ceil_mode=True)[0]
        return (torch.einsum("mc,chw->mhw", wt, p) + b[:, None, None]).contiguous()
    return net


@pytest.mark.parametrize("M", [21, 81])
def test_device_chain_on_one_stream_equals_host_chain(torch_cuda, M):
    torch = torch_cuda
    H, W = 375, 500
    sizes = (241, 321, 401) if M == 21 else (481,)
    im = synth.make_image(np.random.RandomState(M), H, W, "photo")
    rng = np.random.RandomState(M + 1)
    gt = rng.randint(0, M, (H, W)).astype(np.uint8)
    gt[rng.rand(H, W) < 0.05] = 255
    net = _net(torch, M, M)
    shapes = [postprocess.net_input_size(H, W, s) for s in sizes]
    for smooth in (False, True):
        # host chain: the tools' loop with the library's host entry points
        blobs = postprocess.preprocess(im, sizes, M=M)
        scores = [net(torch.from_numpy(b).cuda()).cpu().numpy() for b in blobs]
        host_lab = postprocess.predict_mask_ms(im, scores, smooth=smooth)
        host_cm = api.Confusion(M)
        host_cm.add_host(gt, host_lab)
        # device chain: everything on one side stream, nothing crosses PCIe in between
        eng = pool.engine_for(H, W, M)
        s = torch.cuda.Stream()
        dev_cm = api.Confusion(M)
        with torch.cuda.stream(s):
            d_im = torch.from_numpy(im).cuda()
            d_gt = torch.from_numpy(gt).cuda()
            outs = [torch.empty((1, 3, h, w), device="cuda") for h, w in shapes]
            eng.prepare_net_input_dev(d_im, outs, stream=s.cuda_stream)
            d_scores = [net(o) for o in outs]
            res = torch.empty((H, W), dtype=torch.int32, device="cuda")
            eng.predict_mask_dev(d_scores, d_im, res, params=api.crf_params(1.0), eps=postprocess.EPS,
                                 smooth=smooth, stream=s.cuda_stream)
            dev_cm.add_dev(d_gt, res, stream=s.cuda_stream)
        s.synchronize()
        for o, b in zip(outs, blobs):
            assert np.array_equal(o.cpu().numpy(), b)
        for d, h in zip(d_scores, scores):
            assert np.array_equal(d.cpu().numpy(), h)
        dev_lab = res.cpu().numpy()
        m_dev, inv_dev = dev_cm.read()
        m_host, inv_host = host_cm.read()
        assert len(np.unique(host_lab)) >= 2
        if not smooth:
            assert np.array_equal(dev_lab, host_lab)
            assert np.array_equal(m_dev, m_host) and np.array_equal(inv_dev, inv_host)
        else:   # the mean field's float atomics: near-ties may flip between any two runs
            assert (dev_lab != host_lab).mean() <= 1e-3
            assert np.abs(m_dev.astype(np.int64) - m_host.astype(np.int64)).sum() <= 2e-3 * H * W
        assert m_host.sum() + inv_host.sum() == (gt != 255).sum()
        dev_cm.close()
        host_cm.close()
