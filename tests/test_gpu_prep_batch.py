"""GPU tests of the batched network input of the evaluation tools (dsrg_prepare_net_input_batch_*,
postprocess.preprocess_batch / preprocess_batch_dev) and of the mixed-size device post-processing
(postprocess.predict_masks_dev): bit-exact against the numpy restatement of preprocess() and the per-image call, the
launch count, the entry-point contract, streams and CUDA-graph capture, and the whole device chain against the
per-image host chain."""
import ctypes as C

import numpy as np
import pytest

from dsrg_b200 import _lib, api, pool, postprocess, synth
from oracle import prep_oracle

pytestmark = pytest.mark.gpu

VOC = [(500, 375), (375, 500), (333, 500)]
FIB16 = [45, 1, 2, 3, 5, 8, 13, 21, 34, 55, 89, 7, 12, 60, 100, 16]   # 16 scales, down and up


def _sizes(B, choices, seed):
    rng = np.random.RandomState(seed)
    return [choices[i] for i in rng.randint(0, len(choices), B)]


def _images(shapes, seed, variant="photo"):
    rng = np.random.RandomState(seed)
    return [synth.make_image(rng, H, W, variant) for H, W in shapes]


# name, image shapes, sizes, relative
CASES = [
    ("b1", VOC[:1], (241, 321, 401), False),
    ("b2", VOC[1:], (241, 321, 401), False),
    ("b5", _sizes(5, VOC, 1), (241, 321, 401), False),
    ("b16", _sizes(16, VOC, 2), (241, 321, 401), False),
    ("over_one_launch", _sizes(_lib.PREP_IMAGES_PER_LAUNCH + 6, [(23, 31), (40, 51), (31, 17), (9, 60)], 3),
     (45, 30), False),
    ("coco", [(640, 427), (427, 640), (640, 427)], (481,), False),
    ("relative_ties", [(334, 500), (334, 500), (334, 500)], (0.75, 1, 1.25), True),
    ("edges", [(40, 51), (1, 17), (17, 1), (1, 1), (9, 7)], FIB16, False),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_batch_equals_restatement_and_per_image_call(torch_cuda, case):
    torch = torch_cuda
    name, shapes, sizes, relative = case
    M = 81 if name == "coco" else 21
    ims = _images(shapes, len(shapes) + len(sizes), "noise" if name == "edges" else "photo")
    B = len(ims)
    eng = pool.prep_engine_for(B, torch.cuda.current_device())
    eng.take_launch_count()
    got = postprocess.preprocess_batch(ims, sizes, relative=relative, M=M)
    assert eng.take_launch_count() == postprocess.prep_launches(B)
    want_shapes = [prep_oracle.output_shape(shapes[0][0], shapes[0][1], s, relative) for s in sizes]
    assert [g.shape for g in got] == [(B, 3, h, w) for h, w in want_shapes]
    hit = False
    for b, im in enumerate(ims):
        single = postprocess.preprocess(im, sizes, relative=relative, M=M)
        for k, size in enumerate(sizes):
            want = prep_oracle.preprocess(im, size, relative)
            assert got[k].dtype == np.float32 and np.array_equal(got[k][b], want), (name, b, size)
            assert np.array_equal(got[k][b], single[k][0]), (name, b, size)
            hit |= prep_oracle.hits_cval(im.shape[0], im.shape[1], want.shape[1], want.shape[2])
    if name == "edges":
        assert hit      # the 40 x 51 image has scipy's 0 in its last column at 45
    # _dev equals _host, from a list of per-image tensors and, for one size, from one (B, H, W, 3) tensor
    d_ims = [torch.from_numpy(im).cuda() for im in ims]
    eng.take_launch_count()
    dev = postprocess.preprocess_batch_dev(d_ims, sizes, relative=relative, M=M)
    torch.cuda.synchronize()
    assert eng.take_launch_count() == postprocess.prep_launches(B)
    for k in range(len(sizes)):
        assert np.array_equal(dev[k].cpu().numpy(), got[k]), (name, k)
    if len(set(shapes)) == 1:
        stacked = postprocess.preprocess_batch_dev(torch.stack(d_ims), sizes, relative=relative, M=M)
        for k in range(len(sizes)):
            assert np.array_equal(stacked[k].cpu().numpy(), got[k]), (name, k)


def test_other_mean_and_engine_growth(torch_cuda):
    torch = torch_cuda
    ims = _images([(37, 53), (53, 37)], 9)
    mean = [1.5, -2.0, 0.0]
    got = postprocess.preprocess_batch(ims, [29], mean_pixel=mean)
    for b, im in enumerate(ims):
        assert np.array_equal(got[0][b], prep_oracle.preprocess(im, 29, mean_pixel=np.array(mean)))
    # the network-input engine grows in batch only, and the post-processing engines are left alone
    pool.clear()
    small = pool.prep_engine_for(2, torch.cuda.current_device())
    postprocess.preprocess_batch(_images([(700, 20), (20, 900), (64, 64)], 10), [41])
    big = pool.prep_engine_for(3, torch.cuda.current_device())
    assert big is not small and big.max_batch == 3 and big.capacity == (1, 1)
    assert not pool._ENGINES and not pool._BATCH_ENGINES


def test_bad_arguments_are_refused_before_any_launch(torch_cuda):
    torch = torch_cuda
    dev = torch.cuda.current_device()
    L = _lib.lib()
    eng = api.Engine(4, 1, 1, 1)
    e = C.c_void_p(eng.h)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    shapes = [(24, 40), (31, 17)]
    him = [np.zeros(sh + (3,), np.uint8) for sh in shapes]
    dim = [torch.zeros(sh + (3,), dtype=torch.uint8, device="cuda") for sh in shapes]
    mean = np.array([104.0, 117.0, 123.0])
    hout = [np.zeros((2, 3, 8, 9), np.float32), np.zeros((2, 3, 5, 5), np.float32)]
    dout = [torch.zeros((2, 3, 8, 9), device="cuda"), torch.zeros((2, 3, 5, 5), device="cuda")]

    def args(dev_variant, **kw):
        a = dict(images=[t.data_ptr() for t in dim] if dev_variant else [x.ctypes.data for x in him],
                 Hs=[h for h, _ in shapes], Ws=[w for _, w in shapes], B=2, n=2, hs=[8, 5], ws=[9, 5],
                 mean=C.c_void_p(mean.ctypes.data),
                 outs=[o.data_ptr() for o in dout] if dev_variant else [o.ctypes.data for o in hout])
        a.update(kw)
        arr = lambda t, v: None if v is None else (t * len(v))(*v)   # noqa: E731
        r = [e, arr(C.c_void_p, a["images"]), arr(C.c_int, a["Hs"]), arr(C.c_int, a["Ws"]), a["B"], a["n"],
             arr(C.c_int, a["hs"]), arr(C.c_int, a["ws"]), a["mean"], arr(C.c_void_p, a["outs"])]
        return r + [s] if dev_variant else r

    big = 1 << 16
    bad = [dict(images=None), dict(images=[None, None]), dict(Hs=None), dict(Ws=None), dict(Hs=[24, 0]),
           dict(Ws=[-1, 17]), dict(Hs=[big, 17], Ws=[big // 2, 17]), dict(B=0), dict(B=5), dict(B=-1),
           dict(n=0), dict(n=17, hs=[8] * 17, ws=[9] * 17), dict(hs=None), dict(ws=None), dict(hs=[0, 5]),
           dict(ws=[9, -5]), dict(hs=[big, 5], ws=[big // 2, 5]), dict(mean=None), dict(outs=None),
           dict(outs=[None, None])]
    eng.take_launch_count()
    for dev_variant, fn in ((True, L.dsrg_prepare_net_input_batch_dev), (False, L.dsrg_prepare_net_input_batch_host)):
        for kw in bad:
            rc = fn(*args(dev_variant, **kw))
            assert rc == _lib.E_INVALID, (dev_variant, kw, rc)
            assert eng.take_launch_count() == 0, (dev_variant, kw)
            assert torch.cuda.current_device() == dev
        assert fn(*args(dev_variant)) == _lib.OK, L.dsrg_last_error()
        assert eng.take_launch_count() == 1
    assert L.dsrg_prepare_net_input_batch_host(None, *args(False)[1:]) == _lib.E_INVALID
    assert L.dsrg_last_error().decode() == "engine is NULL"
    torch.cuda.synchronize()
    for d, h in zip(dout, hout):
        assert np.array_equal(d.cpu().numpy(), h)
    eng.close()

    # the Python side: ValueError before anything is queued, on the network-input engine and on the batch engine
    pool.clear()
    peng = pool.prep_engine_for(2, dev)
    peng.take_launch_count()
    beng = pool.batch_engine_for(2, 64, 64, 21, dev)
    beng.take_launch_count()
    d_ims = [torch.from_numpy(x).cuda() for x in _images(shapes, 4)]
    big_scores = [torch.zeros((2, 21, 100, 100), device="cuda")]   # more pixels than the 64 x 64 engine holds
    calls = [
        lambda: postprocess.preprocess_batch_dev(d_ims, [0.75], relative=True),       # two shapes for one size
        lambda: postprocess.preprocess_batch_dev(d_ims, []),
        lambda: postprocess.preprocess_batch_dev([d_ims[0].float(), d_ims[1]], [41]),
        lambda: postprocess.preprocess_batch_dev([d_ims[0].cpu(), d_ims[1]], [41]),
        lambda: postprocess.preprocess_batch_dev([d_ims[0][:, ::2], d_ims[1]], [41]),  # not contiguous
        lambda: postprocess.preprocess_batch_dev(d_ims, [41], mean_pixel=(1.0, 2.0)),
        lambda: postprocess.preprocess_batch_dev(d_ims, [41], M=0),
        lambda: postprocess.preprocess_batch_dev(d_ims, [41], out=[torch.empty((2, 3, 41, 40), device="cuda")]),
        lambda: postprocess.preprocess_batch_dev(d_ims, [41, 5], out=[torch.empty((2, 3, 41, 41), device="cuda")]),
        lambda: postprocess.preprocess_batch_dev(torch.stack([d_ims[0], d_ims[0]]).transpose(1, 2), [41]),
        lambda: postprocess.preprocess_batch([x.cpu().numpy() for x in d_ims], [1.5], relative=True),
        lambda: postprocess.predict_masks_dev(d_ims, [torch.zeros((3, 21, 5, 5), device="cuda")]),
        lambda: postprocess.predict_masks_dev(d_ims, [torch.zeros((2, 21, 5, 5), device="cuda")], mode="x"),
        lambda: postprocess.predict_masks_dev(d_ims, [torch.zeros((2, 21, 5, 5), device="cuda")],
                                              labels=torch.zeros((2, 20), device="cuda")),
        lambda: postprocess.predict_masks_dev(d_ims, big_scores),
        lambda: postprocess.net_input_shapes([(24, 40)], list(range(1, 18))),               # 17 sizes
        lambda: postprocess.preprocess_batch_dev(d_ims, list(range(1, 18))),
        lambda: postprocess.preprocess_batch_dev(d_ims[:1], [1 << 16], relative=True),    # planes of 2^31 and more
        lambda: postprocess.preprocess_batch_dev([d_ims[0], d_ims[1][:0]], [41]),          # an image of no rows
    ]
    size = (beng.H, beng.W)
    for i, call in enumerate(calls):
        with pytest.raises(ValueError):
            call()
        assert peng.take_launch_count() == 0, i
        assert beng.take_launch_count() == 0, i
        assert pool._BATCH_ENGINES[(21, dev)] is beng and (beng.H, beng.W) == size, i   # neither replaced nor re-shaped
        assert torch.cuda.current_device() == dev
    # without an engine, the capacity check creates none
    pool.clear()
    with pytest.raises(ValueError):
        postprocess.predict_masks_dev(d_ims, big_scores)
    assert not pool._BATCH_ENGINES


def _net(torch, M, seed):
    """A fixed stand-in for the network: 8x8 average pooling (41 x 41 at 321), then a 1x1 convolution to M channels
    written out channel by channel, so that every image's scores are the same arithmetic whatever the batch."""
    g = torch.Generator().manual_seed(seed)
    wt = (torch.randn(M, 3, generator=g) * 0.05).cuda()
    b = (torch.randn(M, generator=g) * 0.5).cuda()

    def net(x):   # x (B, 3, h, w) -> (B, M, h', w')
        p = torch.nn.functional.avg_pool2d(x, 8, 8, ceil_mode=True)
        out = wt[None, :, 0, None, None] * p[:, None, 0]
        out = out + wt[None, :, 1, None, None] * p[:, None, 1]
        out = out + wt[None, :, 2, None, None] * p[:, None, 2]
        return (out + b[None, :, None, None]).contiguous()
    return net


def test_side_stream_and_captured_chain(torch_cuda):
    torch = torch_cuda
    M, H, W, sizes = 21, 375, 500, (241, 321, 401)
    net = _net(torch, M, 3)
    ims = _images([(H, W)] * 4, 21)
    want = postprocess.preprocess_batch(ims, sizes)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_in = torch.from_numpy(np.stack(ims)).cuda()
        outs = postprocess.preprocess_batch_dev(d_in, sizes)
    s.synchronize()
    for o, w in zip(outs, want):
        assert np.array_equal(o.cpu().numpy(), w)

    def step():
        x = postprocess.preprocess_batch_dev(d_in, sizes, out=outs)
        return postprocess.predict_mask_batch_dev(d_in, [net(o) for o in x], smooth=False, out=res)

    res = torch.empty((4, H, W), dtype=torch.int32, device="cuda")
    with torch.cuda.stream(s):   # warm-up: every engine exists at this batch before the capture
        step()
    s.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    torch.cuda.synchronize()
    new = _images([(H, W)] * 4, 22)
    d_in.copy_(torch.from_numpy(np.stack(new)))
    graph.replay()
    torch.cuda.synchronize()
    replayed = [o.cpu().numpy() for o in outs], res.cpu().numpy()
    eager_in = postprocess.preprocess_batch(new, sizes)
    for r, w in zip(replayed[0], eager_in):
        assert np.array_equal(r, w)
    eager = step()
    torch.cuda.synchronize()
    assert np.array_equal(replayed[1], eager.cpu().numpy())
    assert len(np.unique(replayed[1])) >= 2


def _returns_while_the_stream_is_busy(torch, stream, fn):
    """Run fn() behind a long device-side sleep on `stream` and check that it came back to the host while the sleep
    still ran: any wait for the device, torch's or the library's own (cudaDeviceSynchronize, a stream or event
    synchronisation), would have waited for the sleep.  Returns fn's result once the stream has finished."""
    with torch.cuda.stream(stream):
        torch.cuda._sleep(2_000_000_000)   # about a second at the H100's SM clock
        got = fn()
        busy = not stream.query()
    stream.synchronize()
    assert busy, "the call waited for the device"
    return got


def test_predict_masks_dev_keeps_input_order_without_sync(torch_cuda):
    torch = torch_cuda
    M = 21
    shapes = [(375, 500), (500, 375), (333, 500), (375, 500), (500, 375)]
    ims = _images(shapes, 31)
    net = _net(torch, M, 5)
    d_ims = [torch.from_numpy(im).cuda() for im in ims]
    rng = np.random.RandomState(8)
    tags = (rng.rand(len(ims), M) < 0.2).astype(np.float32)
    d_tags = torch.from_numpy(tags).cuda()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        scores = [net(x) for x in postprocess.preprocess_batch_dev(d_ims, (241, 321, 401))]
    for mode, sc, lab, smooth in (("ms", scores, None, False), ("gt", scores[1:2], d_tags, False),
                                  ("ms", scores, None, True)):
        with torch.cuda.stream(side):   # warm-up: the engine's capacity for this batch and its largest image
            postprocess.predict_masks_dev(d_ims, sc, labels=lab, mode=mode, smooth=smooth)
        side.synchronize()
        reshapes = []
        orig = api.Engine.set_size

        def counting(self, H, W, ordered=False):
            if (int(H), int(W)) != (self.H, self.W):
                reshapes.append(ordered)
            return orig(self, H, W, ordered)
        def call():
            torch.cuda.set_sync_debug_mode("error")
            try:
                return postprocess.predict_masks_dev(d_ims, sc, labels=lab, mode=mode, smooth=smooth)
            finally:
                torch.cuda.set_sync_debug_mode("default")
        api.Engine.set_size = counting
        try:
            got = _returns_while_the_stream_is_busy(torch, side, call)
        finally:
            api.Engine.set_size = orig
        # one re-shape per size group after the first, none of them waiting for the device
        assert len(reshapes) >= 2 and all(reshapes), reshapes
        assert [tuple(g.shape) for g in got] == shapes and all(g.dtype == torch.int32 for g in got)
        if smooth:
            continue
        for i, im in enumerate(d_ims):
            alone = postprocess.predict_mask_batch_dev(im[None], [s[i:i + 1] for s in sc],
                                                       None if lab is None else lab[i:i + 1], mode, smooth=False)
            assert torch.equal(got[i], alone[0]), (mode, i)


def test_preprocess_batch_dev_does_not_wait_for_the_device(torch_cuda):
    torch = torch_cuda
    d_ims = [torch.from_numpy(im).cuda() for im in _images([(375, 500), (500, 375), (333, 500)], 33)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        postprocess.preprocess_batch_dev(d_ims, (241, 321, 401))   # the engine exists at this batch
    got = _returns_while_the_stream_is_busy(torch, side,
                                            lambda: postprocess.preprocess_batch_dev(d_ims, (241, 321, 401)))
    want = postprocess.preprocess_batch([im.cpu().numpy() for im in d_ims], (241, 321, 401))
    for g, w in zip(got, want):
        assert np.array_equal(g.cpu().numpy(), w)


CHAINS = [
    (21, _sizes(6, VOC, 41), (241, 321, 401)),
    (81, [(640, 427), (427, 640), (640, 427)], (481,)),
]


@pytest.mark.parametrize("M,shapes,sizes", CHAINS, ids=["voc21", "coco81"])
def test_device_chain_equals_per_image_host_chain(torch_cuda, M, shapes, sizes):
    torch = torch_cuda
    ims = _images(shapes, M)
    rng = np.random.RandomState(M + 1)
    gts = []
    for H, W in shapes:
        gt = rng.randint(0, M, (H, W)).astype(np.uint8)
        gt[rng.rand(H, W) < 0.05] = 255
        gts.append(gt)
    net = _net(torch, M, M)
    for smooth in (False, True):
        # host chain: the tools' loop, one image at a time
        host_cm = api.Confusion(M)
        host_lab, host_probs = [], []
        for im, gt in zip(ims, gts):
            blobs = postprocess.preprocess(im, sizes, M=M)
            scores = [net(torch.from_numpy(b).cuda())[0].cpu().numpy() for b in blobs]
            lab, probs = postprocess.predict_mask_ms(im, scores, smooth=smooth, return_probs=True)
            host_cm.add_host(gt, lab)
            host_lab.append(lab)
            host_probs.append(probs)
        # device chain: one network batch per scale, post-processing grouped by size, counted on the device
        dev_cm = api.Confusion(M)
        d_ims = [torch.from_numpy(im).cuda() for im in ims]
        d_gts = [torch.from_numpy(gt).cuda() for gt in gts]
        fc8 = [net(x) for x in postprocess.preprocess_batch_dev(d_ims, sizes, M=M)]
        preds = postprocess.predict_masks_dev(d_ims, fc8, smooth=smooth)
        for g, p in zip(d_gts, preds):
            dev_cm.add_dev(g, p)
        torch.cuda.synchronize()
        m_dev, inv_dev = dev_cm.read()
        m_host, inv_host = host_cm.read()
        if not smooth:
            for p, h in zip(preds, host_lab):
                assert np.array_equal(p.cpu().numpy(), h)
            assert np.array_equal(m_dev, m_host) and np.array_equal(inv_dev, inv_host)
        else:   # the mean field's float atomics: only near-ties may flip
            flips = 0
            for p, h, q in zip(preds, host_lab, host_probs):
                top2 = np.sort(q, axis=-1)[..., -2:]
                differ = p.cpu().numpy() != h
                assert (top2[..., 1] - top2[..., 0])[differ].max(initial=0.0) <= 2e-4
                flips += int(differ.sum())
            assert np.abs(m_dev.astype(np.int64) - m_host.astype(np.int64)).sum() <= 2 * flips
            assert np.array_equal(inv_dev, inv_host)
        assert len(np.unique(np.concatenate([h.ravel() for h in host_lab]))) >= 2
        dev_cm.close()
        host_cm.close()
