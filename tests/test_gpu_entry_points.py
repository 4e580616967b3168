"""GPU tests of the engine entry points' shared prologue and of the *_host staging path: the batch range and the
NULL-pointer rule are refused before anything is launched, each *_dev entry point computes what its *_host twin
computes, and the *_host layers leave the retained CRF marginals alone."""
import ctypes as C

import numpy as np
import pytest

from dsrg_b200 import _lib, api, synth

pytestmark = pytest.mark.gpu

MAXB, H, W, M = 2, 24, 24, 21
HI = WI = 16      # raw image size of prepare_image / annotation
SH = SW = 12      # score map size of zoom_scores / predict_mask
NHWC, NCHW = _lib.LAYOUT_NHWC, _lib.LAYOUT_NCHW


def _p(x):
    """c_void_p of a torch CUDA tensor, a numpy array or a ctypes array."""
    if hasattr(x, "data_ptr"):
        return C.c_void_p(x.data_ptr())
    if isinstance(x, np.ndarray):
        return C.c_void_p(x.ctypes.data)
    return C.cast(x, C.c_void_p)


class Ctx(object):
    """An engine and one set of valid arguments for every engine entry point, device and host."""

    def __init__(self, torch):
        self.eng = api.Engine(MAXB, H, W, M)
        self.L = _lib.lib()
        rng = np.random.RandomState(7)
        n = MAXB * M * H * W
        self.hf = [rng.uniform(0.05, 1.0, n).astype(np.float32) for _ in range(4)]
        lab = np.zeros((MAXB, M), np.float32)
        lab[:, 0] = lab[0, 3] = lab[1, 5] = 1
        self.hlab = lab
        self.himg = rng.randint(0, 256, (MAXB, H, W, 3)).astype(np.uint8)
        self.hraw = [rng.uniform(0, 255, (MAXB, 3, HI, WI)).astype(np.float32) for _ in range(2)]
        self.hi32 = [np.zeros(MAXB * H * W, np.int32) for _ in range(2)]
        self.df = [torch.from_numpy(a).cuda() for a in self.hf]
        self.dlab = torch.from_numpy(lab).cuda()
        self.dimg = torch.from_numpy(self.himg).cuda()
        self.draw = [torch.from_numpy(a).cuda() for a in self.hraw]
        self.di32 = torch.zeros(MAXB * H * W, dtype=torch.int32, device="cuda")
        self.params = api.crf_params(scale_factor=1.0)
        self.mean = np.array([104.0, 117.0, 123.0])
        # annotation index lists for MAXB images (one spare offset for B = MAXB + 1, which is refused unread)
        self.toff = np.array([0, 1, 2, 2], np.int32)
        self.tags = np.array([3, 5], np.int32)
        self.coff = np.array([0, 1, 2, 2], np.int32)
        self.cidx = np.array([[3, 5], [1, 2], [4, 6]], np.int32)
        self.flip = np.array([0, 1], np.int32)
        self.hsc = [rng.randn(M, SH, SW).astype(np.float32)]
        self.dsc = [torch.from_numpy(a).cuda() for a in self.hsc]
        self.hs = (C.c_int * 1)(SH)
        self.ws = (C.c_int * 1)(SW)
        self.hptrs = (C.c_void_p * 1)(self.hsc[0].ctypes.data)
        self.dptrs = (C.c_void_p * 1)(self.dsc[0].data_ptr())
        self.sel = np.array([0, 3, 5], np.int32)
        self.stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        # outputs of the lattice read-outs (tile views: 3 tiles of up to 256 local vertices)
        self.counts = np.zeros(3, np.int64)
        self.tl = [np.zeros(4, np.int32), np.zeros(4, np.uint8), np.zeros(4 * 256 * 2, np.int32),
                   np.zeros(6 * H * W, np.uint16)]
        self.off = np.zeros(6 * H * W, np.int32)

    def calls(self):
        """name -> (argument list with "B" for the batch size, required pointer positions)."""
        e, s, prm = C.c_void_p(self.eng.h), self.stream, C.byref(self.params)
        f, d, lab, dlab = [_p(a) for a in self.hf], [_p(a) for a in self.df], _p(self.hlab), _p(self.dlab)
        img, dimg, raw, draw = _p(self.himg), _p(self.dimg), [_p(a) for a in self.hraw], [_p(a) for a in self.draw]
        i32, di32, mean = [_p(a) for a in self.hi32], _p(self.di32), _p(self.mean)
        toff, tags, coff, cidx, flip = [_p(a) for a in (self.toff, self.tags, self.coff, self.cidx, self.flip)]
        sel = _p(self.sel)
        return {
            "dsrg_crf_batch_dev": ([e, "B", d[0], NHWC, dimg, prm, d[1], NHWC, s], [2, 4, 5, 6]),
            "dsrg_crf_batch_host": ([e, "B", f[0], NHWC, img, prm, f[1], NHWC], [2, 4, 5, 6]),
            "dsrg_crf_map_batch_dev": ([e, "B", d[0], NHWC, dimg, prm, di32, s], [2, 4, 5, 6]),
            "dsrg_srg_batch_dev": ([e, "B", dlab, d[0], d[1], 0.99, 0.85, 0, d[2], None, s], [2, 3, 4, 8]),
            "dsrg_srg_batch_host": ([e, "B", lab, f[0], f[1], 0.99, 0.85, 0, f[2], None], [2, 3, 4, 8]),
            "dsrg_dsrg_forward_dev": ([e, "B", dlab, d[0], d[1], dimg, prm, 0.99, 0.85, d[2], None, s],
                                      [2, 3, 4, 5, 6, 9]),
            "dsrg_dsrg_forward_host": ([e, "B", lab, f[0], f[1], img, prm, 0.99, 0.85, f[2], None], [2, 3, 4, 5, 6, 9]),
            "dsrg_softmax_forward_dev": ([e, "B", d[0], d[1], s], [2, 3]),
            "dsrg_softmax_backward_dev": ([e, "B", d[0], d[1], d[2], s], [2, 3, 4]),
            "dsrg_constrainloss_forward_dev": ([e, "B", d[0], d[1], d[2], s], [2, 3, 4]),
            "dsrg_constrainloss_backward_dev": ([e, "B", d[0], d[1], d[2], d[3], s], [2, 3, 4, 5]),
            "dsrg_softmax_forward_host": ([e, "B", f[0], f[1]], [2, 3]),
            "dsrg_softmax_backward_host": ([e, "B", f[0], f[1], f[2]], [2, 3, 4]),
            "dsrg_constrainloss_forward_host": ([e, "B", f[0], f[1], f[2]], [2, 3, 4]),
            "dsrg_constrainloss_backward_host": ([e, "B", f[0], f[1], f[2], f[3]], [2, 3, 4, 5]),
            "dsrg_prepare_image_dev": ([e, "B", HI, WI, draw[0], mean, dimg, s], [4, 5, 6]),
            "dsrg_prepare_image_host": ([e, "B", HI, WI, raw[0], mean, img], [4, 5, 6]),
            "dsrg_annotation_forward_dev": ([e, "B", toff, tags, coff, cidx, flip, draw[0], HI, WI, dlab, d[0],
                                             draw[1], s], [2, 4, 7, 10, 11]),
            "dsrg_annotation_forward_host": ([e, "B", toff, tags, coff, cidx, flip, raw[0], HI, WI, lab, f[0], raw[1]],
                                             [2, 4, 7, 10, 11]),
            "dsrg_crflayer_forward_dev": ([e, "B", d[0], dimg, prm, d[1], None, s], [2, 3, 4, 5]),
            "dsrg_crflayer_forward_host": ([e, "B", f[0], img, prm, f[1], None], [2, 3, 4, 5]),
            "dsrg_srg_last_crf_host": ([e, "B", lab, f[1], 0.99, 0.85, f[2]], [2, 3, 6]),
            "dsrg_crf_last_marginals_host": ([e, "B", f[3], NCHW], [2]),
            "dsrg_seedloss_forward_dev": ([e, "B", d[0], d[1], d[2], s], [2, 3, 4]),
            "dsrg_seedloss_backward_dev": ([e, "B", 2, d[0], d[1], 1.0, d[2], s], [3, 4, 6]),
            "dsrg_seedloss_forward_host": ([e, "B", f[0], f[1], f[2]], [2, 3, 4]),
            "dsrg_seedloss_backward_host": ([e, "B", 2, f[0], f[1], 1.0, f[2]], [3, 4, 6]),
            "dsrg_seedloss_plain_forward_dev": ([e, "B", d[0], d[1], d[2], s], [2, 3, 4]),
            "dsrg_seedloss_plain_backward_dev": ([e, "B", 2, d[0], d[1], d[2], s], [3, 4, 5]),
            "dsrg_seedloss_plain_forward_host": ([e, "B", f[0], f[1], f[2]], [2, 3, 4]),
            "dsrg_seedloss_plain_backward_host": ([e, "B", 2, f[0], f[1], f[2]], [3, 4, 5]),
            "dsrg_expandloss_forward_dev": ([e, "B", d[0], dlab, 0.996, 0.999, d[2], s], [2, 3, 6]),
            "dsrg_expandloss_backward_dev": ([e, "B", 2, d[0], dlab, 0.996, 0.999, d[2], s], [3, 4, 7]),
            "dsrg_expandloss_forward_host": ([e, "B", f[0], lab, 0.996, 0.999, f[2]], [2, 3, 6]),
            "dsrg_expandloss_backward_host": ([e, "B", 2, f[0], lab, 0.996, 0.999, f[2]], [3, 4, 7]),
            "dsrg_engine_lattice_sizes": ([e, "B", _p(self.hi32[0]), _p(self.hi32[1])], []),
            "dsrg_engine_copy_norm": ([e, 1, "B", f[3]], [3]),
            "dsrg_engine_lattice_bary": ([e, 1, MAXB - 1, f[3]], [3]),
            "dsrg_engine_lattice_idle": ([e, 1, _p(self.counts)], [2]),
            "dsrg_engine_tile_views": ([e, 1, MAXB - 1] + [_p(a) for a in self.tl] + [f[3]], [7]),
            "dsrg_zoom_scores_dev": ([e, _p(self.dsc[0]), SH, SW, d[3], 0, s], [1, 4]),
            "dsrg_zoom_scores_host": ([e, _p(self.hsc[0]), SH, SW, f[3], 0], [1, 4]),
            "dsrg_predict_mask_dev": ([e, _lib.POST_SUM_SCORES, 1, _p(self.dptrs), _p(self.hs), _p(self.ws), dimg,
                                       1e-5, 1, prm, sel, 3, di32, None, s], [3, 4, 5, 6, 9, 10, 12]),
            "dsrg_predict_mask_host": ([e, _lib.POST_SUM_SCORES, 1, _p(self.hptrs), _p(self.hs), _p(self.ws), img,
                                        1e-5, 1, prm, sel, 3, i32[0], None], [3, 4, 5, 6, 9, 10, 12]),
        }

    def call(self, name, args, B):
        return getattr(self.L, name)(*[B if a == "B" else a for a in args])


@pytest.fixture(scope="module")
def ctx(torch_cuda):
    c = Ctx(torch_cuda)
    yield c
    c.eng.close()


def test_every_batched_entry_point_is_covered(ctx):
    from test_entry_points_cpu import engine_functions
    calls = ctx.calls()
    for name in engine_functions():
        args = _lib.SIGNATURES[name][1]
        if len(args) > 1 and args[1] is _lib.C.c_int and name.endswith(("_dev", "_host")):
            assert name in calls, name


def test_batch_range_is_refused_before_any_launch(ctx, torch_cuda):
    torch = torch_cuda
    dev = torch.cuda.current_device()
    batched = {k: v for k, v in ctx.calls().items() if "B" in v[0]}
    assert len(batched) == 37
    ctx.eng.take_launch_count()
    for name, (args, _) in batched.items():
        for B in (0, MAXB + 1):
            rc = ctx.call(name, args, B)
            assert rc == _lib.E_INVALID, (name, B, rc)
            assert "batch %d outside [1, %d]" % (B, MAXB) in ctx.L.dsrg_last_error().decode(), name
    assert ctx.eng.take_launch_count() == 0
    assert torch.cuda.current_device() == dev


def test_null_arguments_are_refused_before_any_launch(ctx, torch_cuda):
    if ctx.L.dsrg_version() < 102:
        pytest.skip("libraries before version 102 launch some entry points on NULL pointers")
    torch = torch_cuda
    dev = torch.cuda.current_device()
    ctx.eng.take_launch_count()
    for name, (args, required) in ctx.calls().items():
        for k in required:
            bad = list(args)
            bad[k] = None
            rc = ctx.call(name, bad, MAXB)
            assert rc == _lib.E_INVALID, (name, k, rc)
            assert ctx.eng.take_launch_count() == 0, (name, k)
    assert torch.cuda.current_device() == dev
    # the same argument lists are valid as they stand
    torch.cuda.synchronize()
    for name, (args, _) in ctx.calls().items():
        if "_last_" in name:
            assert ctx.call("dsrg_crf_batch_host", ctx.calls()["dsrg_crf_batch_host"][0], MAXB) == _lib.OK
        rc = ctx.call(name, args, MAXB)
        assert rc == _lib.OK, (name, rc, ctx.L.dsrg_last_error().decode())
    torch.cuda.synchronize()


def test_lattice_read_outs_refuse_bad_indices(ctx, torch_cuda):
    """which outside {0, 1} and an image index outside [0, max_batch) are refused like a NULL output."""
    calls = ctx.calls()
    ctx.eng.take_launch_count()
    for name in ("dsrg_engine_lattice_tables", "dsrg_engine_lattice_bary", "dsrg_engine_lattice_idle",
                 "dsrg_engine_tile_views"):
        args = calls[name][0] if name in calls else [C.c_void_p(ctx.eng.h), 1, MAXB - 1, _p(ctx.off), None]
        bad = [(1, v) for v in (-1, 2)] + ([(2, v) for v in (-1, MAXB)] if name != "dsrg_engine_lattice_idle" else [])
        for k, v in bad:
            a = list(args)
            a[k] = v
            assert ctx.call(name, a, MAXB) == _lib.E_INVALID, (name, k, v)
            assert "bad argument" in ctx.L.dsrg_last_error().decode(), (name, k, v)
        assert ctx.call(name, args, MAXB) == _lib.OK, name
    assert ctx.eng.take_launch_count() == 0


def _batch(B=2, Hh=41, Ww=41):
    b = synth.make_batch(B, Hh, Ww, cues="random", start=30)
    probs = b["probs"].copy()
    probs[probs < 1e-4] = 1e-4
    return b, probs


def test_softmax_and_constrainloss_dev_match_host(torch_cuda):
    torch = torch_cuda
    L = _lib.lib()
    b, probs = _batch()
    eng = api.Engine(2, 41, 41, M)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rng = np.random.RandomState(3)
    preds = rng.randn(*probs.shape).astype(np.float32) * 3
    top = rng.randn(*probs.shape).astype(np.float32)
    logs = np.log(probs[:, ::-1].copy())
    d = {k: torch.from_numpy(v).cuda() for k, v in dict(preds=preds, top=top, probs=probs, logs=logs).items()}
    out, out2 = torch.empty_like(d["probs"]), torch.empty_like(d["probs"])
    loss = torch.zeros(1, device="cuda")

    _lib.check(L.dsrg_softmax_forward_dev(C.c_void_p(eng.h), 2, _p(d["preds"]), _p(out), s))
    np.testing.assert_array_equal(out.cpu().numpy(), eng.softmax_forward_host(preds))
    _lib.check(L.dsrg_softmax_backward_dev(C.c_void_p(eng.h), 2, _p(d["preds"]), _p(d["top"]), _p(out), s))
    np.testing.assert_array_equal(out.cpu().numpy(), eng.softmax_backward_host(preds, top))
    _lib.check(L.dsrg_constrainloss_forward_dev(C.c_void_p(eng.h), 2, _p(d["probs"]), _p(d["logs"]), _p(loss), s))
    want = eng.constrainloss_forward_host(probs, logs)
    assert abs(float(loss.item()) - want) <= 1e-6 * abs(want)    # float atomics sum the terms
    _lib.check(L.dsrg_constrainloss_backward_dev(C.c_void_p(eng.h), 2, _p(d["probs"]), _p(d["logs"]), _p(out),
                                                 _p(out2), s))
    gp, gl = eng.constrainloss_backward_host(probs, logs)
    np.testing.assert_array_equal(out.cpu().numpy(), gp)
    np.testing.assert_array_equal(out2.cpu().numpy(), gl)
    eng.close()


def test_losses_dev_match_host(torch_cuda):
    torch = torch_cuda
    b, probs = _batch()
    seeds = b["cues"]
    labels = b["labels"].astype(np.float32)
    eng = api.Engine(2, 41, 41, M)
    dp, ds, dl = (torch.from_numpy(a).cuda() for a in (probs, seeds, labels))
    grad = torch.empty_like(dp)

    terms = torch.zeros(2, device="cuda")
    eng.seedloss_forward_dev(dp, ds, terms)
    np.testing.assert_array_equal(terms.cpu().numpy(), eng.seedloss_forward_host(probs, seeds))
    eng.seedloss_backward_dev(dp, ds, grad, top_diff=0.5)
    np.testing.assert_array_equal(grad.cpu().numpy(), eng.seedloss_backward_host(probs, seeds, top_diff=0.5))

    terms = torch.zeros(1, device="cuda")
    eng.seedloss_plain_forward_dev(dp, ds, terms)
    np.testing.assert_array_equal(terms.cpu().numpy(), eng.seedloss_plain_forward_host(probs, seeds))
    eng.seedloss_plain_backward_dev(dp, ds, grad)
    np.testing.assert_array_equal(grad.cpu().numpy(), eng.seedloss_plain_backward_host(probs, seeds))

    terms = torch.zeros(3, device="cuda")
    eng.expandloss_forward_dev(dp, dl, terms)
    np.testing.assert_array_equal(terms.cpu().numpy(), eng.expandloss_forward_host(probs, labels))
    eng.expandloss_backward_dev(dp, dl, grad)
    np.testing.assert_array_equal(grad.cpu().numpy(), eng.expandloss_backward_host(probs, labels))
    eng.close()


def test_preprocessing_dev_match_host(torch_cuda):
    torch = torch_cuda
    eng = api.Engine(2, 41, 41, M)
    rng = np.random.RandomState(11)
    images = rng.uniform(-120, 140, (2, 3, 53, 47)).astype(np.float32)
    out = torch.empty((2, 41, 41, 3), dtype=torch.uint8, device="cuda")
    eng.prepare_image_dev(torch.from_numpy(images).cuda(), out)
    np.testing.assert_array_equal(out.cpu().numpy(), eng.prepare_image_host(images))

    scores = rng.randn(M, 17, 13).astype(np.float32)
    zo = torch.empty((41, 41, M), device="cuda")
    eng.zoom_scores_dev(torch.from_numpy(scores).cuda(), zo)
    np.testing.assert_array_equal(zo.cpu().numpy(), eng.zoom_scores_host(scores))

    tags = [np.array([3, -2]), np.array([7])]
    cues = [np.array([[0, 3, -1], [1, 40, 5], [2, 0, -3]]), np.array([[7], [20], [30]])]
    flip = [1, 0]
    lab, dense, im = eng.annotation_forward_host(tags, cues, flip=flip, images=images)
    dlab = torch.empty((2, 1, 1, M), device="cuda")
    ddense = torch.empty((2, M, 41, 41), device="cuda")
    dimo = torch.empty(images.shape, device="cuda")
    eng.annotation_forward_dev(tags, cues, dlab, ddense, flip=flip, images=torch.from_numpy(images).cuda(),
                               images_out=dimo)
    np.testing.assert_array_equal(dlab.cpu().numpy(), lab)
    np.testing.assert_array_equal(ddense.cpu().numpy(), dense)
    np.testing.assert_array_equal(dimo.cpu().numpy(), im)
    eng.close()


def test_crf_dev_match_host(torch_cuda):
    torch = torch_cuda
    b, probs = _batch()
    image = b["image"]
    params = api.crf_params(scale_factor=12.0)
    unary = np.log(probs).transpose(0, 2, 3, 1).copy()   # NHWC
    eng = api.Engine(2, 41, 41, M)
    host_a = eng.crf_host(unary, image, params)
    host_b = eng.crf_host(unary, image, params)
    noise = np.abs(host_a - host_b).max()              # float atomics: two passes differ in the last bits
    du, dimg = torch.from_numpy(unary).cuda(), torch.from_numpy(image).cuda()
    out = torch.empty_like(du)
    eng.crf_dev(du, dimg, params, out)
    q = out.cpu().numpy()
    assert noise <= 1e-4 and np.abs(q - host_a).max() <= 1e-4, (noise, np.abs(q - host_a).max())

    labels = torch.empty((2, 41, 41), dtype=torch.int32, device="cuda")
    eng.crf_map_dev(du, dimg, params, labels)
    lm = labels.cpu().numpy()
    top2 = np.sort(q, axis=-1)[..., -2:]
    clear = top2[..., 1] - top2[..., 0] > 1e-4
    assert clear.mean() > 0.5
    np.testing.assert_array_equal(lm[clear], q.argmax(-1)[clear])

    p_host = probs.copy()
    res_host = np.empty_like(probs)
    log_host = eng.crflayer_forward_host(p_host, image, params, result=res_host)
    dp = torch.from_numpy(probs).cuda()
    dlog, dres = torch.empty_like(dp), torch.empty_like(dp)
    eng.crflayer_forward_dev(dp, dimg, params, dlog, result=dres)
    np.testing.assert_array_equal(dp.cpu().numpy(), p_host)                  # the in-place clamp
    assert np.abs(dres.cpu().numpy() - res_host).max() <= 1e-4
    assert np.isfinite(log_host).all()
    eng.close()


def test_retained_marginals_survive_the_other_host_layers(torch_cuda):
    b, probs = _batch()
    labels, cues, image = b["labels"].astype(np.float32), b["cues"], b["image"]
    params = api.crf_params(scale_factor=12.0)
    eng = api.Engine(2, 41, 41, M)
    eng.crflayer_forward_host(probs.copy(), image, params, result=np.empty_like(probs))
    seeds_a = eng.srg_last_crf_host(labels, cues, 0.99, 0.85)
    rng = np.random.RandomState(5)
    preds = rng.randn(*probs.shape).astype(np.float32)
    logs = np.log(probs[:, ::-1].copy())
    eng.softmax_forward_host(preds)
    eng.softmax_backward_host(preds, probs)
    eng.constrainloss_forward_host(probs, logs)
    eng.constrainloss_backward_host(probs, logs)
    eng.seedloss_forward_host(probs, cues)
    eng.seedloss_backward_host(probs, cues)
    eng.expandloss_forward_host(probs, labels)
    eng.expandloss_backward_host(probs, labels)
    eng.annotation_forward_host([np.array([3]), np.array([5])], [np.array([[3], [1], [1]]), np.array([[5], [2], [2]])],
                                images=rng.uniform(0, 255, (2, 3, 41, 41)).astype(np.float32))
    eng.prepare_image_host(rng.uniform(0, 255, (2, 3, 50, 50)).astype(np.float32))
    seeds_b = eng.srg_last_crf_host(labels, cues, 0.99, 0.85)
    np.testing.assert_array_equal(seeds_b, seeds_a)
    eng.close()
