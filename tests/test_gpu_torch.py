"""GPU tests of dsrg_b200.nn, the PyTorch interface of the stage-1 head: each Function against the drop-in Caffe
layer on the same arrays, DSRGHead against the CPU oracles on its own marginals, one mean-field pass per step, the
upstream gradient, side streams, autocast and CUDA-graph capture."""
import numpy as np
import pytest

import fake_caffe

fake_caffe.install()
import pylayers  # noqa: E402
from dsrg_b200 import api, nn, synth  # noqa: E402
from oracle import crf_oracle, loss_oracle, srg_oracle  # noqa: E402

pytestmark = pytest.mark.gpu

B, H, W, HI = 4, 41, 41, 321   # train-s: 41 x 41 score maps of 321 x 321 crops (train-s.prototxt)
MF_TAGS = {"mf_init", "mf_zero", "mf_blur_spatial", "mf_blur_bilateral", "mf_tile", "mf_tile_hybrid"}


def step_inputs(seed, M=21, n=B):
    """Seeded train-s blobs: fc8 whose softmax is synth's probabilities (some below the 1e-4 clamp), the network
    input (mean-subtracted BGR), the (N, 1, 1, M) labels and the cues."""
    batch = synth.make_batch(n, H, W, C=M, cues="cam", image="smooth", start=300 + seed)
    rng = np.random.RandomState(seed)
    fc8 = (np.log(batch["probs"]) + 0.3 * rng.randn(n, M, H, W)).astype(np.float32)
    fc8[0, 5, :4, :4] = -40.0
    images = rng.rand(n, 3, HI, HI) * 255.0 - np.array([104.0, 117.0, 123.0])[None, :, None, None]
    images = ((images + np.roll(images, 1, 2) + np.roll(images, 1, 3)) / 3).astype(np.float32)
    return dict(fc8=fc8, images=images, labels=batch["labels"].reshape(n, 1, 1, M).astype(np.float32),
                cues=batch["cues"].astype(np.float32), probs=batch["probs"].astype(np.float32))


def T(a, torch):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def bits(a):
    a = np.ascontiguousarray(a, np.float32)
    return a.view(np.int32)


def cpu(t):
    t = t.detach()
    return (t.float() if t.is_floating_point() else t).cpu().numpy()   # bf16 has no numpy dtype


def head_step(torch, inp, head=None, fc8=None, autocast=False):
    """One DSRGHead step, forward (under autocast to bf16 if asked) and backward: (loss_seed, loss_constrain, seeds,
    d fc8, probs_c, log_crf)."""
    head = head or nn.DSRGHead()
    fc8 = T(inp["fc8"], torch).requires_grad_() if fc8 is None else fc8
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        ls, lc, seeds = head(fc8, T(inp["images"], torch), T(inp["labels"], torch), T(inp["cues"], torch))
    probs_c, log_crf = lc.grad_fn.saved_tensors   # what ConstrainLoss was fed
    (ls + lc).backward()
    return dict(ls=float(ls.detach()), lc=float(lc.detach()), seeds=cpu(seeds), grad=cpu(fc8.grad),
                probs_c=cpu(probs_c), log_crf=cpu(log_crf))


def clip_safe(probs_c, log_crf):
    """Elements whose ConstrainLoss ratio sits clear of the clip bounds 0.05 and 20 (test_gpu_annot_coco.py)."""
    ratio = np.exp(log_crf.astype(np.float64)) / probs_c
    return (np.abs(ratio - 0.05) > 1e-5) & (np.abs(ratio - 20) > 1e-3)


def assert_steps_close(a, b, grad_rtol=2e-4):
    """Two runs of one step: losses within 1e-4 relative, seed maps differing in at most 1e-3 of the pixels, and
    d fc8 within grad_rtol at the pixels clear of the clip bounds, in the images whose seed maps agree (a differing
    seed changes the image's seed count, hence every gradient of that image)."""
    for k in ("ls", "lc"):
        assert abs(a[k] - b[k]) <= 1e-4 * abs(b[k]), (k, a[k], b[k])
    assert int((a["seeds"] != b["seeds"]).sum()) <= 1e-3 * a["seeds"].size
    same = [i for i in range(a["seeds"].shape[0]) if np.array_equal(a["seeds"][i], b["seeds"][i])]
    assert len(same) * 2 >= a["seeds"].shape[0], same
    safe = (clip_safe(a["probs_c"], a["log_crf"]) & clip_safe(b["probs_c"], b["log_crf"])).all(axis=1, keepdims=True)
    safe = np.broadcast_to(safe, a["grad"].shape)[same]
    ga, gb = a["grad"][same], b["grad"][same]
    np.testing.assert_allclose(ga[safe], gb[safe], rtol=grad_rtol, atol=1e-5 * np.abs(gb).max())


# ---- 1. each function against its drop-in layer on the same arrays ----
def test_softmax_matches_the_layer_bit_for_bit(torch_cuda):
    torch = torch_cuda
    inp = step_inputs(1)
    fc8 = T(inp["fc8"], torch).requires_grad_()
    probs = nn.softmax(fc8)
    layer, bottom, top = fake_caffe.run_layer(pylayers.SoftmaxLayer, [inp["fc8"]])
    assert np.array_equal(bits(cpu(probs)), bits(top[0].data))
    diff = np.random.RandomState(5).randn(*inp["fc8"].shape).astype(np.float32)
    top[0].diff[...] = diff
    layer.backward(top, [True], bottom)
    g, = torch.autograd.grad(probs, fc8, T(diff, torch))
    assert np.array_equal(bits(cpu(g)), bits(bottom[0].diff))


def test_softmax_refuses_more_than_32_labels(torch_cuda):
    torch = torch_cuda
    with pytest.raises(api.DsrgError, match="at most 32 labels"):
        nn.softmax(torch.zeros(2, 33, 9, 9, device="cuda"))


def _assert_loss_close(got, want):
    got, want = np.float32(float(got.detach()) if hasattr(got, "detach") else got), np.float32(want)
    assert abs(got - want) <= np.spacing(abs(want)), (got, want)


@pytest.mark.parametrize("which", ["balanced", "seed", "expand"])
def test_seed_losses_match_the_layers(torch_cuda, which):
    torch = torch_cuda
    inp = step_inputs(2)
    probs = np.maximum(inp["probs"], np.float32(1e-4))
    seeds = inp["cues"].copy()
    seeds[1, 1:] = 0   # one image without foreground seeds
    fn, cls, second = {"balanced": (nn.balanced_seed_loss, pylayers.BalancedSeedLossLayer, seeds),
                       "seed": (nn.seed_loss, pylayers.SeedLossLayer, inp["cues"]),
                       "expand": (nn.expand_loss, pylayers.ExpandLossLayer, inp["labels"])}[which]
    p = T(probs, torch).requires_grad_()
    loss = fn(p, T(second, torch))
    layer, bottom, top = fake_caffe.run_layer(cls, [probs, second])
    layer.backward(top, [True, False], bottom)
    _assert_loss_close(loss, top[0].data[0])
    g, = torch.autograd.grad(loss, p)
    assert np.array_equal(bits(cpu(g)), bits(bottom[0].diff))


def test_constrain_loss_matches_the_layer(torch_cuda):
    torch = torch_cuda
    inp = step_inputs(3)
    probs = np.maximum(inp["probs"], np.float32(1e-4))
    rng = np.random.RandomState(3)
    logs = np.log(loss_oracle.softmax_layer_forward(np.log(probs) + rng.randn(*probs.shape))).astype(np.float32)
    p, lg = T(probs, torch).requires_grad_(), T(logs, torch).requires_grad_()
    loss = nn.constrain_loss(p, lg)
    layer, bottom, top = fake_caffe.run_layer(pylayers.ConstrainLossLayer, [probs, logs])
    layer.backward(top, [True, True], bottom)
    _assert_loss_close(loss, top[0].data[0])
    gp, gl = torch.autograd.grad(loss, (p, lg))
    assert np.array_equal(bits(cpu(gp)), bits(bottom[0].diff))
    assert np.array_equal(bits(cpu(gl)), bits(bottom[1].diff))


def test_crf_layer_clamps_a_copy(torch_cuda):
    torch = torch_cuda
    inp = step_inputs(4)
    probs = inp["probs"].copy()
    probs[0, 5, :4, :4] = 1e-6
    p = T(probs, torch)
    log_crf, probs_c = nn.crf_layer(p, T(inp["images"], torch))
    assert np.array_equal(cpu(probs_c), np.maximum(probs, np.float32(1e-4)))
    assert np.array_equal(cpu(p), probs)   # the caller's tensor is not written
    want = crf_oracle.refinement(probs.copy(), inp["images"], 12.0)
    assert np.abs(np.exp(cpu(log_crf)) - want).max() <= 1e-4


# ---- 2. dsrg_crflayer_backward_dev on given arrays ----
@pytest.mark.parametrize("shape", [(3, 7, 17, 23), (4, 21, 41, 41), (1, 81, 5, 3)])
def test_crflayer_backward_is_numpy_float32(torch_cuda, shape):
    torch = torch_cuda
    rng = np.random.RandomState(sum(shape))
    result = rng.rand(*shape).astype(np.float32)
    diff = (rng.randn(*shape) * 10.0 ** rng.randint(-30, 30, shape)).astype(np.float32)
    flat_r, flat_d = result.reshape(-1), diff.reshape(-1)
    flat_r[:6] = [0.0, 1.0, 1e-8, np.nextafter(np.float32(1), np.float32(0)), 2.0, 0.5]
    flat_d[:6] = [1e-45, -3e38, np.inf, 1.5, -0.0, 3e-39]   # no NaN: its payload is the platform's
    eng = api.Engine(shape[0], shape[2], shape[3], shape[1])
    grad = torch.empty(shape, device="cuda")
    eng.crflayer_backward_dev(T(result, torch), T(diff, torch), grad)
    torch.cuda.synchronize()
    with np.errstate(all="ignore"):
        want = (1 - result) * diff
    assert want.dtype == np.float32
    assert np.array_equal(bits(cpu(grad)), bits(want))
    eng.close()


# ---- 3. DSRGHead against the oracles on its own marginals ----
def test_head_against_the_oracles(torch_cuda):
    torch = torch_cuda
    inp = step_inputs(6)
    fc8 = T(inp["fc8"], torch).requires_grad_()
    ls, lc, seeds = nn.DSRGHead()(fc8, T(inp["images"], torch), T(inp["labels"], torch), T(inp["cues"], torch))
    r = crf_oracle.renormalise(nn.cached_engine(21, H, W, fc8.device.index).crf_last_marginals_host(B))
    probs_c, log_crf = (cpu(t).astype(np.float64) for t in lc.grad_fn.saved_tensors)
    (ls + lc).backward()
    seeds = cpu(seeds)
    for b in range(B):
        assert np.array_equal(seeds[b], srg_oracle.srg_closed_form(inp["labels"][b, 0, 0], inp["cues"][b], r[b],
                                                                   0.99, 0.85))
    assert np.abs(np.exp(log_crf) - r).max() <= 1e-4
    assert np.array_equal(probs_c, np.maximum(cpu(nn.softmax(fc8)), np.float32(1e-4)))
    _assert_loss_close(ls, loss_oracle.balanced_seed_loss(probs_c, seeds))
    assert abs(float(lc.detach()) - loss_oracle.constrain_loss(probs_c, log_crf)) <= 2e-5 * abs(float(lc.detach()))
    # d loss / d fc8: softmax backward of (seed-loss gradient + constrain gradient + (1 - r) x constrain log-gradient)
    gp, gl = loss_oracle.constrain_loss_grad(probs_c, log_crf)
    top = loss_oracle.balanced_seed_loss_grad(probs_c, seeds) + gp + (1 - r) * gl
    want = loss_oracle.softmax_layer_backward(inp["fc8"], top)
    safe = np.broadcast_to(clip_safe(probs_c, log_crf).all(axis=1, keepdims=True), want.shape)
    got = cpu(fc8.grad)
    np.testing.assert_allclose(got[safe], want[safe], rtol=2e-4, atol=1e-5 * np.abs(want).max())


def test_81_labels_composed_against_the_oracles(torch_cuda):
    """At 81 labels (COCO) softmax refuses; the other functions compose train-s's head on given probabilities."""
    torch = torch_cuda
    inp = step_inputs(7, M=81)
    probs = inp["probs"].copy()
    probs[0, 5, :4, :4] = 1e-6
    p = T(probs, torch).requires_grad_()
    images, labels, cues = (T(inp[k], torch) for k in ("images", "labels", "cues"))
    log_crf, probs_c = nn.crf_layer(p, images)
    seeds = nn.dsrg_seeds(labels, probs_c, cues, images)
    r = crf_oracle.renormalise(nn.cached_engine(81, H, W, p.device.index).crf_last_marginals_host(B))
    ls, lc = nn.balanced_seed_loss(probs_c, seeds), nn.constrain_loss(probs_c, log_crf)
    (ls + lc).backward()
    seeds, pc, lg = cpu(seeds), cpu(probs_c).astype(np.float64), cpu(log_crf).astype(np.float64)
    assert np.array_equal(cpu(probs_c), np.maximum(probs, np.float32(1e-4)))
    for b in range(B):   # the seeds grow on the marginals of dsrg_seeds' own pass
        assert np.array_equal(seeds[b], srg_oracle.srg_closed_form(inp["labels"][b, 0, 0], inp["cues"][b], r[b],
                                                                   0.99, 0.85))
    assert np.abs(np.exp(lg) - r).max() <= 1e-4
    rc = np.exp(lg)
    gp, gl = loss_oracle.constrain_loss_grad(pc, lg)
    want = loss_oracle.balanced_seed_loss_grad(pc, seeds) + gp + (1 - rc) * gl
    safe = clip_safe(pc, lg)
    got = cpu(p.grad)
    np.testing.assert_allclose(got[safe], want[safe], rtol=2e-4, atol=1e-5 * np.abs(want).max())


# ---- 4. one mean-field pass per step ----
def _mf_counts(eng):
    return {k: n for k, (_, n) in eng.profile_read().items() if k in MF_TAGS}


def test_head_runs_one_mean_field_pass(torch_cuda):
    torch = torch_cuda
    inp = step_inputs(8)
    fc8, images, labels, cues = (T(inp[k], torch) for k in ("fc8", "images", "labels", "cues"))
    head = nn.DSRGHead()
    head(fc8, images, labels, cues)
    eng = nn.cached_engine(21, H, W, fc8.device.index)
    eng.profile(True)
    try:
        eng.profile_read()
        probs = nn.softmax(fc8)
        pc = probs.clone()
        image = torch.empty((B, H, W, 3), dtype=torch.uint8, device="cuda")
        eng.prepare_image_dev(images, image)
        eng.crflayer_forward_dev(pc, image, api.crf_params(12.0), torch.empty_like(pc), torch.empty_like(pc))
        one = _mf_counts(eng)
        assert one.get("mf_tile", 0) == 11 and one.get("mf_blur_bilateral", 0) > 0, one
        head(fc8, images, labels, cues)
        assert _mf_counts(eng) == one
        log_crf, probs_c = nn.crf_layer(probs, images)
        nn.dsrg_seeds(labels, probs_c, cues, images)
        assert _mf_counts(eng) == {k: 2 * n for k, n in one.items()}
    finally:
        eng.profile(False)


# ---- 5. the upstream gradient ----
def test_upstream_gradient_is_honoured(torch_cuda):
    torch = torch_cuda
    inp = step_inputs(9)
    fc8 = T(inp["fc8"], torch).requires_grad_()
    ls, lc, _ = nn.DSRGHead()(fc8, T(inp["images"], torch), T(inp["labels"], torch), T(inp["cues"], torch))
    loss = ls + lc
    g1, = torch.autograd.grad(loss, fc8, retain_graph=True)
    g2, = torch.autograd.grad(1024 * loss, fc8, retain_graph=True)
    assert torch.equal(g2, 1024 * g1)
    assert float(g1.abs().max()) > 0
    opt = torch.optim.SGD([fc8], lr=0.0)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 16)
    scaler.scale(loss).backward()
    scaler.unscale_(opt)
    assert torch.equal(fc8.grad, g1)
    scaler.step(opt)
    scaler.update()


# ---- 6. streams, autocast, capture ----
def test_side_stream_step_matches_the_default_stream(torch_cuda):
    torch = torch_cuda
    inp = step_inputs(10)
    head = nn.DSRGHead()
    ref = head_step(torch, inp, head)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        got = head_step(torch, inp, head)
    torch.cuda.current_stream().wait_stream(side)
    assert_steps_close(got, ref)


def test_bf16_under_autocast_matches_float32(torch_cuda):
    torch = torch_cuda
    inp = step_inputs(11)
    fc8_bf = T(inp["fc8"], torch).to(torch.bfloat16)
    ref = head_step(torch, dict(inp, fc8=cpu(fc8_bf.float())))
    x = fc8_bf.clone().requires_grad_()
    got = head_step(torch, inp, fc8=x, autocast=True)
    assert x.grad.dtype == torch.bfloat16
    # the gradient of a bf16 input is rounded to bf16 (relative error up to 2^-9)
    assert_steps_close(got, ref, grad_rtol=2e-4 + 2.0 ** -8)


def test_step_captured_in_a_cuda_graph(torch_cuda):
    torch = torch_cuda
    head = nn.DSRGHead()
    a, b = step_inputs(12), step_inputs(13)
    fc8 = T(a["fc8"], torch).requires_grad_()
    images, labels, cues = (T(a[k], torch) for k in ("images", "labels", "cues"))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):   # warm-up: engines, graphs of the engine's own passes
        for _ in range(3):
            fc8.grad = None
            ls, lc, _ = head(fc8, images, labels, cues)
            (ls + lc).backward()
    del ls, lc   # no autograd node of the warm-up may outlive it into the capture
    torch.cuda.current_stream().wait_stream(side)
    fc8.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        s_ls, s_lc, s_seeds = head(fc8, images, labels, cues)
        s_pc, s_lg = s_lc.grad_fn.saved_tensors
        (s_ls + s_lc).backward()
    with torch.no_grad():
        for t, k in ((fc8, "fc8"), (images, "images"), (labels, "labels"), (cues, "cues")):
            t.copy_(T(b[k], torch))
    graph.replay()
    torch.cuda.synchronize()
    got = dict(ls=float(s_ls.detach()), lc=float(s_lc.detach()), seeds=cpu(s_seeds), grad=cpu(fc8.grad),
               probs_c=cpu(s_pc), log_crf=cpu(s_lg))
    ref = head_step(torch, b, head)
    assert not np.array_equal(got["seeds"], head_step(torch, a, head)["seeds"])   # the replay saw the new inputs
    assert_steps_close(got, ref)
    graph.replay()   # and again, on the same inputs
    torch.cuda.synchronize()
    assert abs(float(s_ls.detach()) - ref["ls"]) <= 1e-4 * abs(ref["ls"])


# ---- the two new entry points' prologue: batch range, NULL pointers, the retained pass ----
def test_new_entry_points_refuse_bad_arguments(torch_cuda):
    import ctypes as C
    from dsrg_b200 import _lib
    torch = torch_cuda
    L, eng = _lib.lib(), api.Engine(2, 9, 11, 5)
    e, s = C.c_void_p(eng.h), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    a, b, c = (C.c_void_p(torch.rand(2, 5, 9, 11, device="cuda").data_ptr()) for _ in range(3))
    lab = C.c_void_p(torch.ones(2, 5, device="cuda").data_ptr())
    for B in (0, 3):
        assert L.dsrg_crflayer_backward_dev(e, a, b, B, c, s) == _lib.E_INVALID
        assert L.dsrg_srg_last_crf_dev(e, lab, a, B, 0.99, 0.85, c, s) == _lib.E_INVALID
    for args in ((None, b, c), (a, None, c), (a, b, None)):
        assert L.dsrg_crflayer_backward_dev(e, args[0], args[1], 2, args[2], s) == _lib.E_INVALID
        assert L.dsrg_srg_last_crf_dev(e, args[0], args[1], 2, 0.99, 0.85, args[2], s) == _lib.E_INVALID
    assert L.dsrg_crflayer_backward_dev(None, a, b, 2, c, s) == _lib.E_INVALID
    # no mean-field pass held yet, then one over 2 images: only B = 2 may read it
    assert L.dsrg_srg_last_crf_dev(e, lab, a, 2, 0.99, 0.85, c, s) == _lib.E_STATE
    image = torch.zeros(2, 9, 11, 3, dtype=torch.uint8, device="cuda")
    probs = torch.full((2, 5, 9, 11), 0.2, device="cuda")
    eng.crflayer_forward_dev(probs, image, api.crf_params(12.0), torch.empty_like(probs))
    assert L.dsrg_srg_last_crf_dev(e, lab, a, 1, 0.99, 0.85, c, s) == _lib.E_STATE
    assert L.dsrg_srg_last_crf_dev(e, lab, a, 2, 0.99, 0.85, c, s) == _lib.OK
    torch.cuda.synchronize()
    eng.close()


def test_host_twin_argument_order_is_refused(torch_cuda):
    """The batch size of the two new entry points follows their arrays.  A call made with plain ints in the order of
    dsrg_srg_last_crf_host / dsrg_crflayer_forward_dev (B second) lands a device pointer in the batch argument; its low
    32 bits (a multiple of the allocator's 512-byte alignment) are outside [1, max_batch], so the batch-range check
    refuses the call before anything is read or written."""
    from dsrg_b200 import _lib
    torch = torch_cuda
    L, eng = _lib.lib(), api.Engine(4, 9, 11, 5)
    s = torch.cuda.current_stream().cuda_stream
    lab = torch.ones(4, 5, device="cuda")
    t = [torch.rand(4, 5, 9, 11, device="cuda") for _ in range(3)]
    eng.crflayer_forward_dev(t[0].clone(), torch.zeros(4, 9, 11, 3, dtype=torch.uint8, device="cuda"),
                             api.crf_params(12.0), t[1])
    torch.cuda.synchronize()
    before = [x.clone() for x in t]
    for B in (1, 4):
        assert L.dsrg_srg_last_crf_dev(eng.h, B, lab.data_ptr(), t[0].data_ptr(), 0.99, 0.85, t[2].data_ptr(),
                                       s) == _lib.E_INVALID
        assert "batch" in L.dsrg_last_error().decode()
        assert L.dsrg_crflayer_backward_dev(eng.h, B, t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(),
                                            s) == _lib.E_INVALID
        assert "batch" in L.dsrg_last_error().decode()
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(t, before))
    eng.close()
