"""PyTorch interface of the stage-1 DSRG head: autograd Functions over the C ABI, on the device.

Every layer of train-s.prototxt's head (:746-812, Softmax -> CRF -> DSRG -> BalancedSeedLoss + ConstrainLoss) is a
``torch.autograd.Function`` whose forward and backward are the library's ``*_dev`` entry points, queued on the
current stream of the inputs' device.  Nothing is read back to the host and nothing synchronises it, so a training
step can be captured in a ``torch.cuda.CUDAGraph``.  Torch itself only allocates, makes the defensive copy of the
probabilities the CRF clamps in place, multiplies by the upstream gradient and forms the scalar losses from the
device-resident sums.

Semantics follow the drop-in Caffe layers (dsrg_b200/dropin/pylayers):

* ``crf_layer`` returns ``(log_crf, probs_c)``.  ``probs_c`` is ``probs`` clamped at 1e-4, the blob every later
  layer of train-s reads (CRFLayer clamps its bottom in place and Caffe's split tops share it); its gradient passes
  the clamp unchanged, as Caffe's summed diffs do.  The caller's ``probs`` is never written.
* The losses' backward passes multiply by the upstream gradient (the loss scale under ``GradScaler``), which the
  Caffe layers ignore.
* ``DSRGHead`` runs one mean-field pass per step: the DSRG seeds grow on the marginals the CRF layer has just
  computed (``dsrg_srg_last_crf_dev``), where the composition ``crf_layer`` + ``dsrg_seeds`` runs two.
* ``dense_crf`` is the CRF alone with its exact gradient (DenseCRF::gradient, densecrf.cpp:238-297): the mean field
  run backwards to the unaries and, when they are tensors, the two Potts weights.  ``crf_layer`` and ``DSRGHead``
  keep the reference's ``(1 - result) * top_diff``.

Engines are cached per (labels, height, width, device) and recreated when a larger batch arrives.  Autograd runs
a backward on the forward's stream and device, so one engine is never driven from two threads at once.

A step captured in a CUDA graph uses the cached engine's buffers.  Two rules follow:
* Replacing the engine frees them.  A captured step must not be replayed once a larger batch has reached the same
  (labels, height, width, device); a larger batch during a capture raises RuntimeError.
* The engine orders its eager calls across streams, but a graph replay leaves no mark it can wait for.  Replays and
  eager steps on the same engine must run on one stream, or be ordered by the caller.
"""
import math
import threading

import torch

from . import api

MAX_LABELS = 255   # DSRG_MAX_LABELS_WIDE: Softmax alone stops at 32 (DSRG_MAX_LABELS) and says so with DsrgError
_MEAN_PIXEL = (104.0, 117.0, 123.0)   # pylayers.py:72, :317

_ENGINES = {}
_ENGINES_LOCK = threading.Lock()


def cached_engine(M, H, W, device):
    """The engine this module uses for M labels of H x W maps on CUDA device index `device`, or None if none has
    been created yet (for introspection: profiling, the retained marginals)."""
    return _ENGINES.get((int(M), int(H), int(W), int(device)))


def _engine(B, M, H, W, device):
    key = (int(M), int(H), int(W), int(device))
    with _ENGINES_LOCK:
        eng = _ENGINES.get(key)
        if eng is None or eng.max_batch < B:
            if eng is not None:
                # the old engine's buffers go: a CUDA graph captured on it must not be replayed afterwards, and
                # inside a capture the engine can neither be freed nor created
                if torch.cuda.is_current_stream_capturing():
                    raise RuntimeError("a batch of %d reached the engine for %d labels of %dx%d maps (created for %d) "
                                       "during CUDA-graph capture: run a step with the largest batch before capturing"
                                       % (B, M, H, W, eng.max_batch))
                eng.close()   # waits for the device
            eng = _ENGINES[key] = api.Engine(int(B), int(H), int(W), int(M), device=int(device))
        return eng


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _tensor(t, name, ndim):
    if not isinstance(t, torch.Tensor):
        raise ValueError("%s must be a torch.Tensor, not %s" % (name, type(t).__name__))
    if t.dtype != torch.float32:
        raise ValueError("%s must be float32 (got %s)" % (name, t.dtype))
    if t.dim() != ndim:
        raise ValueError("%s must have %d dimensions (got shape %s)" % (name, ndim, tuple(t.shape)))


def _maps(t, name="probs"):
    """(N, M, H, W) float32 tensor with 1 <= M <= 255, made contiguous.  Its companions are checked against it
    (same device), and then the device itself (_cuda), so that every shape error is found first."""
    _tensor(t, name, 4)
    if t.shape[1] > MAX_LABELS or min(t.shape) < 1:
        raise ValueError("%s must be (N, M, H, W) with 1 <= M <= %d (got shape %s)"
                         % (name, MAX_LABELS, tuple(t.shape)))
    return t.contiguous()


def _cuda(t, name="probs"):
    if not t.is_cuda:
        raise ValueError("%s must be a CUDA tensor (got device %s)" % (name, t.device))
    return t


def _like(t, ref, name):
    """A second (N, M, H, W) array of the same shape and device as `ref`."""
    _tensor(t, name, 4)
    if t.shape != ref.shape or t.device != ref.device:
        raise ValueError("%s must have the shape %s on %s (got %s on %s)" % (name, tuple(ref.shape), ref.device,
                                                                          tuple(t.shape), t.device))
    return t.contiguous()


def _labels(t, ref):
    """Image-level labels (N, 1, 1, M) or (N, M) -> contiguous (N, M)."""
    N, M = ref.shape[:2]
    if not isinstance(t, torch.Tensor) or t.dim() not in (2, 4):
        raise ValueError("labels must be an (N, 1, 1, M) or (N, M) tensor")
    _tensor(t, "labels", t.dim())
    if tuple(t.shape) not in ((N, M), (N, 1, 1, M)) or t.device != ref.device:
        raise ValueError("labels must be (%d, 1, 1, %d) or (%d, %d) on %s (got %s on %s)"
                         % (N, M, N, M, ref.device, tuple(t.shape), t.device))
    return t.contiguous().view(N, M)


def _images(t, ref):
    """The network input (N, 3, Hi, Wi), mean-subtracted BGR."""
    _tensor(t, "images", 4)
    if t.shape[0] != ref.shape[0] or t.shape[1] != 3 or t.device != ref.device:
        raise ValueError("images must be (%d, 3, Hi, Wi) on %s (got %s on %s)" % (ref.shape[0], ref.device,
                                                                              tuple(t.shape), t.device))
    return t.contiguous()


def _engine_for(t):
    N, M, H, W = t.shape
    return _engine(N, M, H, W, t.device.index)


def _crf_image(eng, images, probs):
    """pylayers.py:70-75 + the ubyte cast of CRF.py:32: the network input zoomed to the map size."""
    N, _, H, W = probs.shape
    image = torch.empty((N, H, W, 3), dtype=torch.uint8, device=probs.device)
    return eng.prepare_image_dev(images, image, _MEAN_PIXEL, stream=_stream(probs))


def _crf_forward(eng, probs, images, scale_factor):
    """CRFLayer.forward on a copy of probs: -> (log_crf, probs_c, result)."""
    s = _stream(probs)
    probs_c = probs.clone()   # clamped in place by the pass: the caller's tensor stays as it was
    image = _crf_image(eng, images, probs)
    log_crf, result = torch.empty_like(probs), torch.empty_like(probs)
    eng.crflayer_forward_dev(probs_c, image, api.crf_params(scale_factor), log_crf, result, stream=s)
    return log_crf, probs_c, result


def _crf_backward(result, g_log, g_probs_c):
    """d probs = (1 - result) * d log_crf + d probs_c (the clamp passes the gradient unchanged)."""
    grad = None
    if g_log is not None:
        g_log = g_log.contiguous()
        grad = torch.empty_like(result)
        _engine_for(result).crflayer_backward_dev(result, g_log, grad, stream=_stream(result))
    if g_probs_c is not None:
        grad = g_probs_c.clone() if grad is None else grad.add_(g_probs_c)
    return grad


def _scaled(grad, g):
    """A loss gradient times the upstream gradient (a 0-dim device tensor: 1, or the loss scale)."""
    return grad.mul_(g.to(grad.dtype))


_fwd = torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
_bwd = torch.amp.custom_bwd(device_type="cuda")


class _Softmax(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, fc8):
        x = _cuda(_maps(fc8, "fc8"), "fc8")
        probs = torch.empty_like(x)
        _engine_for(x).softmax_forward_dev(x, probs, stream=_stream(x))
        ctx.save_for_backward(x)
        return probs

    @staticmethod
    @_bwd
    def backward(ctx, g):
        x, = ctx.saved_tensors
        grad = torch.empty_like(x)
        _engine_for(x).softmax_backward_dev(x, g.contiguous(), grad, stream=_stream(x))
        return grad


class _CrfLayer(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, probs, images, scale_factor):
        probs = _maps(probs)
        images = _images(images, probs)
        _cuda(probs)
        log_crf, probs_c, result = _crf_forward(_engine_for(probs), probs, images, scale_factor)
        ctx.save_for_backward(result)
        return log_crf, probs_c

    @staticmethod
    @_bwd
    def backward(ctx, g_log, g_probs_c):
        result, = ctx.saved_tensors
        return _crf_backward(result, g_log, g_probs_c), None, None


class _DsrgSeeds(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, labels, probs, cues, images, th1, th2, scale_factor):
        probs = _maps(probs)
        labels, cues, images = _labels(labels, probs), _like(cues, probs, "cues"), _images(images, probs)
        _cuda(probs)
        eng = _engine_for(probs)
        s = _stream(probs)
        p = probs.clone()   # refinement() clamps its input in place (pylayers.py:312)
        image = _crf_image(eng, images, probs)
        seeds = torch.empty_like(probs)
        eng.dsrg_forward_dev(labels, p, cues, image, api.crf_params(scale_factor), th1, th2, seeds, stream=s)
        return seeds

    @staticmethod
    @_bwd
    def backward(ctx, g):
        return None, g, None, None, None, None, None   # straight through to probs (pylayers.py:307-308)


class _CrfDsrg(torch.autograd.Function):
    """CRFLayer and DSRGLayer of train-s on one mean-field pass: the seeds grow on the marginals the CRF layer
    leaves in the engine.  -> (log_crf, probs_c, seeds); the seeds carry no gradient."""

    @staticmethod
    @_fwd
    def forward(ctx, probs, images, labels, cues, th1, th2, scale_factor):
        probs = _maps(probs)
        images, labels, cues = _images(images, probs), _labels(labels, probs), _like(cues, probs, "cues")
        _cuda(probs)
        eng = _engine_for(probs)
        log_crf, probs_c, result = _crf_forward(eng, probs, images, scale_factor)
        seeds = torch.empty_like(probs)
        eng.srg_last_crf_dev(labels, cues, th1, th2, seeds, stream=_stream(probs))
        ctx.save_for_backward(result)
        ctx.mark_non_differentiable(seeds)
        return log_crf, probs_c, seeds

    @staticmethod
    @_bwd
    def backward(ctx, g_log, g_probs_c, _g_seeds):
        result, = ctx.saved_tensors
        return _crf_backward(result, g_log, g_probs_c), None, None, None, None, None, None


class _BalancedSeedLoss(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, probs, seeds):
        probs = _maps(probs)
        seeds = _like(seeds, probs, "seeds")
        _cuda(probs)
        terms = torch.empty(2, dtype=torch.float32, device=probs.device)
        _engine_for(probs).seedloss_forward_dev(probs, seeds, terms, stream=_stream(probs))
        ctx.save_for_backward(probs, seeds)
        t = terms.double()   # the drop-in forms -(t0 + t1) / N in Python floats
        return (-(t[0] + t[1]) / probs.shape[0]).float()

    @staticmethod
    @_bwd
    def backward(ctx, g):
        probs, seeds = ctx.saved_tensors
        grad = torch.empty_like(probs)
        _engine_for(probs).seedloss_backward_dev(probs, seeds, grad, n_global=probs.shape[0], top_diff=1.0,
                                                 stream=_stream(probs))
        return _scaled(grad, g), None


class _ConstrainLoss(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, probs, log_crf):
        probs = _maps(probs)
        log_crf = _like(log_crf, probs, "log_crf")
        _cuda(probs)
        loss = torch.empty(1, dtype=torch.float32, device=probs.device)
        _engine_for(probs).constrainloss_forward_dev(probs, log_crf, loss, stream=_stream(probs))
        ctx.save_for_backward(probs, log_crf)
        return loss.view(())

    @staticmethod
    @_bwd
    def backward(ctx, g):
        probs, log_crf = ctx.saved_tensors
        gp, gl = torch.empty_like(probs), torch.empty_like(probs)
        _engine_for(probs).constrainloss_backward_dev(probs, log_crf, gp, gl, stream=_stream(probs))
        return _scaled(gp, g), _scaled(gl, g)


class _SeedLoss(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, probs, seeds):
        probs = _maps(probs)
        seeds = _like(seeds, probs, "seeds")
        _cuda(probs)
        terms = torch.empty(1, dtype=torch.float32, device=probs.device)
        _engine_for(probs).seedloss_plain_forward_dev(probs, seeds, terms, stream=_stream(probs))
        ctx.save_for_backward(probs, seeds)
        return (-terms.double()[0] / probs.shape[0]).float()

    @staticmethod
    @_bwd
    def backward(ctx, g):
        probs, seeds = ctx.saved_tensors
        grad = torch.empty_like(probs)
        _engine_for(probs).seedloss_plain_backward_dev(probs, seeds, grad, n_global=probs.shape[0],
                                                       stream=_stream(probs))
        return _scaled(grad, g), None


class _ExpandLoss(torch.autograd.Function):
    @staticmethod
    @_fwd
    def forward(ctx, probs, labels, q_fg, q_bg):
        probs = _maps(probs)
        labels = _labels(labels, probs)
        _cuda(probs)
        terms = torch.empty(3, dtype=torch.float32, device=probs.device)
        _engine_for(probs).expandloss_forward_dev(probs, labels, terms, q_fg, q_bg, stream=_stream(probs))
        ctx.save_for_backward(probs, labels)
        ctx.q = (q_fg, q_bg)
        t = terms.double()
        return (-(t[0] + t[1] + t[2]) / probs.shape[0]).float()

    @staticmethod
    @_bwd
    def backward(ctx, g):
        probs, labels = ctx.saved_tensors
        grad = torch.empty_like(probs)
        _engine_for(probs).expandloss_backward_dev(probs, labels, grad, n_global=probs.shape[0], q_fg=ctx.q[0],
                                                   q_bg=ctx.q[1], stream=_stream(probs))
        return _scaled(grad, g), None, None, None


FUSED_LABELS = 32   # DSRG_MAX_LABELS: the CRF gradient runs on the fused kernels only
_POTTS_DEFAULT = (10.0, 3.0)   # CRF.py:31-32: w1 (bilateral), w2 (spatial)


def _potts_weight(w, name, ref):
    if w is None:
        return None
    if not isinstance(w, torch.Tensor) or w.dim() != 0 or not w.is_floating_point() or w.device != ref.device:
        raise ValueError("%s must be None or a 0-dim floating-point tensor on %s (got %r)"
                         % (name, ref.device, w if not isinstance(w, torch.Tensor) else (w.dtype, tuple(w.shape), w.device)))
    return w


def _potts_tensor(w1, w2, ref):
    """The device {w1, w2} the kernels read in place of params' weights (a None one is CRF()'s), or None for both."""
    if w1 is None and w2 is None:
        return None
    potts = torch.empty(2, dtype=torch.float32, device=ref.device)
    for i, (w, d) in enumerate(zip((w1, w2), _POTTS_DEFAULT)):
        if w is None:
            potts[i].fill_(d)
        else:
            potts[i].copy_(w.detach())
    return potts


def _train_entry(wide, feat, compat, theta):
    """The Engine methods (forward, backward) of one differentiable CRF call: the label-chunked path (wide) or the
    fused one, on caller-given features (feat) or the image, with the matrices (compat) or the Potts weights, and
    with a given theta (on the image path its backward also writes dL/dtheta; the features carry theta_sp's)."""
    if feat:
        return (("crf_forward_train_wide_feat_dev", "crf_backward_wide_feat_dev") if wide
                else ("crf_forward_train_feat_dev", "crf_backward_feat_dev"))
    if wide:
        return "crf_forward_train_wide_dev", "crf_backward_wide_theta_dev" if theta else "crf_backward_wide_dev"
    if compat:
        return "crf_forward_train_compat_dev", "crf_backward_compat_theta_dev" if theta else "crf_backward_compat_dev"
    return "crf_forward_train_dev", "crf_backward_theta_dev" if theta else "crf_backward_dev"


class _DenseCrfTrain(torch.autograd.Function):
    """dense_crf / dense_crf_wide on the image's lattice or on caller-given features (x, feat), with the Potts weights
    (w1, w2) or the matrices (compat (2, M, M) {mu_bi, mu_sp}), and learnable bandwidths theta_bi (5,) / theta_sp (2,)
    whose values params already carries.  wide: the label-chunked entry points above 32 labels."""

    @staticmethod
    @_fwd
    def forward(ctx, unary, x, w1, w2, compat, theta_bi, theta_sp, params, wide, feat):
        fwd, ctx.bwd = _train_entry(wide, feat, compat is not None, theta_bi is not None or theta_sp is not None)
        q_hist = torch.empty((params.n_iters + 1,) + tuple(unary.shape), dtype=torch.float32, device=unary.device)
        potts = _potts_tensor(w1, w2, unary)
        weights = {"potts": potts} if compat is None else {"compat": compat}
        getattr(_engine_for(unary), fwd)(unary, x, params, q_hist=q_hist, stream=_stream(unary), **weights)
        ctx.save_for_backward(q_hist, x, potts, compat)
        ctx.params, ctx.feat = params, feat
        ctx.theta = [(t.device, t.dtype) if t is not None else None for t in (theta_bi, theta_sp)]
        return q_hist[params.n_iters].clone()

    @staticmethod
    @_bwd
    def backward(ctx, g):
        q_hist, x, potts, compat = ctx.saved_tensors
        need = ctx.needs_input_grad
        B, f32 = q_hist.shape[1], {"dtype": torch.float32, "device": q_hist.device}
        grad_u = torch.empty(q_hist.shape[1:], **f32)
        # the backward's optional arguments, by keyword
        if compat is None:
            kw = {"potts": potts, "grad_potts": None}
            if potts is not None and (need[2] or need[3]):
                kw["grad_potts"] = torch.empty((B, 2), **f32)
        else:
            kw = {"compat": compat, "grad_compat": torch.empty((B, 2) + compat.shape[1:], **f32) if need[4] else None}
        if ctx.feat:
            kw["grad_features"] = torch.empty_like(x)
            if ctx.theta[1] is not None and need[6]:
                kw["grad_theta_sp"] = torch.empty((B, 2), **f32)
        elif ctx.theta != [None, None]:   # a given theta's backward writes dL/dtheta whether or not it is needed
            kw["grad_theta"] = torch.empty((B, 7), **f32)
        getattr(_engine_for(grad_u), ctx.bwd)(q_hist, x, ctx.params, grad_q=g.contiguous(), grad_unary=grad_u,
                                               stream=_stream(grad_u), **kw)
        grad_potts, grad_c = kw.get("grad_potts"), kw.get("grad_compat")
        gw1 = grad_potts[:, 0].sum() if grad_potts is not None and need[2] else None
        gw2 = grad_potts[:, 1].sum() if grad_potts is not None and need[3] else None
        gc = None if grad_c is None else grad_c.sum(0)
        gt = (None, None)
        if "grad_theta" in kw:
            gt = kw["grad_theta"].sum(0)
            gt = (gt[0:5], gt[5:7])
        elif "grad_theta_sp" in kw:
            gt = (None, kw["grad_theta_sp"].sum(0))
        gt = [t.to(spec[0], spec[1]) if t is not None and spec is not None and n else None
              for t, spec, n in zip(gt, ctx.theta, need[5:7])]
        gx = kw["grad_features"] if ctx.feat and need[1] else None
        return grad_u, gx, gw1, gw2, gc, gt[0], gt[1], None, None, None


def _features(t, N, H, W, device):
    """The bilateral features (N, 5, H, W) float32 on `device`, made contiguous."""
    if (not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or tuple(t.shape) != (N, 5, H, W)
            or t.device != device):
        raise ValueError("features_bi must be a (%d, 5, %d, %d) float32 tensor on %s (got %r)"
                         % (N, H, W, device,
                            t if not isinstance(t, torch.Tensor) else (t.dtype, tuple(t.shape), t.device)))
    return t.contiguous()


def _image(t, ref):
    """The image (N, H, W, 3) uint8 at ref's map size and on its device, made contiguous."""
    N, _, H, W = ref.shape
    if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8 or tuple(t.shape) != (N, H, W, 3) \
            or t.device != ref.device:
        raise ValueError("image must be a (%d, %d, %d, 3) uint8 tensor on %s" % (N, H, W, ref.device))
    return t.contiguous()


def _theta_values(theta, name, n, ref):
    """A learnable bandwidth vector's values as floats (one synchronising copy for a CUDA tensor)."""
    if theta is None:
        return None
    if (not isinstance(theta, torch.Tensor) or tuple(theta.shape) != (n,) or not theta.is_floating_point()
            or (theta.device.type != "cpu" and theta.device != ref.device)):
        raise ValueError("%s must be None or a (%d,) floating-point tensor on the CPU or on %s (got %r)"
                         % (name, n, ref.device,
                            theta if not isinstance(theta, torch.Tensor) else (theta.dtype, tuple(theta.shape),
                                                                               theta.device)))
    if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
        # a CUDA theta is copied to the host here, and the backward copies a CPU theta's gradient back to the host
        raise ValueError("%s is read on the host to build the lattices: it cannot be given inside CUDA-graph "
                         "capture" % name)
    v = [float(x) for x in theta.detach().to("cpu", torch.float64)]
    if not all(math.isfinite(x) and x > 0 for x in v):
        raise ValueError("%s must be positive and finite (got %r)" % (name, v))
    return v


def _set_theta(params, th_bi, th_sp):
    """params with the values of a given theta_bi / theta_sp in place of its sigmas."""
    if th_bi is not None:
        (params.theta_alpha_x, params.theta_alpha_y, params.theta_beta_r, params.theta_beta_g,
         params.theta_beta_b) = th_bi
    if th_sp is not None:
        params.theta_gamma_x, params.theta_gamma_y = th_sp
    return params


def _compat_matrix(mu, name, ref, M):
    if not isinstance(mu, torch.Tensor) or tuple(mu.shape) != (M, M) or not mu.is_floating_point() \
            or mu.device != ref.device:
        raise ValueError("%s must be None or an (%d, %d) floating-point tensor on %s (got %r)"
                         % (name, M, M, ref.device,
                            mu if not isinstance(mu, torch.Tensor) else (mu.dtype, tuple(mu.shape), mu.device)))
    return mu.float()


def _train_args(unary, image, scale_factor, color_factor, maxiter, w1, w2, compat_bi, compat_sp, theta_bi, theta_sp,
                features_bi, wide):
    """dense_crf's and dense_crf_wide's arguments, every check before the first launch -> the arguments of
    _DenseCrfTrain.  wide: dense_crf_wide, which takes any label count and runs 32 or fewer as dense_crf does."""
    if torch.is_autocast_enabled("cuda"):   # what custom_fwd(cast_inputs=float32) does, before the checks
        unary = unary.float() if isinstance(unary, torch.Tensor) and unary.is_floating_point() else unary
        if isinstance(features_bi, torch.Tensor) and features_bi.is_floating_point():
            features_bi = features_bi.float()
    u = _maps(unary, "unary")
    N, M, H, W = u.shape
    if not wide and M > FUSED_LABELS:
        raise ValueError("dense_crf supports at most %d labels (got %d); dense_crf_wide takes up to %d"
                         % (FUSED_LABELS, M, MAX_LABELS))
    feat = features_bi is not None
    if feat:
        if image is not None:
            raise ValueError("image is not used when features_bi is given: pass None")
        if theta_bi is not None:
            raise ValueError("theta_bi and features_bi are two forms of the bilateral features: give one of them")
        x = _features(features_bi, N, H, W, u.device)
    else:
        x = _image(image, u)
    th_bi, th_sp = _theta_values(theta_bi, "theta_bi", 5, u), _theta_values(theta_sp, "theta_sp", 2, u)
    _cuda(u, "unary")
    w1, w2 = _potts_weight(w1, "w1", u), _potts_weight(w2, "w2", u)
    if int(maxiter) < 0:
        raise ValueError("maxiter must be >= 0 (got %d)" % maxiter)
    params = _set_theta(api.crf_params(float(scale_factor), float(color_factor), int(maxiter)), th_bi, th_sp)
    compat = None
    if compat_bi is not None or compat_sp is not None:
        compat = _compat_stack(u, M, w1, w2, compat_bi, compat_sp)
        w1 = w2 = None
    return u, x, w1, w2, compat, theta_bi, theta_sp, params, M > FUSED_LABELS, feat


def dense_crf(unary, image, scale_factor=1.0, color_factor=13, maxiter=10, w1=None, w2=None, compat_bi=None,
              compat_sp=None, theta_bi=None, theta_sp=None, features_bi=None):
    """The dense CRF of CRF() (CRF/krahenbuhl2013/CRF.py:4-37) as a differentiable layer: unary (N, M, H, W) float32,
    M <= 32, the values CRF(image, unary) takes (energy = -unary); image (N, H, W, 3) uint8 at the map size ->
    marginals (N, M, H, W) after `maxiter` mean-field iterations.  The backward is the exact gradient of the
    marginals (the mean field run backwards, DenseCRF::gradient): to `unary` and, when given as 0-dim CUDA tensors,
    to the Potts weights w1 (bilateral) and w2 (spatial), whose gradient is the sum over the batch.  None means
    CRF()'s 10 and 3, without a gradient.  The forward keeps every iteration's marginals for the backward:
    (maxiter + 1) * N * M * H * W * 4 bytes of device memory.

    compat_bi / compat_sp: (M, M) label-compatibility matrices of the bilateral / spatial kernel, learnable in place
    of w1 / w2 (not together with them): the message to label l is -sum_l' mu[l, l'] F(Q)[l'], so Potts(w) is
    -w * I, the reference's MatrixCompatibility(m) is (m + m.T) / 2 and its DiagonalCompatibility(v) is diag(v).
    A matrix left None is -w * I of its weight (w1 / w2, or CRF()'s 10 / 3).  Their gradients are summed over the
    batch.

    theta_bi (5,) = (theta_alpha_x, theta_alpha_y, theta_beta_r, theta_beta_g, theta_beta_b) and theta_sp (2,) =
    (theta_gamma_x, theta_gamma_y): learnable kernel bandwidths, floating-point tensors on the CPU or on unary's
    device, in place of the values scale_factor / color_factor give (a None one keeps those).  Their gradient is the
    exact derivative of the function the device computes with every pixel's simplex held, summed over the batch and
    returned on the tensor's own device and dtype; it works with the Potts weights and with the matrices.  The
    lattice build takes the sigmas as host values, so the forward reads a given theta on the host: one synchronising
    copy for a CUDA tensor, which is why a given theta is refused inside CUDA-graph capture.

    features_bi (N, 5, H, W) float32 on unary's device: the bilateral kernel's features, in place of
    (x/theta_alpha_x, y/theta_alpha_y, r/theta_beta_r, g/theta_beta_g, b/theta_beta_b) of an image, which must then be
    None (theta_bi too).  The lattice is built on the given values as they are; the spatial kernel keeps the sigmas of
    scale_factor (or theta_sp).  The gradient to features_bi is dL/df per pixel, exact with every pixel's simplex held,
    so a learned transform of any guidance (the reference's FULL_KERNEL is f = P @ raw) trains through autograd.  The
    features are never read on the host: without theta_sp a step can be captured in a CUDA graph.  Keep every feature
    within +-150 (the CRF does not change when a channel is shifted, so centre them): an image whose lattice keys leave
    the packed range gets NaN marginals and gradients (Engine.feature_range_flags names it)."""
    return _DenseCrfTrain.apply(*_train_args(unary, image, scale_factor, color_factor, maxiter, w1, w2, compat_bi,
                                             compat_sp, theta_bi, theta_sp, features_bi, wide=False))


def _compat_stack(u, M, w1, w2, compat_bi, compat_sp):
    """(2, M, M) {mu_bi, mu_sp}, a missing matrix built as -w I of its weight."""
    mats = []
    for mu, w, d, name, wname in ((compat_bi, w1, _POTTS_DEFAULT[0], "compat_bi", "w1"),
                                  (compat_sp, w2, _POTTS_DEFAULT[1], "compat_sp", "w2")):
        if mu is None:   # Potts: -w I, through which autograd carries w's gradient
            eye = torch.eye(M, dtype=torch.float32, device=u.device)
            mats.append(-(w.float() if w is not None else d) * eye)
        elif w is not None:
            raise ValueError("%s and %s are two forms of one term: give one of them" % (name, wname))
        else:
            mats.append(_compat_matrix(mu, name, u, M))
    return torch.stack(mats)


def dense_crf_wide(unary, image, scale_factor=1.0, color_factor=13, maxiter=10, w1=None, w2=None, compat_bi=None,
                   compat_sp=None, theta_bi=None, theta_sp=None, features_bi=None):
    """dense_crf for any label count from 1 to 255 (COCO's 81 classes), with every parameter dense_crf learns learnable
    as there: the Potts weights or the label-compatibility matrices, the kernel bandwidths theta_bi / theta_sp and the
    caller-given bilateral features features_bi (same arguments, same checks, same gradients).  At 32 labels or fewer
    it is dense_crf itself; above that the mean field and its exact backward run on the label-chunked kernels, whose
    per-label cost is several times the fused path's.  Nothing is read on the host unless a theta is given (its values
    build the lattices), so without one a step can be captured in a CUDA graph.  The forward keeps every iteration's
    marginals: (maxiter + 1) * N * M * H * W * 4 bytes, 120 MB at batch 20 @ 41x41 with 81 labels."""
    return _DenseCrfTrain.apply(*_train_args(unary, image, scale_factor, color_factor, maxiter, w1, w2, compat_bi,
                                             compat_sp, theta_bi, theta_sp, features_bi, wide=True))


def _learned_crf(ref, N, M, H, W, params, w1=None, w2=None, compat_bi=None, compat_sp=None, theta_bi=None,
                 theta_sp=None, features_bi=None):
    """The learned CRF's inference arguments, checked as dense_crf checks them: params takes the sigmas and, on the
    Potts path, the weights (read on the host, so refused inside CUDA-graph capture); returns (features, compat) for
    the device, either of them None.  ref: any tensor on the CRF's device."""
    f = None
    if features_bi is not None:
        if theta_bi is not None:
            raise ValueError("theta_bi and features_bi are two forms of the bilateral features: give one of them")
        f = _features(features_bi, N, H, W, ref.device)
    th_bi, th_sp = _theta_values(theta_bi, "theta_bi", 5, ref), _theta_values(theta_sp, "theta_sp", 2, ref)
    w1, w2 = _potts_weight(w1, "w1", ref), _potts_weight(w2, "w2", ref)
    _set_theta(params, th_bi, th_sp)
    if compat_bi is not None or compat_sp is not None:
        with torch.no_grad():   # a missing matrix is -w I of its weight, formed on the device
            return f, _compat_stack(ref, M, w1, w2, compat_bi, compat_sp).contiguous()
    given = [(i, w) for i, w in enumerate((w1, w2)) if w is not None]
    if given:
        if torch.cuda.is_current_stream_capturing():
            raise ValueError("w1 / w2 are read on the host at inference: they cannot be given inside CUDA-graph "
                             "capture (pass compat_bi / compat_sp = -w I to keep them on the device)")
        vals = torch.stack([w.detach().to(torch.float64) for _, w in given]).cpu().tolist()   # one synchronising copy
        for (i, _), v in zip(given, vals):
            setattr(params, "w1" if i == 0 else "w2", v)
    return f, None


def dense_crf_inference(unary, image, scale_factor=1.0, color_factor=13, maxiter=10, w1=None, w2=None,
                        compat_bi=None, compat_sp=None, theta_bi=None, theta_sp=None, features_bi=None):
    """dense_crf's forward at inference cost: the same arguments, semantics and checks as dense_crf / dense_crf_wide,
    for 1 to 255 labels, returning the (N, M, H, W) marginals after `maxiter` iterations without autograd and without
    keeping the iterates (the output is the only allocation).  So a CRF trained with dense_crf evaluates and
    pseudo-labels with the same parameters.
      w1 / w2, theta_bi / theta_sp : read on the host (one synchronising copy each), so refused inside CUDA-graph
                                     capture; on the matrix path a weight only forms -w I of a missing matrix, on the
                                     device
      compat_bi / compat_sp        : read on the device (a matrix left None is -w I of its weight)
      features_bi                  : read on the device, in place of image (which must then be None); an image whose
                                     lattice keys leave the packed range gets NaN marginals (Engine.feature_range_flags)
    A call with only matrices and features can be captured.  With no learned argument it is Engine.crf_dev's Potts
    inference itself."""
    if torch.is_autocast_enabled("cuda"):
        unary = unary.float() if isinstance(unary, torch.Tensor) and unary.is_floating_point() else unary
        if isinstance(features_bi, torch.Tensor) and features_bi.is_floating_point():
            features_bi = features_bi.float()
    u = _maps(unary, "unary")
    if features_bi is None:
        image = _image(image, u)
    elif image is not None:
        raise ValueError("image is not used when features_bi is given: pass None")
    if int(maxiter) < 0:
        raise ValueError("maxiter must be >= 0 (got %d)" % maxiter)
    _cuda(u, "unary")
    params = api.crf_params(float(scale_factor), float(color_factor), int(maxiter))
    f, compat = _learned_crf(u, *u.shape, params, w1, w2, compat_bi, compat_sp, theta_bi, theta_sp, features_bi)
    eng = _engine_for(u)
    out = torch.empty(u.shape, dtype=torch.float32, device=u.device)
    s = _stream(u)
    if f is None and compat is None:
        return eng.crf_dev(u, image, params, out, api.LAYOUT_NCHW, api.LAYOUT_NCHW, stream=s)
    return eng.crf_learned_dev(u, image, params, out, features=f,
                               compat=compat, unary_layout=api.LAYOUT_NCHW, out_layout=api.LAYOUT_NCHW, stream=s)


class _DenseCrfEnergy(torch.autograd.Function):
    """dense_crf_energy's terms (N, 4) and their gradient to q and unary; the parameters carry none.  wide: the
    label-chunked entry points above 32 labels."""

    @staticmethod
    @_fwd
    def forward(ctx, q, unary, image, features, compat, params, wide):
        terms = torch.empty((q.shape[0], 4), dtype=torch.float32, device=q.device)
        fwd = _engine_for(q).crf_energy_wide_dev if wide else _engine_for(q).crf_energy_dev
        fwd(q, unary, image, params, terms, features=features, compat=compat, stream=_stream(q))
        ctx.save_for_backward(q, unary, image, features, compat)
        ctx.params, ctx.wide = params, wide
        return terms

    @staticmethod
    @_bwd
    def backward(ctx, g):
        q, unary, image, features, compat = ctx.saved_tensors
        grad_q = torch.empty_like(q)
        grad_u = torch.empty_like(q) if unary is not None and ctx.needs_input_grad[1] else None
        eng = _engine_for(q)
        bwd = eng.crf_energy_backward_wide_dev if ctx.wide else eng.crf_energy_backward_dev
        bwd(q, unary, image, ctx.params, g.float().contiguous(), grad_q, grad_unary=grad_u, features=features,
            compat=compat, stream=_stream(q))
        return grad_q if ctx.needs_input_grad[0] else None, grad_u, None, None, None, None, None


def _energy_args(q, unary, image, scale_factor, color_factor, w1, w2, compat_bi, compat_sp, theta_bi, theta_sp,
                 features_bi, wide):
    """dense_crf_energy's and dense_crf_energy_wide's arguments, every check before the first launch -> the arguments
    of _DenseCrfEnergy.  wide: dense_crf_energy_wide, which takes 1 to 255 labels and runs 32 or fewer as
    dense_crf_energy does."""
    if torch.is_autocast_enabled("cuda"):
        q = q.float() if isinstance(q, torch.Tensor) and q.is_floating_point() else q
        unary = unary.float() if isinstance(unary, torch.Tensor) and unary.is_floating_point() else unary
        if isinstance(features_bi, torch.Tensor) and features_bi.is_floating_point():
            features_bi = features_bi.float()
    name_of = "dense_crf_energy_wide" if wide else "dense_crf_energy"
    for name, t in (("w1", w1), ("w2", w2), ("compat_bi", compat_bi), ("compat_sp", compat_sp),
                    ("theta_bi", theta_bi), ("theta_sp", theta_sp), ("features_bi", features_bi)):
        if isinstance(t, torch.Tensor) and t.requires_grad:
            raise ValueError("%s requires grad: %s differentiates q and unary only (detach it)" % (name, name_of))
    qq = _maps(q, "q")
    M = qq.shape[1]
    if not wide and M > FUSED_LABELS:
        raise ValueError("dense_crf_energy supports at most %d labels (got %d)" % (FUSED_LABELS, M))
    u = None if unary is None else _like(unary, qq, "unary")
    if features_bi is None:
        image = _image(image, qq)
    elif image is not None:
        raise ValueError("image is not used when features_bi is given: pass None")
    _cuda(qq, "q")
    params = api.crf_params(float(scale_factor), float(color_factor), 0)
    f, compat = _learned_crf(qq, *qq.shape, params, w1, w2, compat_bi, compat_sp, theta_bi, theta_sp, features_bi)
    return qq, u, image, f, compat, params, M > FUSED_LABELS


def dense_crf_energy(q, unary, image, scale_factor=1.0, color_factor=13, w1=None, w2=None, compat_bi=None,
                     compat_sp=None, theta_bi=None, theta_sp=None, features_bi=None):
    """The dense CRF's energy of q (N, M, H, W), M <= 32, per term: (N, 4) = (entropy sum Q log max(Q, 1e-20), unary
    -sum unary Q, spatial sum Q mu_sp F_sp(Q), bilateral sum Q mu_bi F_bi(Q)), so ``.sum(1)`` is the reference's
    DenseCRF::klDivergence of each image.  q is any non-negative array: marginals, a softmax, or a one-hot label map
    (whose result is that labelling's energy under the reference's convention).  Like the reference, the pairwise
    terms carry no 1/2: every pair of pixels counts twice.  unary (N, M, H, W) holds the values CRF(image, unary)
    takes (energy = -unary), or None for no unary term.

    The parameters are dense_crf_inference's, with its checks and semantics (w1 / w2 and theta_bi / theta_sp read on
    the host; compat_bi / compat_sp and features_bi on the device, features_bi in place of image).  The result is
    differentiable to q and unary: the pairwise gradient is mu F(Q) + mu^T F^T(Q) with the device's transposed blur,
    exact for the function the device computes.  A term's pairwise energy alone (``terms[:, 2:].sum()``) is the
    dense-CRF regulariser of weakly-supervised segmentation.  The parameters get no gradient: a parameter tensor that
    requires grad is refused.  A features_bi image whose lattice keys leave the packed range gets NaN terms and
    gradients.  dense_crf_energy_wide takes up to 255 labels."""
    return _DenseCrfEnergy.apply(*_energy_args(q, unary, image, scale_factor, color_factor, w1, w2, compat_bi,
                                               compat_sp, theta_bi, theta_sp, features_bi, wide=False))


def dense_crf_energy_wide(q, unary, image, scale_factor=1.0, color_factor=13, w1=None, w2=None, compat_bi=None,
                          compat_sp=None, theta_bi=None, theta_sp=None, features_bi=None):
    """dense_crf_energy for any label count from 1 to 255 (COCO's 81 classes): the same arguments, checks, terms and
    gradients to q and unary.  At 32 labels or fewer it is dense_crf_energy itself; above that the energy and its
    gradient run on the label-chunked kernels, with the same operation order per value and no device memory beyond
    dense_crf_energy's per-block sums."""
    return _DenseCrfEnergy.apply(*_energy_args(q, unary, image, scale_factor, color_factor, w1, w2, compat_bi,
                                               compat_sp, theta_bi, theta_sp, features_bi, wide=True))


def softmax(fc8):
    """SoftmaxLayer (pylayers.py:23-51): probs = (softmax(fc8) + 1e-4) / sum over labels.  fc8 (N, M, H, W),
    M <= 32 (more labels raise the library's DsrgError)."""
    return _Softmax.apply(fc8)


def crf_layer(probs, images, scale_factor=12.0):
    """CRFLayer (pylayers.py:54-92): probs (N, M, H, W), images (N, 3, Hi, Wi) the network input ->
    (log_crf, probs_c): the log of the renormalised CRF marginals, and probs clamped at 1e-4.  Backward:
    (1 - marginals) * d log_crf + d probs_c."""
    return _CrfLayer.apply(probs, images, float(scale_factor))


def dsrg_seeds(labels, probs, cues, images, th1=0.99, th2=0.85, scale_factor=12.0):
    """DSRGLayer (pylayers.py:277-344), with its own mean-field pass: labels (N, 1, 1, M) or (N, M), probs and cues
    (N, M, H, W), images (N, 3, Hi, Wi) -> seeds (N, M, H, W).  The gradient of the seeds goes straight to probs
    (pylayers.py:307-308)."""
    return _DsrgSeeds.apply(labels, probs, cues, images, float(th1), float(th2), float(scale_factor))


def balanced_seed_loss(probs, seeds):
    """BalancedSeedLossLayer (pylayers.py:120-152): the mean over this batch; no gradient to seeds."""
    return _BalancedSeedLoss.apply(probs, seeds)


def constrain_loss(probs, log_crf):
    """ConstrainLossLayer (pylayers.py:154-180): gradients to both inputs."""
    return _ConstrainLoss.apply(probs, log_crf)


def seed_loss(probs, seeds):
    """SEC's SeedLossLayer (pylayers.py:95-118): no floor on the seed count; no gradient to seeds."""
    return _SeedLoss.apply(probs, seeds)


def expand_loss(probs, labels, q_fg=0.996, q_bg=0.999):
    """SEC's ExpandLossLayer (pylayers.py:183-233), global weighted rank pooling over planes of at most 8192
    pixels; labels (N, 1, 1, M) or (N, M).  No gradient to labels."""
    return _ExpandLoss.apply(probs, labels, float(q_fg), float(q_bg))


class DSRGHead(torch.nn.Module):
    """The stage-1 head of train-s.prototxt (:746-812): Softmax -> CRF -> DSRG -> BalancedSeedLoss + ConstrainLoss,
    with one mean-field pass per step shared by the CRF and DSRG layers.

    forward(fc8, images, labels, cues) -> (loss_seed, loss_constrain, seeds):
      fc8    (N, M, H, W) scores, M <= 32       images (N, 3, Hi, Wi) the network input, mean-subtracted BGR
      labels (N, 1, 1, M) or (N, M) image tags  cues   (N, M, H, W) localisation cues
    all CUDA float32 (cast to float32 under autocast).  The seeds carry no gradient."""

    def __init__(self, th1=0.99, th2=0.85, scale_factor=12.0):
        super().__init__()
        self.th1, self.th2, self.scale_factor = float(th1), float(th2), float(scale_factor)

    def forward(self, fc8, images, labels, cues):
        if torch.is_autocast_enabled("cuda"):   # what custom_fwd(cast_inputs=float32) does, before the checks
            fc8, images, labels, cues = (t.float() if isinstance(t, torch.Tensor) and t.is_floating_point() else t
                                         for t in (fc8, images, labels, cues))
        # every input is checked before the first launch
        x = _maps(fc8, "fc8")
        _images(images, x), _labels(labels, x), _like(cues, x, "cues"), _cuda(x, "fc8")
        probs = softmax(fc8)
        log_crf, probs_c, seeds = _CrfDsrg.apply(probs, images, labels, cues, self.th1, self.th2, self.scale_factor)
        return balanced_seed_loss(probs_c, seeds), constrain_loss(probs_c, log_crf), seeds

    def extra_repr(self):
        return "th1=%g, th2=%g, scale_factor=%g" % (self.th1, self.th2, self.scale_factor)
