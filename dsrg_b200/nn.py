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

Engines are cached per (labels, height, width, device) and recreated when a larger batch arrives.  Autograd runs
a backward on the forward's stream and device, so one engine is never driven from two threads at once.

A step captured in a CUDA graph uses the cached engine's buffers.  Two rules follow:
* Replacing the engine frees them.  A captured step must not be replayed once a larger batch has reached the same
  (labels, height, width, device); a larger batch during a capture raises RuntimeError.
* The engine orders its eager calls across streams, but a graph replay leaves no mark it can wait for.  Replays and
  eager steps on the same engine must run on one stream, or be ordered by the caller.
"""
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
