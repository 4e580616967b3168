"""One batch-1 engine per label count, shared by the per-image callers (krahenbuhl2013.CRF, the
inference post-processing): the evaluation tools feed images of many different sizes
(training/tools/test-ms.py:86-87), so the engine is sized for the largest image seen so far and
re-shaped per call (dsrg_engine_set_size) instead of being re-created.  The batched post-processing has its own
engines (batch_engine_for), pooled the same way."""
from . import api as _api

_ENGINES = {}      # (M, device) -> Engine
_ROUND = 64        # capacity granularity, so that slightly larger images do not force a new engine


def engine_for(H, W, M, device=None):
    """device None: the calling thread's current CUDA device (dsrg_current_device)."""
    H, W, M = int(H), int(W), int(M)
    if device is None:
        from . import _lib
        device = _lib.lib().dsrg_current_device()
    key = (M, int(device))
    eng = _ENGINES.get(key)
    if eng is not None:
        hc, wc = eng.capacity
        if H > hc or W > wc:
            eng.close()
            eng = None
            H0, W0 = max(H, hc), max(W, wc)
        else:
            H0, W0 = hc, wc
    else:
        H0, W0 = H, W
    if eng is None:
        up = lambda v: (v + _ROUND - 1) // _ROUND * _ROUND  # noqa: E731
        eng = _api.Engine(1, up(H0), up(W0), M, device)
        _ENGINES[key] = eng
    eng.set_size(H, W)
    return eng


_BATCH_ENGINES = {}   # (M, device) -> Engine of the batched post-processing


def batch_capacity(B, H, W, M, device):
    """(max_batch, H capacity, W capacity) of the engine batch_engine_for(B, H, W, M, device) returns, read without
    creating or changing an engine."""
    B, H, W = int(B), int(H), int(W)
    eng = _BATCH_ENGINES.get((int(M), int(device)))
    if eng is not None:
        hc, wc = eng.capacity
        if B <= eng.max_batch and H <= hc and W <= wc:
            return eng.max_batch, hc, wc
        B, H, W = max(B, eng.max_batch), max(H, hc), max(W, wc)
    up = lambda v: (v + _ROUND - 1) // _ROUND * _ROUND  # noqa: E731
    return B, up(H), up(W)


def batch_engine_for(B, H, W, M, device=None, select=True):
    """The engine of the batched callers (postprocess.predict_masks_*, predict_mask_batch_dev): one per label count
    and device, apart from the batch-1 one of engine_for so the two keep their own graphs and buffers.  Its size
    capacity is rounded up like engine_for's and its batch capacity grows to the largest batch requested.
    With `select` the engine is re-shaped to H x W without waiting for the device (dsrg_engine_set_size_ordered): its
    callers drive it through the entry points only, each of which orders its pass after the engine's previous one.
    Without, only the capacity is ensured."""
    B, H, W, M = int(B), int(H), int(W), int(M)
    if device is None:
        from . import _lib
        device = _lib.lib().dsrg_current_device()
    key = (M, int(device))
    eng = _BATCH_ENGINES.get(key)
    cap = batch_capacity(B, H, W, M, device)
    if eng is not None and (eng.max_batch,) + eng.capacity != cap:
        eng.close()
        eng = None
    if eng is None:
        eng = _api.Engine(cap[0], cap[1], cap[2], M, device)
        _BATCH_ENGINES[key] = eng
    if select:
        eng.set_size(H, W, ordered=True)   # host state only, so it may also run inside a stream capture
    return eng


_PREP_ENGINES = {}    # device -> Engine of the batched network input


def prep_engine_for(B, device):
    """The engine of postprocess.preprocess_batch*: the network input reads no engine buffer and neither reads nor
    changes the engine's size, so this one is 1 x 1 with one label, per device, and grows in batch only.  Neither of
    the post-processing engines grows to the largest image of a list on its account.  Inside a CUDA-graph capture it
    can be neither created nor replaced: RuntimeError."""
    B, device = int(B), int(device)
    eng = _PREP_ENGINES.get(device)
    if eng is None or B > eng.max_batch:
        import torch
        if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("a batch of %d images reached the network-input engine of device %d (%s) during "
                               "CUDA-graph capture: run the largest batch once before capturing"
                               % (B, device, "none yet" if eng is None else "made for %d" % eng.max_batch))
        if eng is not None:
            eng.close()
        eng = _api.Engine(B, 1, 1, 1, device)
        _PREP_ENGINES[device] = eng
    return eng


def clear():
    for eng in list(_ENGINES.values()) + list(_BATCH_ENGINES.values()) + list(_PREP_ENGINES.values()):
        eng.close()
    _ENGINES.clear()
    _BATCH_ENGINES.clear()
    _PREP_ENGINES.clear()
