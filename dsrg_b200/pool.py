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


def batch_engine_for(B, H, W, M, device=None):
    """The engine of the batched callers (postprocess.predict_masks_*, predict_mask_batch_dev): one per label count
    and device, apart from the batch-1 one of engine_for so the two keep their own graphs and buffers.  Its size
    capacity is rounded up like engine_for's and its batch capacity grows to the largest batch requested."""
    B, H, W, M = int(B), int(H), int(W), int(M)
    if device is None:
        from . import _lib
        device = _lib.lib().dsrg_current_device()
    key = (M, int(device))
    eng = _BATCH_ENGINES.get(key)
    B0, H0, W0 = B, H, W
    if eng is not None:
        hc, wc = eng.capacity
        if B > eng.max_batch or H > hc or W > wc:
            B0, H0, W0 = max(B, eng.max_batch), max(H, hc), max(W, wc)
            eng.close()
            eng = None
    if eng is None:
        up = lambda v: (v + _ROUND - 1) // _ROUND * _ROUND  # noqa: E731
        eng = _api.Engine(B0, up(H0), up(W0), M, device)
        _BATCH_ENGINES[key] = eng
    eng.set_size(H, W)   # a no-op when the size is already selected (so it may run inside a stream capture)
    return eng


def clear():
    for eng in list(_ENGINES.values()) + list(_BATCH_ENGINES.values()):
        eng.close()
    _ENGINES.clear()
    _BATCH_ENGINES.clear()
