"""Python host side of the C ABI: thin wrappers, no compute.

`Engine` mirrors dsrg_engine.  Device arrays are torch CUDA tensors used purely as memory
containers (``data_ptr()``); host arrays are numpy.  Every method maps 1:1 onto an entry point of
include/dsrg_b200.h -- see that header for the reference interface each one replaces.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import (LAYOUT_NCHW, LAYOUT_NHWC, POST_SUM_SCORES, POST_ZOOM_PROBS, CrfParams, DsrgError,  # noqa: F401
                   check)


def crf_params(scale_factor=1.0, color_factor=13, maxiter=10):
    """The pairwise parameters CRF() uses (CRF/krahenbuhl2013/CRF.py:31-32)."""
    p = CrfParams()
    _lib.lib().dsrg_crf_params_default(C.byref(p), float(scale_factor), float(color_factor), int(maxiter))
    return p


def _dptr(t):
    """Device pointer of a contiguous torch CUDA tensor (or None)."""
    if t is None:
        return None
    if not t.is_cuda or not t.is_contiguous():
        raise ValueError("expected a contiguous CUDA tensor")
    return C.c_void_p(t.data_ptr())


def _hptr(a, dtype):
    if a is None:
        return None
    if not isinstance(a, np.ndarray) or a.dtype != dtype or not a.flags["C_CONTIGUOUS"]:
        raise ValueError("expected a C-contiguous numpy array of dtype %s" % np.dtype(dtype))
    return C.c_void_p(a.ctypes.data)


def _stream(stream):
    if stream is None:
        import torch
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)
    return C.c_void_p(int(stream))


class _PinnedBlock(object):
    """Owner of one dsrg_host_alloc block; the numpy arrays built over it keep it alive through the ctypes
    buffer they wrap (numpy's ``base`` chain), and the block is returned with dsrg_host_free when the last of
    them is gone."""

    def __init__(self, L, nbytes):
        self._L = L
        self.ptr = L.dsrg_host_alloc(nbytes)
        if not self.ptr:
            raise DsrgError(_lib.E_NOMEM, L.dsrg_last_error().decode())

    def __del__(self):
        if getattr(self, "ptr", None):
            try:
                self._L.dsrg_host_free(self.ptr)
            except Exception:
                pass
            self.ptr = None


def pinned_empty(shape, dtype):
    """numpy array over pinned host memory from dsrg_host_alloc (freed when the array and its views are)."""
    L = _lib.lib()
    dtype = np.dtype(dtype)
    n = max(int(np.prod(shape)) * dtype.itemsize, 16)
    block = _PinnedBlock(L, n)
    buf = (C.c_char * n).from_address(block.ptr)
    buf._dsrg_block = block   # the ctypes object is the base of every array below: it carries the owner
    return np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)


class Engine(object):
    """dsrg_engine: all device buffers for batches of up to ``max_batch`` H x W x M problems."""

    def __init__(self, max_batch, H, W, M=21, device=None):
        """device None: the calling thread's current CUDA device (dsrg_current_device: what caffe.set_device /
        torch.cuda.set_device selected, or DSRG_B200_DEVICE)."""
        self._L = _lib.lib()
        if device is None:
            device = self._L.dsrg_current_device()
        self.max_batch, self.H, self.W, self.M, self.device = int(max_batch), int(H), int(W), int(M), int(device)
        self.h = self._L.dsrg_engine_create(self.device, self.max_batch, self.H, self.W, self.M)
        if not self.h:
            raise DsrgError(_lib.E_CUDA, self._L.dsrg_last_error().decode())

    def close(self):
        if getattr(self, "h", None):
            self._L.dsrg_engine_destroy(self.h)
            self.h = None

    __del__ = close

    @property
    def device_bytes(self):
        return self._L.dsrg_engine_device_bytes(self.h)

    def set_size(self, H, W, ordered=False):
        """Select an image size within the capacity the engine was created with (no reallocation).  Waits for the
        device when the size changes, unless `ordered`: then the caller drives this engine only through its entry
        points (dsrg_engine_set_size_ordered), and no replay of a CUDA graph of its own holds the engine's launches."""
        fn = self._L.dsrg_engine_set_size_ordered if ordered else self._L.dsrg_engine_set_size
        check(fn(self.h, int(H), int(W)))
        self.H, self.W = int(H), int(W)

    @property
    def capacity(self):
        v = [C.c_int() for _ in range(4)]
        check(self._L.dsrg_engine_get_size(self.h, *[C.byref(x) for x in v]))
        return v[2].value, v[3].value

    def set_host_chunk(self, images):
        check(self._L.dsrg_engine_set_host_chunk(self.h, int(images)))

    def set_graphs(self, enable):
        """CUDA-graph replay of repeated device passes (default on; needs a non-default stream)."""
        check(self._L.dsrg_engine_set_graphs(self.h, int(bool(enable))))

    @property
    def graph_replays(self):
        return int(self._L.dsrg_engine_graph_replays(self.h))

    @property
    def hybrid_tiles(self):
        """Tiles of the last mean-field pass that took the hybrid path (textured images); synchronises."""
        n = int(self._L.dsrg_engine_hybrid_tiles(self.h))
        if n < 0:
            raise DsrgError(_lib.last_error())
        return n

    def take_launch_count(self):
        return int(self._L.dsrg_engine_take_launch_count(self.h))

    # ---- device entry points (torch tensors as containers) ----
    def crf_dev(self, unary, image, params, out, unary_layout=LAYOUT_NHWC, out_layout=LAYOUT_NHWC, stream=None):
        B = image.shape[0]
        check(self._L.dsrg_crf_batch_dev(self.h, B, _dptr(unary), unary_layout, _dptr(image), C.byref(params),
                                         _dptr(out), out_layout, _stream(stream)))
        return out

    def crf_forward_train_dev(self, unary, image, params, q_hist, potts=None, stream=None):
        """The CRF forward that keeps Q_0..Q_T for the backward: unary (B, M, H, W), image (B, H, W, 3) uint8,
        q_hist (T+1, B, M, H, W) with q_hist[T] the marginals; potts an optional device float32 [2] {w1, w2} read in
        place of params.w1 / w2."""
        B = unary.shape[0]
        check(self._L.dsrg_crf_forward_train_dev(self.h, _dptr(unary), B, _dptr(image), C.byref(params), _dptr(potts),
                                                 _dptr(q_hist), _stream(stream)))
        return q_hist

    def crf_backward_dev(self, q_hist, image, params, grad_q, grad_unary, grad_potts=None, potts=None, stream=None):
        """DenseCRF::gradient for grad_q = dL/dQ_T (B, M, H, W): grad_unary = dL/dunary (B, M, H, W) and, if given,
        grad_potts (B, 2) = {dL/dw1, dL/dw2} per image.  image, params and potts as in the forward."""
        B = grad_q.shape[0]
        check(self._L.dsrg_crf_backward_dev(self.h, _dptr(q_hist), B, _dptr(image), C.byref(params), _dptr(potts),
                                            _dptr(grad_q), _dptr(grad_unary), _dptr(grad_potts), _stream(stream)))
        return grad_unary

    def crf_forward_train_compat_dev(self, unary, image, params, compat, q_hist, stream=None):
        """crf_forward_train_dev with label-compatibility matrices in place of the Potts weights: compat a device
        float32 (2, M, M) {mu_bi, mu_sp}, t = unary - mu_sp F_sp(Q) - mu_bi F_bi(Q); params.w1 / w2 are ignored."""
        B = unary.shape[0]
        check(self._L.dsrg_crf_forward_train_compat_dev(self.h, _dptr(unary), B, _dptr(image), C.byref(params),
                                                        _dptr(compat), _dptr(q_hist), _stream(stream)))
        return q_hist

    def crf_backward_compat_dev(self, q_hist, image, params, compat, grad_q, grad_unary, grad_compat=None,
                                stream=None):
        """The backward of crf_forward_train_compat_dev: grad_unary (B, M, H, W) and, if given, grad_compat
        (B, 2, M, M) = dL/d{mu_bi, mu_sp} per image."""
        B = grad_q.shape[0]
        check(self._L.dsrg_crf_backward_compat_dev(self.h, _dptr(q_hist), B, _dptr(image), C.byref(params),
                                                   _dptr(compat), _dptr(grad_q), _dptr(grad_unary),
                                                   _dptr(grad_compat), _stream(stream)))
        return grad_unary

    def crf_backward_theta_dev(self, q_hist, image, params, grad_q, grad_unary, grad_theta, grad_potts=None,
                               potts=None, stream=None):
        """crf_backward_dev that also writes grad_theta (B, 7) = dL/dtheta per image in dsrg_crf_params' order
        (theta_alpha_x, theta_alpha_y, theta_beta_r, theta_beta_g, theta_beta_b, theta_gamma_x, theta_gamma_y)."""
        B = grad_q.shape[0]
        check(self._L.dsrg_crf_backward_theta_dev(self.h, _dptr(q_hist), B, _dptr(image), C.byref(params),
                                                  _dptr(potts), _dptr(grad_q), _dptr(grad_unary), _dptr(grad_potts),
                                                  _dptr(grad_theta), _stream(stream)))
        return grad_unary

    def crf_backward_compat_theta_dev(self, q_hist, image, params, compat, grad_q, grad_unary, grad_theta,
                                      grad_compat=None, stream=None):
        """crf_backward_compat_dev that also writes grad_theta (B, 7) as crf_backward_theta_dev does."""
        B = grad_q.shape[0]
        check(self._L.dsrg_crf_backward_compat_theta_dev(self.h, _dptr(q_hist), B, _dptr(image), C.byref(params),
                                                         _dptr(compat), _dptr(grad_q), _dptr(grad_unary),
                                                         _dptr(grad_compat), _dptr(grad_theta), _stream(stream)))
        return grad_unary

    def crf_forward_train_feat_dev(self, unary, features, params, q_hist, potts=None, compat=None, stream=None):
        """crf_forward_train_dev with caller-given bilateral features: features (B, 5, H, W) float32 on the device
        replace (x/theta_alpha, y/theta_alpha, rgb/theta_beta), taken as they are; params gives the spatial sigmas, the
        iterations and (without potts / compat) the weights.  potts {w1, w2} or compat (2, M, M) {mu_bi, mu_sp}, not
        both.  An image whose lattice keys leave the packed range gets NaN in every iterate (feature_range_flags)."""
        B = unary.shape[0]
        check(self._L.dsrg_crf_forward_train_feat_dev(self.h, _dptr(unary), B, _dptr(features), C.byref(params),
                                                      _dptr(potts), _dptr(compat), _dptr(q_hist), _stream(stream)))
        return q_hist

    def crf_backward_feat_dev(self, q_hist, features, params, grad_q, grad_unary, grad_features, potts=None,
                              compat=None, grad_potts=None, grad_compat=None, grad_theta_sp=None, stream=None):
        """The backward of crf_forward_train_feat_dev: grad_unary (B, M, H, W), grad_features (B, 5, H, W) = dL/df per
        pixel and, if given, grad_potts (B, 2) (Potts), grad_compat (B, 2, M, M) (matrices) and grad_theta_sp (B, 2) =
        dL/d{theta_gamma_x, theta_gamma_y}.  A flagged image's gradients are NaN."""
        B = grad_q.shape[0]
        check(self._L.dsrg_crf_backward_feat_dev(self.h, _dptr(q_hist), B, _dptr(features), C.byref(params),
                                                 _dptr(potts), _dptr(compat), _dptr(grad_q), _dptr(grad_unary),
                                                 _dptr(grad_features), _dptr(grad_potts), _dptr(grad_compat),
                                                 _dptr(grad_theta_sp), _stream(stream)))
        return grad_unary

    def crf_energy_dev(self, q, unary, image, params, terms, features=None, potts=None, compat=None, stream=None):
        """The CRF's energy of q (B, M, H, W) (DenseCRF::klDivergence), per term: terms (B, 4) = {entropy, unary,
        spatial pairwise, bilateral pairwise}, whose sum is the reference's value.  unary (B, M, H, W) or None, image
        (B, H, W, 3) uint8 or None with features (B, 5, H, W); potts {w1, w2} or compat (2, M, M) {mu_bi, mu_sp}, not
        both (neither: params.w1 / w2).  At most 32 labels."""
        B = q.shape[0]
        check(self._L.dsrg_crf_energy_dev(self.h, _dptr(q), B, _dptr(unary), _dptr(image), _dptr(features),
                                          C.byref(params), _dptr(potts), _dptr(compat), _dptr(terms), _stream(stream)))
        return terms

    def crf_energy_backward_dev(self, q, unary, image, params, grad_terms, grad_q, grad_unary=None, features=None,
                                potts=None, compat=None, stream=None):
        """The gradient of crf_energy_dev's terms for grad_terms (B, 4): grad_q (B, M, H, W) and, if given, grad_unary
        (B, M, H, W).  The other arguments as crf_energy_dev's."""
        B = q.shape[0]
        check(self._L.dsrg_crf_energy_backward_dev(self.h, _dptr(q), B, _dptr(unary), _dptr(image), _dptr(features),
                                                   C.byref(params), _dptr(potts), _dptr(compat), _dptr(grad_terms),
                                                   _dptr(grad_q), _dptr(grad_unary), _stream(stream)))
        return grad_q

    def crf_energy_wide_dev(self, q, unary, image, params, terms, features=None, potts=None, compat=None,
                            stream=None):
        """crf_energy_dev above 32 labels (33 to 255), on the label-chunked kernels: the same arguments and terms.  An
        engine of 32 labels or fewer refuses."""
        B = q.shape[0]
        check(self._L.dsrg_crf_energy_wide_dev(self.h, _dptr(q), B, _dptr(unary), _dptr(image), _dptr(features),
                                               C.byref(params), _dptr(potts), _dptr(compat), _dptr(terms),
                                               _stream(stream)))
        return terms

    def crf_energy_backward_wide_dev(self, q, unary, image, params, grad_terms, grad_q, grad_unary=None,
                                     features=None, potts=None, compat=None, stream=None):
        """crf_energy_backward_dev above 32 labels (33 to 255): the gradient of crf_energy_wide_dev's terms."""
        B = q.shape[0]
        check(self._L.dsrg_crf_energy_backward_wide_dev(self.h, _dptr(q), B, _dptr(unary), _dptr(image),
                                                        _dptr(features), C.byref(params), _dptr(potts),
                                                        _dptr(compat), _dptr(grad_terms), _dptr(grad_q),
                                                        _dptr(grad_unary), _stream(stream)))
        return grad_q

    def crf_forward_train_wide_dev(self, unary, image, params, q_hist, potts=None, compat=None, stream=None):
        """crf_forward_train_dev / crf_forward_train_compat_dev above 32 labels (33 to 255): potts {w1, w2} or compat
        (2, M, M) {mu_bi, mu_sp}, not both; neither: params.w1 / w2.  An engine of 32 labels or fewer refuses."""
        B = unary.shape[0]
        check(self._L.dsrg_crf_forward_train_wide_dev(self.h, _dptr(unary), B, _dptr(image), C.byref(params),
                                                      _dptr(potts), _dptr(compat), _dptr(q_hist), _stream(stream)))
        return q_hist

    def crf_backward_wide_dev(self, q_hist, image, params, grad_q, grad_unary, potts=None, compat=None,
                              grad_potts=None, grad_compat=None, stream=None):
        """The backward of crf_forward_train_wide_dev: grad_unary (B, M, H, W) and, if given, grad_potts (B, 2)
        (Potts) or grad_compat (B, 2, M, M) (matrices) per image."""
        B = grad_q.shape[0]
        check(self._L.dsrg_crf_backward_wide_dev(self.h, _dptr(q_hist), B, _dptr(image), C.byref(params),
                                                 _dptr(potts), _dptr(compat), _dptr(grad_q), _dptr(grad_unary),
                                                 _dptr(grad_potts), _dptr(grad_compat), _stream(stream)))
        return grad_unary

    def crf_backward_wide_theta_dev(self, q_hist, image, params, grad_q, grad_unary, grad_theta, potts=None,
                                    compat=None, grad_potts=None, grad_compat=None, stream=None):
        """crf_backward_wide_dev that also writes grad_theta (B, 7) as crf_backward_theta_dev does; its forward is
        crf_forward_train_wide_dev with the same params."""
        B = grad_q.shape[0]
        check(self._L.dsrg_crf_backward_wide_theta_dev(self.h, _dptr(q_hist), B, _dptr(image), C.byref(params),
                                                       _dptr(potts), _dptr(compat), _dptr(grad_q), _dptr(grad_unary),
                                                       _dptr(grad_potts), _dptr(grad_compat), _dptr(grad_theta),
                                                       _stream(stream)))
        return grad_unary

    def crf_forward_train_wide_feat_dev(self, unary, features, params, q_hist, potts=None, compat=None, stream=None):
        """crf_forward_train_feat_dev above 32 labels (33 to 255), on the label-chunked kernels."""
        B = unary.shape[0]
        check(self._L.dsrg_crf_forward_train_wide_feat_dev(self.h, _dptr(unary), B, _dptr(features), C.byref(params),
                                                           _dptr(potts), _dptr(compat), _dptr(q_hist),
                                                           _stream(stream)))
        return q_hist

    def crf_backward_wide_feat_dev(self, q_hist, features, params, grad_q, grad_unary, grad_features, potts=None,
                                   compat=None, grad_potts=None, grad_compat=None, grad_theta_sp=None, stream=None):
        """The backward of crf_forward_train_wide_feat_dev, with crf_backward_feat_dev's outputs."""
        B = grad_q.shape[0]
        check(self._L.dsrg_crf_backward_wide_feat_dev(self.h, _dptr(q_hist), B, _dptr(features), C.byref(params),
                                                      _dptr(potts), _dptr(compat), _dptr(grad_q), _dptr(grad_unary),
                                                      _dptr(grad_features), _dptr(grad_potts), _dptr(grad_compat),
                                                      _dptr(grad_theta_sp), _stream(stream)))
        return grad_unary

    def feature_range_flags(self, B):
        """(B,) bool: which images of the engine's last feature pass (a batch of B) had lattice keys outside the packed
        range, and so NaN results.  Synchronises the device."""
        out = np.zeros(B, np.int32)
        check(self._L.dsrg_engine_feature_range_flags(self.h, B, _hptr(out, np.int32)))
        return out.astype(bool)

    def crf_learned_dev(self, unary, image, params, out, features=None, compat=None, unary_layout=LAYOUT_NHWC,
                        out_layout=LAYOUT_NHWC, stream=None):
        """crf_dev with the learned CRF: compat an optional device float32 (2, M, M) {mu_bi, mu_sp} in place of params.w1
        / w2, features optional (B, 5, H, W) float32 bilateral features in place of the image (then None).  Only the
        marginals are kept; a feature image whose lattice keys leave the packed range gets NaN (feature_range_flags)."""
        B = unary.shape[0]
        check(self._L.dsrg_crf_batch_learned_dev(self.h, _dptr(unary), B, unary_layout, _dptr(image), _dptr(features),
                                                 C.byref(params), _dptr(compat), _dptr(out), out_layout,
                                                 _stream(stream)))
        return out

    def crf_map_dev(self, unary, image, params, labels_out, unary_layout=LAYOUT_NHWC, stream=None):
        B = image.shape[0]
        check(self._L.dsrg_crf_map_batch_dev(self.h, B, _dptr(unary), unary_layout, _dptr(image), C.byref(params),
                                             _dptr(labels_out), _stream(stream)))
        return labels_out

    def srg_dev(self, labels, probs, cues, th1, th2, seeds_out, renorm=False, label_map_out=None, stream=None):
        B = probs.shape[0]
        check(self._L.dsrg_srg_batch_dev(self.h, B, _dptr(labels), _dptr(probs), _dptr(cues), float(th1), float(th2),
                                         int(bool(renorm)), _dptr(seeds_out), _dptr(label_map_out), _stream(stream)))
        return seeds_out

    def dsrg_forward_dev(self, labels, probs, cues, image, params, th1, th2, seeds_out, crf_out=None, stream=None):
        B = probs.shape[0]
        check(self._L.dsrg_dsrg_forward_dev(self.h, B, _dptr(labels), _dptr(probs), _dptr(cues), _dptr(image),
                                            C.byref(params), float(th1), float(th2), _dptr(seeds_out),
                                            _dptr(crf_out), _stream(stream)))
        return seeds_out

    def crflayer_forward_dev(self, probs, image, params, log_out, result=None, stream=None):
        B = probs.shape[0]
        check(self._L.dsrg_crflayer_forward_dev(self.h, B, _dptr(probs), _dptr(image), C.byref(params),
                                                _dptr(log_out), _dptr(result), _stream(stream)))
        return log_out

    def crflayer_backward_dev(self, result, top_diff, grad_out, stream=None):
        """CRFLayer.backward: grad_out = (1 - result) * top_diff in float32, bit-identical to numpy."""
        B = result.shape[0]
        check(self._L.dsrg_crflayer_backward_dev(self.h, _dptr(result), _dptr(top_diff), B, _dptr(grad_out),
                                                 _stream(stream)))
        return grad_out

    def srg_last_crf_dev(self, labels, cues, th1, th2, seeds_out, stream=None):
        """SRG on the marginals of this engine's last CRF pass, on device arrays (one refinement, two consumers)."""
        B = cues.shape[0]
        check(self._L.dsrg_srg_last_crf_dev(self.h, _dptr(labels), _dptr(cues), B, float(th1), float(th2),
                                            _dptr(seeds_out), _stream(stream)))
        return seeds_out

    # ---- SoftmaxLayer / ConstrainLossLayer (device arrays) ----
    def softmax_forward_dev(self, preds, probs_out, stream=None):
        check(self._L.dsrg_softmax_forward_dev(self.h, preds.shape[0], _dptr(preds), _dptr(probs_out),
                                               _stream(stream)))
        return probs_out

    def softmax_backward_dev(self, preds, top_diff, grad_out, stream=None):
        check(self._L.dsrg_softmax_backward_dev(self.h, preds.shape[0], _dptr(preds), _dptr(top_diff),
                                                _dptr(grad_out), _stream(stream)))
        return grad_out

    def constrainloss_forward_dev(self, probs, log_smooth, loss_out, stream=None):
        """loss_out: one float32 on the device."""
        check(self._L.dsrg_constrainloss_forward_dev(self.h, probs.shape[0], _dptr(probs), _dptr(log_smooth),
                                                     _dptr(loss_out), _stream(stream)))
        return loss_out

    def constrainloss_backward_dev(self, probs, log_smooth, grad_probs, grad_log, stream=None):
        check(self._L.dsrg_constrainloss_backward_dev(self.h, probs.shape[0], _dptr(probs), _dptr(log_smooth),
                                                      _dptr(grad_probs), _dptr(grad_log), _stream(stream)))
        return grad_probs, grad_log

    def seedloss_forward_dev(self, probs, seeds, terms_out, stream=None):
        B = probs.shape[0]
        check(self._L.dsrg_seedloss_forward_dev(self.h, B, _dptr(probs), _dptr(seeds), _dptr(terms_out), _stream(stream)))
        return terms_out

    def seedloss_backward_dev(self, probs, seeds, grad_out, n_global=None, top_diff=1.0, stream=None):
        B = probs.shape[0]
        check(self._L.dsrg_seedloss_backward_dev(self.h, B, int(n_global or B), _dptr(probs), _dptr(seeds),
                                                 float(top_diff), _dptr(grad_out), _stream(stream)))
        return grad_out

    # ---- SEC losses: SeedLossLayer / ExpandLossLayer (pylayers.py:95-118, :183-233) ----
    def seedloss_plain_forward_dev(self, probs, seeds, terms_out, stream=None):
        """terms_out[0] = sum_n S(n) / cnt(n); loss = -terms[0] / N_global."""
        B = probs.shape[0]
        check(self._L.dsrg_seedloss_plain_forward_dev(self.h, B, _dptr(probs), _dptr(seeds), _dptr(terms_out),
                                                      _stream(stream)))
        return terms_out

    def seedloss_plain_backward_dev(self, probs, seeds, grad_out, n_global=None, stream=None):
        B = probs.shape[0]
        check(self._L.dsrg_seedloss_plain_backward_dev(self.h, B, int(n_global or B), _dptr(probs), _dptr(seeds),
                                                       _dptr(grad_out), _stream(stream)))
        return grad_out

    def expandloss_forward_dev(self, probs, labels, terms_out, q_fg=0.996, q_bg=0.999, stream=None):
        """terms_out (3 floats): the local sums of the three terms; loss = -sum(terms) / N_global."""
        B = probs.shape[0]
        check(self._L.dsrg_expandloss_forward_dev(self.h, B, _dptr(probs), _dptr(labels), float(q_fg), float(q_bg),
                                                  _dptr(terms_out), _stream(stream)))
        return terms_out

    def expandloss_backward_dev(self, probs, labels, grad_out, n_global=None, q_fg=0.996, q_bg=0.999, stream=None):
        B = probs.shape[0]
        check(self._L.dsrg_expandloss_backward_dev(self.h, B, int(n_global or B), _dptr(probs), _dptr(labels),
                                                   float(q_fg), float(q_bg), _dptr(grad_out), _stream(stream)))
        return grad_out

    def seedloss_plain_forward_host(self, probs, seeds):
        terms = np.zeros(1, np.float32)
        check(self._L.dsrg_seedloss_plain_forward_host(self.h, probs.shape[0], _hptr(probs, np.float32),
                                                       _hptr(seeds, np.float32), _hptr(terms, np.float32)))
        return terms

    def seedloss_plain_backward_host(self, probs, seeds, n_global=None, grad=None):
        if grad is None:
            grad = np.empty(probs.shape, np.float32)
        check(self._L.dsrg_seedloss_plain_backward_host(self.h, probs.shape[0], int(n_global or probs.shape[0]),
                                                        _hptr(probs, np.float32), _hptr(seeds, np.float32),
                                                        _hptr(grad, np.float32)))
        return grad

    def expandloss_forward_host(self, probs, labels, q_fg=0.996, q_bg=0.999):
        """labels: (B,1,1,M) or (B,M) float32 -> the three local sums (see expandloss_forward_dev)."""
        terms = np.zeros(3, np.float32)
        check(self._L.dsrg_expandloss_forward_host(self.h, probs.shape[0], _hptr(probs, np.float32),
                                                   _hptr(labels, np.float32), float(q_fg), float(q_bg),
                                                   _hptr(terms, np.float32)))
        return terms

    def expandloss_backward_host(self, probs, labels, n_global=None, q_fg=0.996, q_bg=0.999, grad=None):
        if grad is None:
            grad = np.empty(probs.shape, np.float32)
        check(self._L.dsrg_expandloss_backward_host(self.h, probs.shape[0], int(n_global or probs.shape[0]),
                                                    _hptr(probs, np.float32), _hptr(labels, np.float32),
                                                    float(q_fg), float(q_bg), _hptr(grad, np.float32)))
        return grad

    # ---- host entry points (numpy; H2D / D2H inside the call) ----
    def crf_host(self, unary, image, params, out=None, unary_layout=LAYOUT_NHWC, out_layout=LAYOUT_NHWC):
        B = image.shape[0]
        if out is None:
            shape = (B, self.H, self.W, self.M) if out_layout == LAYOUT_NHWC else (B, self.M, self.H, self.W)
            out = np.empty(shape, np.float32)
        check(self._L.dsrg_crf_batch_host(self.h, B, _hptr(unary, np.float32), unary_layout, _hptr(image, np.uint8),
                                          C.byref(params), _hptr(out, np.float32), out_layout))
        return out

    def srg_host(self, labels, probs, cues, th1, th2, renorm=False, seeds_out=None, label_map_out=None):
        B = probs.shape[0]
        if seeds_out is None:
            seeds_out = np.empty(probs.shape, np.float32)
        check(self._L.dsrg_srg_batch_host(self.h, B, _hptr(labels, np.float32), _hptr(probs, np.float32),
                                          _hptr(cues, np.float32), float(th1), float(th2), int(bool(renorm)),
                                          _hptr(seeds_out, np.float32), _hptr(label_map_out, np.int32)))
        return seeds_out

    def dsrg_forward_host(self, labels, probs, cues, image, params, th1, th2, seeds_out=None, crf_out=None):
        B = probs.shape[0]
        if seeds_out is None:
            seeds_out = np.empty(probs.shape, np.float32)
        check(self._L.dsrg_dsrg_forward_host(self.h, B, _hptr(labels, np.float32), _hptr(probs, np.float32),
                                             _hptr(cues, np.float32), _hptr(image, np.uint8), C.byref(params),
                                             float(th1), float(th2), _hptr(seeds_out, np.float32),
                                             _hptr(crf_out, np.float32)))
        return seeds_out

    # ---- SoftmaxLayer / ConstrainLossLayer (host blobs) ----
    def softmax_forward_host(self, preds):
        out = np.empty(preds.shape, np.float32)
        check(self._L.dsrg_softmax_forward_host(self.h, preds.shape[0], _hptr(preds, np.float32), _hptr(out, np.float32)))
        return out

    def softmax_backward_host(self, preds, top_diff):
        out = np.empty(preds.shape, np.float32)
        check(self._L.dsrg_softmax_backward_host(self.h, preds.shape[0], _hptr(preds, np.float32),
                                                 _hptr(top_diff, np.float32), _hptr(out, np.float32)))
        return out

    def constrainloss_forward_host(self, probs, log_smooth):
        out = np.zeros(1, np.float32)
        check(self._L.dsrg_constrainloss_forward_host(self.h, probs.shape[0], _hptr(probs, np.float32),
                                                      _hptr(log_smooth, np.float32), _hptr(out, np.float32)))
        return float(out[0])

    def constrainloss_backward_host(self, probs, log_smooth):
        gp, gl = np.empty(probs.shape, np.float32), np.empty(probs.shape, np.float32)
        check(self._L.dsrg_constrainloss_backward_host(self.h, probs.shape[0], _hptr(probs, np.float32),
                                                       _hptr(log_smooth, np.float32), _hptr(gp, np.float32),
                                                       _hptr(gl, np.float32)))
        return gp, gl

    def prepare_image_host(self, images, mean_pixel=(104.0, 117.0, 123.0), out=None):
        """(B,3,Hi,Wi) float32 network input -> (B,H,W,3) uint8 CRF image (pylayers.py:315-319 + CRF.py:32)."""
        B, _, Hi, Wi = images.shape
        if out is None:
            out = np.empty((B, self.H, self.W, 3), np.uint8)
        mean = np.asarray(mean_pixel, np.float64)
        check(self._L.dsrg_prepare_image_host(self.h, B, Hi, Wi, _hptr(images, np.float32), _hptr(mean, np.float64),
                                              _hptr(out, np.uint8)))
        return out

    def prepare_image_dev(self, images, out, mean_pixel=(104.0, 117.0, 123.0), stream=None):
        B, _, Hi, Wi = images.shape
        mean = np.asarray(mean_pixel, np.float64)
        check(self._L.dsrg_prepare_image_dev(self.h, B, Hi, Wi, _dptr(images), _hptr(mean, np.float64), _dptr(out),
                                             _stream(stream)))
        return out

    # ---- network input of the evaluation tools (training/tools/test-ms.py:68-81 and its siblings) ----
    @staticmethod
    def _net_input_args(sizes, mean_pixel):
        n = len(sizes)
        hs = (C.c_int * n)(*[int(h) for h, _ in sizes])
        ws = (C.c_int * n)(*[int(w) for _, w in sizes])
        mean = np.ascontiguousarray(mean_pixel, np.float64)
        if mean.shape != (3,):
            raise ValueError("mean_pixel must have 3 elements")
        return n, hs, ws, mean

    def prepare_net_input_host(self, image, sizes, mean_pixel=(104.0, 117.0, 123.0)):
        """(H,W,3) uint8 image -> one (1,3,h,w) float32 network input per (h, w) of `sizes`: preprocess(image, size)
        of the evaluation tools, bit-exact.  Does not change the engine's size."""
        H, W = image.shape[:2]
        n, hs, ws, mean = self._net_input_args(sizes, mean_pixel)
        outs = [np.empty((1, 3, h, w), np.float32) for h, w in zip(hs, ws)]
        ptrs = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
        check(self._L.dsrg_prepare_net_input_host(self.h, _hptr(image, np.uint8), int(H), int(W), n, hs, ws,
                                                  _hptr(mean, np.float64), ptrs))
        return outs

    def prepare_net_input_dev(self, image, outs, mean_pixel=(104.0, 117.0, 123.0), stream=None):
        """image: (H,W,3) uint8 CUDA tensor; outs: float32 CUDA tensors of shape (3,h,w) or (1,3,h,w), one per
        scale (their shapes give the sizes)."""
        import torch
        if image.dtype != torch.uint8 or image.dim() != 3 or image.shape[2] != 3:
            raise ValueError("image must be an (H, W, 3) uint8 tensor")
        for o in outs:
            if o.dtype != torch.float32 or o.dim() < 3 or o.numel() != 3 * o.shape[-2] * o.shape[-1]:
                raise ValueError("every output must be a float32 (3, h, w) or (1, 3, h, w) tensor")
        n, hs, ws, mean = self._net_input_args([(o.shape[-2], o.shape[-1]) for o in outs], mean_pixel)
        ptrs = (C.c_void_p * n)(*[_dptr(o).value for o in outs])
        check(self._L.dsrg_prepare_net_input_dev(self.h, _dptr(image), int(image.shape[0]), int(image.shape[1]), n,
                                                 hs, ws, _hptr(mean, np.float64), ptrs, _stream(stream)))
        return outs

    @staticmethod
    def _image_sizes(images):
        B = len(images)
        Hs = (C.c_int * B)(*[int(im.shape[0]) for im in images])
        Ws = (C.c_int * B)(*[int(im.shape[1]) for im in images])
        return B, Hs, Ws

    def prepare_net_input_batch_host(self, images, sizes, mean_pixel=(104.0, 117.0, 123.0)):
        """List of B (H_i,W_i,3) uint8 images -> one (B,3,h,w) float32 network input per (h, w) of `sizes`; image b
        of each is bit-identical to prepare_net_input_host of that image alone.  Does not change the engine's size."""
        B, Hs, Ws = self._image_sizes(images)
        n, hs, ws, mean = self._net_input_args(sizes, mean_pixel)
        ims = (C.c_void_p * B)(*[_hptr(im, np.uint8).value for im in images])
        outs = [np.empty((B, 3, h, w), np.float32) for h, w in zip(hs, ws)]
        ptrs = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
        check(self._L.dsrg_prepare_net_input_batch_host(self.h, ims, Hs, Ws, B, n, hs, ws, _hptr(mean, np.float64),
                                                        ptrs))
        return outs

    def prepare_net_input_batch_dev(self, images, outs, mean_pixel=(104.0, 117.0, 123.0), stream=None):
        """images: list of B contiguous (H_i,W_i,3) uint8 CUDA tensors; outs: one contiguous (B,3,h,w) float32 CUDA
        tensor per scale (their shapes give the sizes).  Queued on `stream`; copies nothing from the host."""
        import torch
        for im in images:
            if im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3:
                raise ValueError("every image must be an (H, W, 3) uint8 tensor")
        for o in outs:
            if o.dtype != torch.float32 or o.dim() != 4 or o.shape[:2] != (len(images), 3):
                raise ValueError("every output must be a float32 (B, 3, h, w) tensor with B = %d" % len(images))
        B, Hs, Ws = self._image_sizes(images)
        n, hs, ws, mean = self._net_input_args([(o.shape[2], o.shape[3]) for o in outs], mean_pixel)
        ims = (C.c_void_p * B)(*[_dptr(im).value for im in images])
        ptrs = (C.c_void_p * n)(*[_dptr(o).value for o in outs])
        check(self._L.dsrg_prepare_net_input_batch_dev(self.h, ims, Hs, Ws, B, n, hs, ws, _hptr(mean, np.float64),
                                                       ptrs, _stream(stream)))
        return outs

    def crflayer_forward_host(self, probs, image, params, log_out=None, result=None):
        B = probs.shape[0]
        if log_out is None:
            log_out = np.empty(probs.shape, np.float32)
        check(self._L.dsrg_crflayer_forward_host(self.h, B, _hptr(probs, np.float32), _hptr(image, np.uint8),
                                                 C.byref(params), _hptr(log_out, np.float32), _hptr(result, np.float32)))
        return log_out

    def srg_last_crf_host(self, labels, cues, th1, th2, seeds_out=None):
        """SRG on the marginals of this engine's last CRF pass (one refinement, two consumers)."""
        B = cues.shape[0]
        if seeds_out is None:
            seeds_out = np.empty(cues.shape, np.float32)
        check(self._L.dsrg_srg_last_crf_host(self.h, B, _hptr(labels, np.float32), _hptr(cues, np.float32),
                                             float(th1), float(th2), _hptr(seeds_out, np.float32)))
        return seeds_out

    def crf_last_marginals_host(self, B, layout=None):
        layout = _lib.LAYOUT_NCHW if layout is None else layout
        shape = (B, self.M, self.H, self.W) if layout == _lib.LAYOUT_NCHW else (B, self.H, self.W, self.M)
        out = np.empty(shape, np.float32)
        check(self._L.dsrg_crf_last_marginals_host(self.h, B, _hptr(out, np.float32), int(layout)))
        return out

    def seedloss_forward_host(self, probs, seeds):
        """(term_bg, term_fg) local sums; loss = -(term_bg + term_fg) / N_global."""
        terms = np.zeros(2, np.float32)
        check(self._L.dsrg_seedloss_forward_host(self.h, probs.shape[0], _hptr(probs, np.float32),
                                                 _hptr(seeds, np.float32), _hptr(terms, np.float32)))
        return terms

    def seedloss_backward_host(self, probs, seeds, n_global=None, top_diff=1.0, grad=None):
        if grad is None:
            grad = np.empty(probs.shape, np.float32)
        check(self._L.dsrg_seedloss_backward_host(self.h, probs.shape[0], int(n_global or probs.shape[0]),
                                                  _hptr(probs, np.float32), _hptr(seeds, np.float32),
                                                  float(top_diff), _hptr(grad, np.float32)))
        return grad

    # ---- inference post-processing (training/tools/test-ms.py, generate_train_gt.py) ----
    def zoom_scores_host(self, scores, out=None, accumulate=False):
        """(M,h,w) float32 blob -> (H,W,M): nd.zoom(scores.transpose(1,2,0), (H/h, W/w, 1), order=1), bit-exact."""
        M, h, w = scores.shape
        if out is None:
            if accumulate:
                raise ValueError("accumulate needs `out`")
            out = np.empty((self.H, self.W, self.M), np.float32)
        check(self._L.dsrg_zoom_scores_host(self.h, _hptr(scores, np.float32), h, w, _hptr(out, np.float32),
                                            int(bool(accumulate))))
        return out

    def zoom_scores_dev(self, scores, out, accumulate=False, stream=None):
        M, h, w = scores.shape
        check(self._L.dsrg_zoom_scores_dev(self.h, _dptr(scores), h, w, _dptr(out), int(bool(accumulate)),
                                           _stream(stream)))
        return out

    @staticmethod
    def _post_args(scores, labels_sel):
        n = len(scores)
        hs = (C.c_int * n)(*[int(a.shape[1]) for a in scores])
        ws = (C.c_int * n)(*[int(a.shape[2]) for a in scores])
        sel = np.ascontiguousarray(labels_sel if labels_sel is not None else [], np.int32)
        return n, hs, ws, sel

    def predict_mask_host(self, scores, image, params=None, mode=POST_SUM_SCORES, eps=0.00001, smooth=True,
                          labels_sel=None, want_probs=False):
        """scores: list of (M,h,w) float32 blobs; image (H,W,3) uint8 -> (H,W) int32 label map
        [, (H,W,M) float32 probabilities]."""
        n, hs, ws, sel = self._post_args(scores, labels_sel)
        ptrs = (C.c_void_p * n)(*[_hptr(a, np.float32).value for a in scores])
        result = np.empty((self.H, self.W), np.int32)
        probs = np.empty((self.H, self.W, self.M), np.float32) if want_probs else None
        params = params if params is not None else crf_params()
        check(self._L.dsrg_predict_mask_host(self.h, int(mode), n, ptrs, hs, ws, _hptr(image, np.uint8), float(eps),
                                             int(bool(smooth)), C.byref(params), _hptr(sel, np.int32), int(sel.size),
                                             _hptr(result, np.int32), _hptr(probs, np.float32)))
        return (result, probs) if want_probs else result

    def predict_mask_dev(self, scores, image, result_out, params=None, mode=POST_SUM_SCORES, eps=0.00001,
                         smooth=True, labels_sel=None, probs_out=None, stream=None):
        n, hs, ws, sel = self._post_args(scores, labels_sel)
        ptrs = (C.c_void_p * n)(*[_dptr(a).value for a in scores])
        params = params if params is not None else crf_params()
        check(self._L.dsrg_predict_mask_dev(self.h, int(mode), n, ptrs, hs, ws, _dptr(image), float(eps),
                                            int(bool(smooth)), C.byref(params), _hptr(sel, np.int32), int(sel.size),
                                            _dptr(result_out), _dptr(probs_out), _stream(stream)))
        return result_out

    @staticmethod
    def _post_batch_args(scores):
        n = len(scores)
        if not 1 <= n <= 16:
            raise ValueError("between 1 and 16 score maps, not %d" % n)
        if any(len(a.shape) != 4 or tuple(a.shape[:2]) != tuple(scores[0].shape[:2]) for a in scores):
            raise ValueError("every score map must be (B, M, h, w) with the same B and M")
        hs = (C.c_int * n)(*[int(a.shape[2]) for a in scores])
        ws = (C.c_int * n)(*[int(a.shape[3]) for a in scores])
        return n, int(scores[0].shape[0]), hs, ws

    def predict_mask_batch_host(self, scores, images, params=None, mode=POST_SUM_SCORES, eps=0.00001, smooth=True,
                                sel=None, want_probs=False):
        """scores: list of (B,M,h,w) float32 arrays, one per scale; images (B,H,W,3) uint8 (None when not smooth);
        sel: optional (B,M) int32 rows of label ids ending at the first -1 -> (B,H,W) int32 label maps
        [, (B,H,W,M) float32 probabilities]."""
        n, B, hs, ws = self._post_batch_args(scores)
        ptrs = (C.c_void_p * n)(*[_hptr(a, np.float32).value for a in scores])
        result = np.empty((B, self.H, self.W), np.int32)
        probs = np.empty((B, self.H, self.W, self.M), np.float32) if want_probs else None
        params = params if params is not None else crf_params()
        check(self._L.dsrg_predict_mask_batch_host(self.h, ptrs, hs, ws, n, B, int(mode), _hptr(images, np.uint8),
                                                   float(eps), int(bool(smooth)), C.byref(params),
                                                   _hptr(sel, np.int32), _hptr(result, np.int32),
                                                   _hptr(probs, np.float32)))
        return (result, probs) if want_probs else result

    def predict_mask_batch_dev(self, scores, images, result_out, params=None, mode=POST_SUM_SCORES, eps=0.00001,
                               smooth=True, sel=None, probs_out=None, stream=None):
        """The same on CUDA tensors, queued on `stream`: result_out (B,H,W) int32, probs_out optional (B,H,W,M)
        float32, sel an optional (B,M) int32 tensor read when the pass runs."""
        n, B, hs, ws = self._post_batch_args(scores)
        ptrs = (C.c_void_p * n)(*[_dptr(a).value for a in scores])
        params = params if params is not None else crf_params()
        check(self._L.dsrg_predict_mask_batch_dev(self.h, ptrs, hs, ws, n, B, int(mode), _dptr(images), float(eps),
                                                  int(bool(smooth)), C.byref(params), _dptr(sel), _dptr(result_out),
                                                  _dptr(probs_out), _stream(stream)))
        return result_out

    def predict_mask_batch_learned_dev(self, scores, images, result_out, params, mode=POST_SUM_SCORES, eps=0.00001,
                                       features=None, compat=None, sel=None, probs_out=None, stream=None):
        """predict_mask_batch_dev (smooth) with the learned CRF of crf_learned_dev: images (B,H,W,3) uint8 or
        features (B,5,H,W) float32 (exactly one), compat optional (2, M, M).  A feature image whose lattice keys leave
        the packed range gets -1 in every pixel of its result and NaN in probs_out."""
        n, B, hs, ws = self._post_batch_args(scores)
        ptrs = (C.c_void_p * n)(*[_dptr(a).value for a in scores])
        check(self._L.dsrg_predict_mask_batch_learned_dev(self.h, ptrs, hs, ws, n, B, int(mode), _dptr(images),
                                                          _dptr(features), float(eps), C.byref(params), _dptr(compat),
                                                          _dptr(sel), _dptr(result_out), _dptr(probs_out),
                                                          _stream(stream)))
        return result_out

    # ---- AnnotationLayer.forward (pylayers.py:369-387) ----
    @staticmethod
    def _annot_args(tags, cues, flip):
        """tags: per image 1-D class ids; cues: per image (3,K) int arrays (class,row,col) -> CSR int32."""
        B = len(tags)
        toff = np.zeros(B + 1, np.int32)
        coff = np.zeros(B + 1, np.int32)
        for i in range(B):
            toff[i + 1] = toff[i] + np.asarray(tags[i]).size
            coff[i + 1] = coff[i] + np.asarray(cues[i]).reshape(3, -1).shape[1]
        tg = np.ascontiguousarray(np.concatenate([np.asarray(t).reshape(-1) for t in tags]) if toff[B] else [], np.int32)
        ci = np.ascontiguousarray(np.concatenate([np.asarray(c).reshape(3, -1) for c in cues], axis=1) if coff[B]
                                  else np.zeros((3, 0)), np.int32)
        fl = None if flip is None else np.ascontiguousarray(flip, np.int32)
        return B, toff, tg, coff, ci, fl

    def annotation_forward_host(self, tags, cues, flip=None, images=None):
        """-> labels (B,1,1,M), cues (B,M,H,W)[, images (B,3,Hi,Wi)] float32."""
        B, toff, tg, coff, ci, fl = self._annot_args(tags, cues, flip)
        labels = np.empty((B, 1, 1, self.M), np.float32)
        dense = np.empty((B, self.M, self.H, self.W), np.float32)
        out_im = None if images is None else np.empty(images.shape, np.float32)
        Hi, Wi = (0, 0) if images is None else images.shape[2:]
        check(self._L.dsrg_annotation_forward_host(self.h, B, _hptr(toff, np.int32), _hptr(tg, np.int32),
                                                   _hptr(coff, np.int32), _hptr(ci, np.int32), _hptr(fl, np.int32),
                                                   _hptr(images, np.float32), Hi, Wi, _hptr(labels, np.float32),
                                                   _hptr(dense, np.float32), _hptr(out_im, np.float32)))
        return (labels, dense) if images is None else (labels, dense, out_im)

    def annotation_forward_dev(self, tags, cues, labels_out, cues_out, flip=None, images=None, images_out=None,
                               stream=None):
        B, toff, tg, coff, ci, fl = self._annot_args(tags, cues, flip)
        Hi, Wi = (0, 0) if images is None else images.shape[2:]
        check(self._L.dsrg_annotation_forward_dev(self.h, B, _hptr(toff, np.int32), _hptr(tg, np.int32),
                                                  _hptr(coff, np.int32), _hptr(ci, np.int32), _hptr(fl, np.int32),
                                                  _dptr(images), Hi, Wi, _dptr(labels_out), _dptr(cues_out),
                                                  _dptr(images_out), _stream(stream)))
        return labels_out, cues_out

    # ---- AnnotationLayerCOCO.forward (pylayers.py:432-512) ----
    @staticmethod
    def _coco_args(shapes, flip, new_size, mean_pixel):
        B = len(shapes)
        Hs = (C.c_int * B)(*[int(s[0]) for s in shapes])
        Ws = (C.c_int * B)(*[int(s[1]) for s in shapes])
        fl = None if flip is None else np.ascontiguousarray(flip, np.int32)
        if fl is not None and fl.shape != (B,):
            raise ValueError("flip must have one entry per image")
        mean = np.ascontiguousarray(mean_pixel, np.float64)
        if mean.shape != (3,):
            raise ValueError("mean_pixel must have 3 elements")
        new_h, new_w = (int(v) for v in new_size)
        return B, Hs, Ws, fl, mean, new_h, new_w

    def annotation_coco_forward_host(self, images, label_maps, new_size, mean_pixel, flip=None, ignore_label=255,
                                     out=None):
        """images: B (H_b, W_b, 3) uint8 BGR arrays; label_maps: (B, H, W) uint8 at the engine's size ->
        labels (B,1,1,M), cues (B,M,H,W), images (B,3,new_h,new_w) float32, written into `out` when it is given
        (three C-contiguous float32 arrays of those shapes).  A label value >= M other than ignore_label raises
        DsrgError with numpy's IndexError message."""
        for im in images:
            _hptr(im, np.uint8)
            if im.ndim != 3 or im.shape[2] != 3:
                raise ValueError("every image must be an (H, W, 3) uint8 array")
        B, Hs, Ws, fl, mean, new_h, new_w = self._coco_args([im.shape for im in images], flip, new_size, mean_pixel)
        if label_maps.shape != (B, self.H, self.W):
            raise ValueError("label_maps must have shape (%d, %d, %d)" % (B, self.H, self.W))
        if out is None:
            out = (np.empty((B, 1, 1, self.M), np.float32), np.empty((B, self.M, self.H, self.W), np.float32),
                   np.empty((B, 3, new_h, new_w), np.float32))
        ptrs = (C.c_void_p * B)(*[im.ctypes.data for im in images])
        check(self._L.dsrg_annotation_coco_forward_host(
            self.h, ptrs, Hs, Ws, B, _hptr(label_maps, np.uint8), _hptr(fl, np.int32), new_h, new_w,
            _hptr(mean, np.float64), int(ignore_label), _hptr(out[0], np.float32), _hptr(out[1], np.float32),
            _hptr(out[2], np.float32)))
        return out

    def annotation_coco_forward_dev(self, images, label_maps, labels_out, cues_out, images_out, mean_pixel,
                                    flip=None, ignore_label=255, bad_out=None, stream=None):
        """images: B (H_b, W_b, 3) uint8 CUDA tensors; label_maps: (B, H, W) uint8 CUDA tensor; the outputs are
        float32 CUDA tensors, images_out (B, 3, new_h, new_w) giving the size.  bad_out: optional (B,) int32 CUDA
        tensor, per image the raster index of the first label value >= M other than ignore_label, or -1."""
        import torch
        for im in images:
            if im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3:
                raise ValueError("every image must be an (H, W, 3) uint8 tensor")
        if images_out.dim() != 4:
            raise ValueError("images_out must be a (B, 3, new_h, new_w) tensor")
        B, Hs, Ws, fl, mean, new_h, new_w = self._coco_args([im.shape for im in images], flip,
                                                            images_out.shape[2:], mean_pixel)
        ptrs = (C.c_void_p * B)(*[_dptr(im).value for im in images])
        check(self._L.dsrg_annotation_coco_forward_dev(
            self.h, ptrs, Hs, Ws, B, _dptr(label_maps), _hptr(fl, np.int32), new_h, new_w, _hptr(mean, np.float64),
            int(ignore_label), _dptr(labels_out), _dptr(cues_out), _dptr(images_out), _dptr(bad_out),
            _stream(stream)))
        return labels_out, cues_out, images_out

    # ---- ImageSegDataLayer.forward (layer.py:51-61, SimpleTransformer :147-236) ----
    @staticmethod
    def _seg_args(image_shapes, label_shapes, h_off, w_off, flip, mean):
        B = len(image_shapes)
        ints = lambda v: (C.c_int * B)(*[int(x) for x in v])  # noqa: E731
        if len(h_off) != B or len(w_off) != B or (label_shapes is not None and len(label_shapes) != B):
            raise ValueError("labels, h_off and w_off must have one entry per image")
        Hs, Ws = ints(s[0] for s in image_shapes), ints(s[1] for s in image_shapes)
        Hl = Wl = None
        if label_shapes is not None:
            Hl, Wl = ints(s[0] for s in label_shapes), ints(s[1] for s in label_shapes)
        fl = None if flip is None else np.ascontiguousarray(flip, np.int32)
        if fl is not None and fl.shape != (B,):
            raise ValueError("flip must have one entry per image")
        mean = np.ascontiguousarray(mean, np.float64)
        if mean.shape != (3,):
            raise ValueError("mean must have 3 elements")
        return B, Hs, Ws, Hl, Wl, ints(h_off), ints(w_off), fl, mean

    def seg_data_forward_host(self, images, labels, h_off, w_off, crop_size, mean, scale=1.0, flip=None,
                              swap_rb=False, pad_label=255, out=None):
        """images: B (H_b, W_b, 3) uint8 BGR arrays; labels: B (Hl_b, Wl_b) uint8 arrays, or None for the image-only
        paths; h_off, w_off: per image the window's corner in the padded arrays; flip: B 0/1 flags or None ->
        (images (B, 3, crop_h, crop_w), labels (B, 1, crop_h, crop_w) or None) float32, written into `out` when it is
        given (a pair of C-contiguous float32 arrays of those shapes, the second None without labels).  pad_label is
        the byte the label is padded with, saturate_cast<uchar>(ignore_label)."""
        for im in images:
            _hptr(im, np.uint8)
            if im.ndim != 3 or im.shape[2] != 3:
                raise ValueError("every image must be an (H, W, 3) uint8 array")
        if labels is not None:
            for lab in labels:
                _hptr(lab, np.uint8)
                if lab.ndim != 2:
                    raise ValueError("every label must be an (H, W) uint8 array")
        B, Hs, Ws, Hl, Wl, ho, wo, fl, mean = self._seg_args(
            [im.shape for im in images], None if labels is None else [lab.shape for lab in labels], h_off, w_off,
            flip, mean)
        crop_h, crop_w = (int(v) for v in crop_size)
        if out is None:
            out = (np.empty((B, 3, crop_h, crop_w), np.float32),
                   None if labels is None else np.empty((B, 1, crop_h, crop_w), np.float32))
        ptrs = (C.c_void_p * B)(*[im.ctypes.data for im in images])
        lptrs = None if labels is None else (C.c_void_p * B)(*[lab.ctypes.data for lab in labels])
        check(self._L.dsrg_seg_data_forward_host(
            self.h, ptrs, Hs, Ws, lptrs, Hl, Wl, B, ho, wo, _hptr(fl, np.int32), crop_h, crop_w,
            _hptr(mean, np.float64), float(scale), int(bool(swap_rb)), int(pad_label), _hptr(out[0], np.float32),
            _hptr(out[1], np.float32)))
        return out

    def seg_data_forward_dev(self, images, labels, h_off, w_off, images_out, labels_out, mean, scale=1.0, flip=None,
                             swap_rb=False, pad_label=255, stream=None):
        """images: B (H_b, W_b, 3) uint8 CUDA tensors; labels: B (Hl_b, Wl_b) uint8 CUDA tensors or None;
        images_out (B, 3, crop_h, crop_w), giving the crop size, and labels_out (B, 1, crop_h, crop_w) or None: float32
        CUDA tensors."""
        import torch
        for im in images:
            if im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3:
                raise ValueError("every image must be an (H, W, 3) uint8 tensor")
        if labels is not None:
            for lab in labels:
                if lab.dtype != torch.uint8 or lab.dim() != 2:
                    raise ValueError("every label must be an (H, W) uint8 tensor")
        if images_out.dim() != 4:
            raise ValueError("images_out must be a (B, 3, crop_h, crop_w) tensor")
        B, Hs, Ws, Hl, Wl, ho, wo, fl, mean = self._seg_args(
            [im.shape for im in images], None if labels is None else [lab.shape for lab in labels], h_off, w_off,
            flip, mean)
        ptrs = (C.c_void_p * B)(*[_dptr(im).value for im in images])
        lptrs = None if labels is None else (C.c_void_p * B)(*[_dptr(lab).value for lab in labels])
        crop_h, crop_w = (int(v) for v in images_out.shape[2:])
        check(self._L.dsrg_seg_data_forward_dev(
            self.h, ptrs, Hs, Ws, lptrs, Hl, Wl, B, ho, wo, _hptr(fl, np.int32), crop_h, crop_w,
            _hptr(mean, np.float64), float(scale), int(bool(swap_rb)), int(pad_label), _dptr(images_out),
            _dptr(labels_out), _stream(stream)))
        return images_out, labels_out

    # ---- per-kernel timing ----
    def profile(self, enable):
        check(self._L.dsrg_engine_profile(self.h, int(bool(enable))))

    def profile_read(self):
        """{kernel class: (total ms, launches)} since the last read (synchronises the device)."""
        n = self._L.dsrg_profile_tag_count()
        ms = np.zeros(n, np.float32)
        cnt = np.zeros(n, np.int64)
        check(self._L.dsrg_engine_profile_read(self.h, _hptr(ms, np.float32), _hptr(cnt, np.int64)))
        return {self._L.dsrg_profile_tag_name(t).decode(): (float(ms[t]), int(cnt[t])) for t in range(n) if cnt[t]}

    # ---- introspection ----
    def lattice_sizes(self, B):
        vs = np.zeros(1, np.int32)
        vb = np.zeros(B, np.int32)
        check(self._L.dsrg_engine_lattice_sizes(self.h, B, _hptr(vs, np.int32), _hptr(vb, np.int32)))
        return int(vs[0]), vb

    def lattice_tables(self, which, b):
        """Image b's lattice of the last CRF call (which = 0 spatial, 1 bilateral) in the engine's numbering:
        off (d+1, N) 1-based rows of every (r, pixel), nbr (d+1, V+1, 2) the blur neighbours of rows 0..V."""
        d = 2 if which == 0 else 5
        vs, vb = self.lattice_sizes(b + 1)
        V = vs if which == 0 else int(vb[b])
        off = np.zeros((d + 1, self.H * self.W), np.int32)
        nbr = np.zeros((d + 1, V + 1, 2), np.int32)
        check(self._L.dsrg_engine_lattice_tables(self.h, which, b, _hptr(off, np.int32), _hptr(nbr, np.int32)))
        return off, nbr

    def norms(self, B):
        ns = np.zeros(self.H * self.W, np.float32)
        nb = np.zeros((B, self.H * self.W), np.float32)
        check(self._L.dsrg_engine_copy_norm(self.h, 0, B, _hptr(ns, np.float32)))
        check(self._L.dsrg_engine_copy_norm(self.h, 1, B, _hptr(nb, np.float32)))
        return ns, nb

    def lattice_bary(self, which, b):
        """Image b's barycentric weights of the last CRF call (d+1, N), in the layout of lattice_tables' off."""
        d = 2 if which == 0 else 5
        bary = np.zeros((d + 1, self.H * self.W), np.float32)
        check(self._L.dsrg_engine_lattice_bary(self.h, which, b, _hptr(bary, np.float32)))
        return bary

    def lattice_idle(self, which):
        """(non-empty hash slots, hval entries not -1, vkey entries not kNoKey) of a lattice family, over its whole
        allocation: all 0 between passes.  Synchronises."""
        counts = np.zeros(3, np.int64)
        check(self._L.dsrg_engine_lattice_idle(self.h, which, _hptr(counts, np.int64)))
        return tuple(int(c) for c in counts)


def _pred_host(pred, K):
    """pred as a flat C-contiguous uint8 or int32 array.  Other integer predictions (np.argmax gives int64) are
    narrowed on the host: values outside [0, K) become -1, so they are counted as invalid and never wrapped."""
    pred = np.ascontiguousarray(pred).reshape(-1)
    if pred.dtype in (np.uint8, np.int32):
        return pred
    if pred.dtype.kind not in "iu":
        raise TypeError("pred must be an integer array, not %s" % pred.dtype)
    ok = (pred >= 0) & (pred < K)
    out = np.full(pred.size, -1, np.int32)
    out[ok] = pred[ok]
    return out


class Confusion(object):
    """dsrg_confusion: a K x K uint64 confusion matrix (row = gt, column = pred) on the device, plus the counters
    of pixels that were not binned -- invalid[0]: gt >= K other than 255, invalid[1]: gt < K with pred outside
    [0, K).  The rules are generateM's (training/tools/evaluate.py:61-68): pixels with gt >= K are skipped."""

    def __init__(self, K, device=None):
        self._L = _lib.lib()
        if device is None:
            device = self._L.dsrg_current_device()
        self.K, self.device = int(K), int(device)
        self.h = self._L.dsrg_confusion_create(self.device, self.K)
        if not self.h:
            raise DsrgError(_lib.E_CUDA, self._L.dsrg_last_error().decode())

    def close(self):
        if getattr(self, "h", None):
            self._L.dsrg_confusion_destroy(self.h)
            self.h = None

    __del__ = close

    def reset(self, stream=None):
        """Zero the matrix and the counters (stream None: the legacy default stream; ordered after every add)."""
        check(self._L.dsrg_confusion_reset(self.h, None if stream is None else C.c_void_p(int(stream))))

    def add_host(self, gt, pred):
        """gt: uint8 array; pred: uint8 / int32 (taken as they are) or any other integer array of the same size."""
        gt = np.ascontiguousarray(gt).reshape(-1)
        if gt.dtype != np.uint8:
            raise TypeError("gt must be uint8 (a label PNG), not %s" % gt.dtype)
        pred = _pred_host(pred, self.K)
        if pred.size != gt.size:
            raise ValueError("gt and pred differ in size (%d vs %d)" % (gt.size, pred.size))
        check(self._L.dsrg_confusion_add_host(self.h, gt.size, C.c_void_p(gt.ctypes.data),
                                              C.c_void_p(pred.ctypes.data), pred.itemsize))

    def add_dev(self, gt, pred, stream=None):
        """gt: contiguous uint8 CUDA tensor; pred: contiguous uint8 or int32 CUDA tensor of the same size."""
        import torch
        if gt.dtype != torch.uint8 or pred.dtype not in (torch.uint8, torch.int32):
            raise TypeError("gt must be uint8 and pred uint8 or int32 (got %s, %s)" % (gt.dtype, pred.dtype))
        if gt.numel() != pred.numel():
            raise ValueError("gt and pred differ in size (%d vs %d)" % (gt.numel(), pred.numel()))
        check(self._L.dsrg_confusion_add_dev(self.h, gt.numel(), _dptr(gt), _dptr(pred), pred.element_size(),
                                             _stream(stream)))

    def read(self):
        """(matrix (K, K) uint64, invalid (2,) uint64) after every add so far (synchronises)."""
        m = np.empty((self.K, self.K), np.uint64)
        inv = np.empty(2, np.uint64)
        check(self._L.dsrg_confusion_read(self.h, C.c_void_p(m.ctypes.data), C.c_void_p(inv.ctypes.data)))
        return m, inv


class DenseCRF(object):
    """Same surface as the reference's Cython extension type krahenbuhl2013.wrapper.DenseCRF
    (CRF/krahenbuhl2013/wrapper.pyx:20-60), backed by dsrg_densecrf_* (host pointers)."""

    def __init__(self, W, H, nlabels):
        self._L = _lib.lib()
        self.h = self._L.dsrg_densecrf_create(int(W), int(H), int(nlabels))
        if not self.h:
            raise DsrgError(_lib.E_CUDA, self._L.dsrg_last_error().decode())
        self._n = int(W) * int(H)
        self._m = int(nlabels)

    def __del__(self):
        if getattr(self, "h", None):
            self._L.dsrg_densecrf_destroy(self.h)
            self.h = None

    def set_unary_energy(self, unary_costs):
        u = np.ascontiguousarray(unary_costs, np.float32)  # float[:] memoryview in the reference
        if u.ndim != 1 or u.size != self._n * self._m:
            raise ValueError("unary_costs must be a flat float32 buffer of npixels*nlabels")
        check(self._L.dsrg_densecrf_set_unary_energy(self.h, _hptr(u, np.float32)))

    def add_pairwise_energy(self, w1, theta_alpha_1, theta_alpha_2, theta_betta_1, theta_betta_2, theta_betta_3,
                            w2, theta_gamma_1, theta_gamma_2, im):
        im = np.ascontiguousarray(im, np.uint8)  # unsigned char[:] in the reference
        if im.ndim != 1 or im.size != self._n * 3:
            raise ValueError("im must be a flat uint8 buffer of npixels*3")
        check(self._L.dsrg_densecrf_add_pairwise_energy(self.h, w1, theta_alpha_1, theta_alpha_2, theta_betta_1,
                                                        theta_betta_2, theta_betta_3, w2, theta_gamma_1,
                                                        theta_gamma_2, _hptr(im, np.uint8)))

    def map(self, n_iters=10):
        labels = np.empty(self._n, dtype=np.int32)
        check(self._L.dsrg_densecrf_map(self.h, int(n_iters), _hptr(labels, np.int32)))
        return labels

    def inference(self, n_iters=10):
        probs = np.empty(self._n * self._m, dtype=np.float32)
        check(self._L.dsrg_densecrf_inference(self.h, int(n_iters), _hptr(probs, np.float32)))
        return probs
