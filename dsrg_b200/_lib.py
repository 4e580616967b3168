"""ctypes loader of the C-ABI library (include/dsrg_b200.h).

The CUDA library is the product: if it is missing this module raises -- there is no CPU or
PyTorch fallback anywhere in the package.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DSRG_B200_LIB") or os.path.join(_HERE, "lib", "libdsrg_b200.so")  # env: A/B-test builds

OK, E_INVALID, E_CUDA, E_KEYRANGE, E_STATE, E_NOMEM = 0, -1, -2, -3, -4, -5
LAYOUT_NHWC, LAYOUT_NCHW = 0, 1
POST_SUM_SCORES, POST_ZOOM_PROBS = 0, 1
PREP_IMAGES_PER_LAUNCH = 64      # DSRG_PREP_IMAGES_PER_LAUNCH


class DsrgError(RuntimeError):
    def __init__(self, code, msg):
        RuntimeError.__init__(self, "dsrg_b200 error %d: %s" % (code, msg))
        self.code = code


class CrfParams(C.Structure):
    """dsrg_crf_params (include/dsrg_b200.h)."""
    _fields_ = [("w1", C.c_float), ("theta_alpha_x", C.c_float), ("theta_alpha_y", C.c_float),
                ("theta_beta_r", C.c_float), ("theta_beta_g", C.c_float), ("theta_beta_b", C.c_float),
                ("w2", C.c_float), ("theta_gamma_x", C.c_float), ("theta_gamma_y", C.c_float),
                ("n_iters", C.c_int)]


# name -> (restype, argtypes); this table is also what tests/test_abi.py checks against the header
_vp, _i, _f, _d, _sz, _ll = C.c_void_p, C.c_int, C.c_float, C.c_double, C.c_size_t, C.c_longlong
_pp = C.POINTER(CrfParams)
SIGNATURES = {
    "dsrg_version": (_i, []),
    "dsrg_last_error": (C.c_char_p, []),
    "dsrg_device_count": (_i, []),
    "dsrg_current_device": (_i, []),
    "dsrg_host_alloc": (_vp, [_sz]),
    "dsrg_host_register": (_i, [_vp, _sz]),
    "dsrg_host_unregister": (_i, [_vp]),
    "dsrg_host_free": (None, [_vp]),
    "dsrg_crf_params_default": (None, [_pp, _f, _f, _i]),
    "dsrg_engine_create": (_vp, [_i, _i, _i, _i, _i]),
    "dsrg_engine_destroy": (None, [_vp]),
    "dsrg_engine_device_bytes": (_sz, [_vp]),
    "dsrg_engine_set_size": (_i, [_vp, _i, _i]),
    "dsrg_engine_set_size_ordered": (_i, [_vp, _i, _i]),
    "dsrg_engine_get_size": (_i, [_vp, _vp, _vp, _vp, _vp]),
    "dsrg_engine_set_host_chunk": (_i, [_vp, _i]),
    "dsrg_engine_set_graphs": (_i, [_vp, _i]),
    "dsrg_engine_graph_replays": (_ll, [_vp]),
    "dsrg_engine_take_launch_count": (_ll, [_vp]),
    "dsrg_engine_hybrid_tiles": (_ll, [_vp]),
    "dsrg_crf_batch_dev": (_i, [_vp, _i, _vp, _i, _vp, _pp, _vp, _i, _vp]),
    "dsrg_crf_batch_host": (_i, [_vp, _i, _vp, _i, _vp, _pp, _vp, _i]),
    "dsrg_crf_map_batch_dev": (_i, [_vp, _i, _vp, _i, _vp, _pp, _vp, _vp]),
    "dsrg_srg_batch_dev": (_i, [_vp, _i, _vp, _vp, _vp, _d, _d, _i, _vp, _vp, _vp]),
    "dsrg_srg_batch_host": (_i, [_vp, _i, _vp, _vp, _vp, _d, _d, _i, _vp, _vp]),
    "dsrg_dsrg_forward_dev": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _pp, _d, _d, _vp, _vp, _vp]),
    "dsrg_dsrg_forward_host": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _pp, _d, _d, _vp, _vp]),
    "dsrg_crflayer_forward_dev": (_i, [_vp, _i, _vp, _vp, _pp, _vp, _vp, _vp]),
    "dsrg_softmax_forward_dev": (_i, [_vp, _i, _vp, _vp, _vp]),
    "dsrg_softmax_backward_dev": (_i, [_vp, _i, _vp, _vp, _vp, _vp]),
    "dsrg_constrainloss_forward_dev": (_i, [_vp, _i, _vp, _vp, _vp, _vp]),
    "dsrg_constrainloss_backward_dev": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "dsrg_softmax_forward_host": (_i, [_vp, _i, _vp, _vp]),
    "dsrg_softmax_backward_host": (_i, [_vp, _i, _vp, _vp, _vp]),
    "dsrg_constrainloss_forward_host": (_i, [_vp, _i, _vp, _vp, _vp]),
    "dsrg_constrainloss_backward_host": (_i, [_vp, _i, _vp, _vp, _vp, _vp]),
    "dsrg_prepare_image_dev": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "dsrg_prepare_image_host": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp]),
    "dsrg_prepare_net_input_dev": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "dsrg_prepare_net_input_host": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "dsrg_prepare_net_input_batch_dev": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "dsrg_prepare_net_input_batch_host": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "dsrg_zoom_scores_dev": (_i, [_vp, _vp, _i, _i, _vp, _i, _vp]),
    "dsrg_zoom_scores_host": (_i, [_vp, _vp, _i, _i, _vp, _i]),
    "dsrg_predict_mask_dev": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _f, _i, _pp, _vp, _i, _vp, _vp, _vp]),
    "dsrg_predict_mask_host": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _f, _i, _pp, _vp, _i, _vp, _vp]),
    "dsrg_predict_mask_batch_dev": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _f, _i, _pp, _vp, _vp, _vp, _vp]),
    "dsrg_predict_mask_batch_host": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _f, _i, _pp, _vp, _vp, _vp]),
    "dsrg_annotation_forward_dev": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "dsrg_annotation_forward_host": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "dsrg_annotation_coco_forward_dev": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _vp,
                                              _vp]),
    "dsrg_annotation_coco_forward_host": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp]),
    "dsrg_seg_data_forward_dev": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _i, _vp, _f, _i, _i,
                                       _vp, _vp, _vp]),
    "dsrg_seg_data_forward_host": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _i, _vp, _f, _i, _i,
                                        _vp, _vp]),
    "dsrg_confusion_create": (_vp, [_i, _i]),
    "dsrg_confusion_destroy": (None, [_vp]),
    "dsrg_confusion_reset": (_i, [_vp, _vp]),
    "dsrg_confusion_add_dev": (_i, [_vp, _sz, _vp, _vp, _i, _vp]),
    "dsrg_confusion_add_host": (_i, [_vp, _sz, _vp, _vp, _i]),
    "dsrg_confusion_read": (_i, [_vp, _vp, _vp]),
    "dsrg_wire_pack_mask": (_i, [_vp, _vp, _sz]),
    "dsrg_wire_unpack_mask": (None, [_vp, _vp, _sz]),
    "dsrg_wire_apply_clamp_mask": (None, [_vp, _vp, _sz]),
    "dsrg_crflayer_forward_host": (_i, [_vp, _i, _vp, _vp, _pp, _vp, _vp]),
    "dsrg_crflayer_backward_dev": (_i, [_vp, _vp, _vp, _i, _vp, _vp]),
    "dsrg_srg_last_crf_host": (_i, [_vp, _i, _vp, _vp, _d, _d, _vp]),
    "dsrg_srg_last_crf_dev": (_i, [_vp, _vp, _vp, _i, _d, _d, _vp, _vp]),
    "dsrg_crf_last_marginals_host": (_i, [_vp, _i, _vp, _i]),
    "dsrg_seedloss_forward_host": (_i, [_vp, _i, _vp, _vp, _vp]),
    "dsrg_seedloss_backward_host": (_i, [_vp, _i, _i, _vp, _vp, _f, _vp]),
    "dsrg_seedloss_forward_dev": (_i, [_vp, _i, _vp, _vp, _vp, _vp]),
    "dsrg_seedloss_backward_dev": (_i, [_vp, _i, _i, _vp, _vp, _f, _vp, _vp]),
    "dsrg_seedloss_plain_forward_dev": (_i, [_vp, _i, _vp, _vp, _vp, _vp]),
    "dsrg_seedloss_plain_backward_dev": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp]),
    "dsrg_seedloss_plain_forward_host": (_i, [_vp, _i, _vp, _vp, _vp]),
    "dsrg_seedloss_plain_backward_host": (_i, [_vp, _i, _i, _vp, _vp, _vp]),
    "dsrg_expandloss_forward_dev": (_i, [_vp, _i, _vp, _vp, _d, _d, _vp, _vp]),
    "dsrg_expandloss_backward_dev": (_i, [_vp, _i, _i, _vp, _vp, _d, _d, _vp, _vp]),
    "dsrg_expandloss_forward_host": (_i, [_vp, _i, _vp, _vp, _d, _d, _vp]),
    "dsrg_expandloss_backward_host": (_i, [_vp, _i, _i, _vp, _vp, _d, _d, _vp]),
    "dsrg_profile_tag_count": (_i, []),
    "dsrg_profile_tag_name": (C.c_char_p, [_i]),
    "dsrg_engine_profile": (_i, [_vp, _i]),
    "dsrg_engine_profile_read": (_i, [_vp, _vp, _vp]),
    "dsrg_engine_lattice_sizes": (_i, [_vp, _i, _vp, _vp]),
    "dsrg_engine_lattice_tables": (_i, [_vp, _i, _i, _vp, _vp]),
    "dsrg_engine_copy_norm": (_i, [_vp, _i, _i, _vp]),
    "dsrg_densecrf_create": (_vp, [_i, _i, _i]),
    "dsrg_densecrf_destroy": (None, [_vp]),
    "dsrg_densecrf_npixels": (_i, [_vp]),
    "dsrg_densecrf_nlabels": (_i, [_vp]),
    "dsrg_densecrf_set_unary_energy": (_i, [_vp, _vp]),
    "dsrg_densecrf_add_pairwise_energy": (_i, [_vp] + [_f] * 9 + [_vp]),
    "dsrg_densecrf_map": (_i, [_vp, _i, _vp]),
    "dsrg_densecrf_inference": (_i, [_vp, _i, _vp]),
    "dsrg_densecrf_release_engines": (None, []),
}

_LIB = None


def lib():
    """Load libdsrg_b200.so (built by dsrg_b200/build.py).  Raises if it does not exist."""
    global _LIB
    if _LIB is None:
        try:  # a stale .so silently tests yesterday's kernels: rebuild when a source is newer
            from . import build as _build
            if not os.environ.get("DSRG_B200_LIB") and _build.needs_build():
                _build.build()
        except Exception:  # no nvcc here: fall through to whatever was prebuilt
            pass
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "%s is missing: the CUDA extension was not built (run `python -m dsrg_b200.build` "
                "or __graft_entry__.build()); dsrg_b200 has no CPU fallback" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _LIB = L
    return _LIB


def check(rc):
    if rc != 0:
        raise DsrgError(rc, lib().dsrg_last_error().decode("utf-8", "replace"))
