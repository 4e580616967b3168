"""Which Engine entry points the differentiable dense CRF (nn.dense_crf / dense_crf_wide) calls for each combination
of its arguments, without a GPU: the fused or label-chunked path, Potts weights or matrices, a given theta or none,
the image or caller-given features.  Each entry point is its own graph cache and its own set of first-call buffers,
so a combination must keep the pair it has always used."""
import pytest

from dsrg_b200 import api, nn

# (wide, feat, compat, theta) -> (forward, backward)
TABLE = {
    (False, False, False, False): ("crf_forward_train_dev", "crf_backward_dev"),
    (False, False, False, True): ("crf_forward_train_dev", "crf_backward_theta_dev"),
    (False, False, True, False): ("crf_forward_train_compat_dev", "crf_backward_compat_dev"),
    (False, False, True, True): ("crf_forward_train_compat_dev", "crf_backward_compat_theta_dev"),
    (False, True, False, False): ("crf_forward_train_feat_dev", "crf_backward_feat_dev"),
    (False, True, False, True): ("crf_forward_train_feat_dev", "crf_backward_feat_dev"),
    (False, True, True, False): ("crf_forward_train_feat_dev", "crf_backward_feat_dev"),
    (False, True, True, True): ("crf_forward_train_feat_dev", "crf_backward_feat_dev"),
    (True, False, False, False): ("crf_forward_train_wide_dev", "crf_backward_wide_dev"),
    (True, False, False, True): ("crf_forward_train_wide_dev", "crf_backward_wide_theta_dev"),
    (True, False, True, False): ("crf_forward_train_wide_dev", "crf_backward_wide_dev"),
    (True, False, True, True): ("crf_forward_train_wide_dev", "crf_backward_wide_theta_dev"),
    (True, True, False, False): ("crf_forward_train_wide_feat_dev", "crf_backward_wide_feat_dev"),
    (True, True, False, True): ("crf_forward_train_wide_feat_dev", "crf_backward_wide_feat_dev"),
    (True, True, True, False): ("crf_forward_train_wide_feat_dev", "crf_backward_wide_feat_dev"),
    (True, True, True, True): ("crf_forward_train_wide_feat_dev", "crf_backward_wide_feat_dev"),
}


@pytest.mark.parametrize("wide,feat,compat,theta", sorted(TABLE))
def test_train_entry(wide, feat, compat, theta):
    fwd, bwd = nn._train_entry(wide, feat, compat, theta)
    assert (fwd, bwd) == TABLE[wide, feat, compat, theta]
    assert callable(getattr(api.Engine, fwd)) and callable(getattr(api.Engine, bwd))
