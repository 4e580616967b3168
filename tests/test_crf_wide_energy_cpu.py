"""The CRF energy above 32 labels without a GPU: the float64 restatement (oracle/crf_energy_oracle.py) against the
reference's own klDivergence at 33, 40 and 81 labels (tests/golden/crf_wide_energy_ref.npz), the label-chunked entry
points' declarations, and the refusals of nn.dense_crf_energy_wide that need no device."""
import os
import re

import numpy as np
import pytest

from crf_energy_cases import library_mus, problem
from crf_wide_energy_cases import GOLDEN, GOLDEN_CASES, golden_inputs
from dsrg_b200 import _lib
from oracle import crf_energy_oracle as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# The reference sums each pairwise term in float32, sequentially over the N * M products, after a float32 filter;
# test_crf_energy_cpu.py bounds that at 2^-18 of the magnitude sum for up to 21 labels.  At 81 labels a sum has about
# four times the products, so its random-walk rounding about twice the error (sqrt(81 / 21)): the largest measured
# here is 7.7e-7 of the magnitude sum (2^-20.3), a quarter of the same bar, which therefore stays.
GOLDEN_REL = 2.0 ** -18


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_restatement_reproduces_the_reference_kl_divergence_above_32_labels(name):
    q, unary, p, m, image, feats = golden_inputs(name)
    assert q.shape[-1] > 32
    want = np.load(os.path.join(ROOT, "tests", "golden", GOLDEN))[name + "/terms"]
    got, scale = E.terms(problem(image, p, feats), q, unary, library_mus(m))
    assert np.all(np.abs(got - want) <= GOLDEN_REL * scale + 1e-12), (got, want, scale)
    if unary is None:
        assert got[1] == 0.0 and want[1] == 0.0


def test_wide_symbols_are_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "dsrg_b200.h")).read()
    L = _lib.lib()
    for name in ("dsrg_crf_energy_wide_dev", "dsrg_crf_energy_backward_wide_dev"):
        assert re.search(r"\bint %s\(" % name, header), name
        assert name in _lib.SIGNATURES
        getattr(L, name)
    # the same arguments as the fused pair
    assert _lib.SIGNATURES["dsrg_crf_energy_wide_dev"] == _lib.SIGNATURES["dsrg_crf_energy_dev"]
    assert _lib.SIGNATURES["dsrg_crf_energy_backward_wide_dev"] == _lib.SIGNATURES["dsrg_crf_energy_backward_dev"]
    assert L.dsrg_version() >= 119


def test_dense_crf_energy_wide_refusals_without_gpu():
    torch = pytest.importorskip("torch")
    from dsrg_b200 import nn
    q = torch.zeros(1, 40, 4, 5)
    img = torch.zeros(1, 4, 5, 3, dtype=torch.uint8)
    f = torch.zeros(1, 5, 4, 5)
    with pytest.raises(ValueError, match="1 <= M <= 255"):
        nn.dense_crf_energy_wide(torch.zeros(1, 256, 4, 5), None, img)
    with pytest.raises(ValueError, match="image is not used"):
        nn.dense_crf_energy_wide(q, None, img, features_bi=f)
    with pytest.raises(ValueError, match="image must be"):
        nn.dense_crf_energy_wide(q, None, None)
    with pytest.raises(ValueError, match="unary must have"):
        nn.dense_crf_energy_wide(q, torch.zeros(1, 39, 4, 5), img)
    for kw in (dict(w1=torch.tensor(3.0, requires_grad=True)),
               dict(compat_bi=torch.zeros(40, 40, requires_grad=True)),
               dict(theta_sp=torch.ones(2, requires_grad=True))):
        with pytest.raises(ValueError, match="requires grad: dense_crf_energy_wide"):
            nn.dense_crf_energy_wide(q, None, img, **kw)
    with pytest.raises(ValueError, match="requires grad"):
        nn.dense_crf_energy_wide(q, None, None, features_bi=f.requires_grad_())
    with pytest.raises(ValueError, match="CUDA tensor"):
        nn.dense_crf_energy_wide(q, None, img)
    with pytest.raises(ValueError, match="CUDA tensor"):   # 32 labels or fewer take the same checks
        nn.dense_crf_energy_wide(torch.zeros(1, 21, 4, 5), None, img)
