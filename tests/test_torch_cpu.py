"""CPU tests of dsrg_b200.nn, the PyTorch interface: it imports without a GPU, and bad inputs raise ValueError
before any engine is created or any kernel launched."""
import pytest
import torch

from dsrg_b200 import nn


@pytest.fixture
def no_engine(monkeypatch):
    """Fail the test if nn asks for an engine."""
    def refuse(*args, **kwargs):
        raise AssertionError("an engine was requested")
    monkeypatch.setattr(nn.api, "Engine", refuse)
    monkeypatch.setattr(nn, "_ENGINES", {})
    yield
    assert nn._ENGINES == {}


def maps(N=2, M=21, H=41, W=41, dtype=torch.float32):
    return torch.rand(N, M, H, W, dtype=dtype)


def test_module_surface():
    for name in ("softmax", "crf_layer", "dsrg_seeds", "balanced_seed_loss", "constrain_loss", "seed_loss",
                 "expand_loss", "DSRGHead", "cached_engine"):
        assert hasattr(nn, name), name
    head = nn.DSRGHead()
    assert (head.th1, head.th2, head.scale_factor) == (0.99, 0.85, 12.0)
    assert isinstance(head, torch.nn.Module) and list(head.parameters()) == []
    assert nn.cached_engine(21, 41, 41, 0) is None or nn.cached_engine(21, 41, 41, 0).M == 21


def test_cpu_tensors_are_refused(no_engine):
    p, im = maps(), torch.rand(2, 3, 321, 321)
    lab = torch.ones(2, 1, 1, 21)
    calls = [lambda: nn.softmax(p), lambda: nn.crf_layer(p, im), lambda: nn.dsrg_seeds(lab, p, p, im),
             lambda: nn.balanced_seed_loss(p, p), lambda: nn.constrain_loss(p, p), lambda: nn.seed_loss(p, p),
             lambda: nn.expand_loss(p, lab), lambda: nn.DSRGHead()(p, im, lab, p)]
    for call in calls:
        with pytest.raises(ValueError, match="CUDA"):
            call()


@pytest.mark.parametrize("dtype", [torch.float64, torch.float16, torch.bfloat16, torch.int32])
def test_wrong_dtypes_are_refused(no_engine, dtype):
    p = maps().to(dtype)
    with pytest.raises(ValueError, match="float32"):
        nn.softmax(p)
    with pytest.raises(ValueError, match="float32"):
        nn.balanced_seed_loss(p, p)
    with pytest.raises(ValueError, match="float32"):
        nn.DSRGHead()(p, torch.rand(2, 3, 65, 65), torch.ones(2, 21), maps())


@pytest.mark.parametrize("shape", [(21, 41, 41), (2, 21, 41, 41, 1), (2, 0, 41, 41), (0, 21, 41, 41)])
def test_wrong_shapes_are_refused(no_engine, shape):
    with pytest.raises(ValueError):
        nn.softmax(torch.rand(shape))
    with pytest.raises(ValueError):
        nn.constrain_loss(torch.rand(shape), torch.rand(shape))


@pytest.mark.parametrize("M", [256, 300])
def test_more_than_255_labels_are_refused(no_engine, M):
    p, im = maps(M=M, H=5, W=5), torch.rand(2, 3, 9, 9)
    for call in (lambda: nn.crf_layer(p, im), lambda: nn.dsrg_seeds(torch.ones(2, M), p, p, im),
                 lambda: nn.balanced_seed_loss(p, p), lambda: nn.expand_loss(p, torch.ones(2, M))):
        with pytest.raises(ValueError, match="255"):
            call()


def test_mismatched_companions_are_refused(no_engine):
    """labels, cues and images must fit probs; checked before the device, so on the CPU too."""
    p = maps()
    head = nn.DSRGHead()
    bad = [(torch.rand(2, 3, 65, 65), torch.ones(2, 20), maps()),         # labels of the wrong width
           (torch.rand(2, 3, 65, 65), torch.ones(2, 1, 21), maps()),      # labels of the wrong rank
           (torch.rand(2, 4, 65, 65), torch.ones(2, 21), maps()),         # images with four channels
           (torch.rand(3, 3, 65, 65), torch.ones(2, 21), maps()),         # images of another batch
           (torch.rand(2, 3, 65, 65), torch.ones(2, 21), maps(H=40))]     # cues of another size
    for im, lab, cues in bad:
        with pytest.raises(ValueError):
            head(p, im, lab, cues)
        with pytest.raises(ValueError):
            nn.dsrg_seeds(lab, p, cues, im)
    with pytest.raises(ValueError):
        nn.balanced_seed_loss(p, maps(N=3))
    with pytest.raises(ValueError):
        nn.softmax(p.numpy())


def test_no_engine_is_replaced_during_capture(monkeypatch):
    """A larger batch during CUDA-graph capture raises instead of freeing the engine a captured step uses."""
    class Held:
        max_batch, closed = 2, False

        def close(self):
            self.closed = True
    held = Held()
    monkeypatch.setattr(nn, "_ENGINES", {(21, 41, 41, 0): held})
    monkeypatch.setattr(nn.torch.cuda, "is_current_stream_capturing", lambda: True)
    with pytest.raises(RuntimeError, match="during CUDA-graph capture"):
        nn._engine(3, 21, 41, 41, 0)
    assert not held.closed and nn.cached_engine(21, 41, 41, 0) is held
    assert nn._engine(2, 21, 41, 41, 0) is held   # a batch it holds is served as before
