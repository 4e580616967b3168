"""The CRF gradients at the training and benchmark batch sizes and on large lattices, every slot against the float64
backward (tests/crf_grad_scale_cases.py: slot b holds problem pi(b) with upstream s_b * G, so its truth is s_b times
the problem's and its bar |s_b| times the problem's bar).

Cases, with the path each one takes (test_crf_grad_scale_cpu.py checks the claims on the oracle's lattices):
* train41, B = 20 @ 41^2, scale factor 12, 21 labels, 10 iterations: Potts with host and device weights, theta + Potts,
  mu; the ungated blur.
* dsrg321, B = 64 @ 321^2 photos: Potts (10 iterations), theta + mu (3); gate 1 of the transposed pair blur, hybrid,
  direct and shared-memory tiles after k_tile_demote.
* gate2, two 224^2 noise images at 6, 24 and 32 labels: theta + Potts through gate 2 of the transposed pair blur.
* switch, helpers.SWITCH_CASES: Potts on both sides of the device-side row gate and the host-side capacity switch.
* one Engine(64, 321, 321, 21) at batches below and at its own, the theta buffers first allocated at B = 3; the same
  engine re-shaped; nn.dense_crf as a training loop whose last batch is partial.
Each batch runs as training steps do: on a side stream, eager, captured into a CUDA graph, then replayed; the replay
is checked.  Each test prints the device memory in use at its end (torch.cuda.mem_get_info), engine still open."""
import numpy as np
import pytest

import helpers
from crf_grad_scale_cases import (CASES, GATE2_LABELS, GATE2_T, PARTIAL_RUNS, RESHAPE, RESHAPE_U, SWITCH_T,
                                  TRAIN_BATCHES, check_mu, check_potts, check_theta, gate2_problems,
                                  mus_for, photo_problems, problem_truths, switch_case, switch_problems, table,
                                  train41_problems)
from crf_grad_cases import grad_params
from dsrg_b200 import api

pytestmark = pytest.mark.gpu
M = helpers.BENCH_M


def _nchw(torch, a):
    return torch.from_numpy(np.ascontiguousarray(np.transpose(a, (0, 3, 1, 2)))).cuda()


def sm_count(torch):
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@pytest.fixture
def device_memory(torch_cuda, request):
    """Prints the device memory in use (all processes) when the test calls it, and what its start and end left."""
    torch = torch_cuda
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    seen = [(total - free) / 2.0 ** 30]

    def sample():
        torch.cuda.synchronize()
        f, _ = torch.cuda.mem_get_info()
        seen.append((total - f) / 2.0 ** 30)
    yield sample
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    f, _ = torch.cuda.mem_get_info()
    print("\n[device memory] %s: %.2f GiB in use at most, %.2f before, %.2f after"
          % (request.node.name, max(seen), seen[0], (total - f) / 2.0 ** 30))


def run(torch, eng, kind, images, unary, G, p, potts=None, mus=None):
    """One batch's forward and backward of `kind` ("potts": crf_backward_dev, "mu": crf_backward_compat_dev,
    "theta": crf_backward_theta_dev, "theta_mu": crf_backward_compat_theta_dev) on a side stream, eager, captured
    and replayed, every output filled with NaN before each run.  -> the replay's (dL/dU (B, H, W, M), the Potts pair
    (B, 2) or dL/dmu (B, 2, M, M), dL/dtheta (B, 7) or None)."""
    B, Mb = unary.shape[0], unary.shape[-1]
    u, g, im = _nchw(torch, unary), _nchw(torch, G), torch.from_numpy(images).cuda()
    q_hist = torch.empty((p.n_iters + 1,) + tuple(u.shape), device="cuda")
    gu = torch.empty_like(u)
    compat = None if mus is None else torch.from_numpy(np.stack(mus).astype(np.float32)).cuda()
    gw = torch.empty((B, 2) if mus is None else (B, 2, Mb, Mb), device="cuda")
    gt = torch.empty((B, 7), device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    r0 = eng.graph_replays
    with torch.cuda.stream(side):
        s = side.cuda_stream
        for _ in range(3):
            for t in (q_hist, gu, gw, gt):
                t.fill_(float("nan"))
            if mus is None:
                eng.crf_forward_train_dev(u, im, p, q_hist, potts=potts, stream=s)
            else:
                eng.crf_forward_train_compat_dev(u, im, p, compat, q_hist, stream=s)
            if kind == "potts":
                eng.crf_backward_dev(q_hist, im, p, g, gu, grad_potts=gw, potts=potts, stream=s)
            elif kind == "mu":
                eng.crf_backward_compat_dev(q_hist, im, p, compat, g, gu, grad_compat=gw, stream=s)
            elif kind == "theta":
                eng.crf_backward_theta_dev(q_hist, im, p, g, gu, gt, grad_potts=gw, potts=potts, stream=s)
            else:
                eng.crf_backward_compat_theta_dev(q_hist, im, p, compat, g, gu, gt, grad_compat=gw, stream=s)
    side.synchronize()
    assert eng.graph_replays > r0, "the third run was not a replay"
    out = (np.transpose(gu.cpu().numpy(), (0, 2, 3, 1)), gw.cpu().numpy(),
           gt.cpu().numpy() if kind.startswith("theta") else None)
    del q_hist, gu, gw, gt, u, g
    return out


def batch(problems, pi, s):
    """The batch of slots pi with upstream gradients s * G."""
    images, unary, G = problems
    return (np.ascontiguousarray(images[pi]), np.ascontiguousarray(unary[pi]),
            (G[pi] * s[:, None, None, None].astype(np.float32)).astype(np.float32))


def check_slots(what, truths, kind, pi, s, out):
    """Every slot of a run's output against its problem's truths, scaled.  truths: {kind: [per problem]}."""
    gU, gw, gt = out
    for b, (u, sb) in enumerate(zip(pi, s)):
        w = "%s slot %d (problem %d, s = %g):" % (what, b, u, sb)
        if kind in ("potts", "theta"):
            check_potts(truths["potts"][u], sb, gU[b], gw[b], w)
        else:
            check_mu(truths["mu"][u], sb, gU[b], gw[b], w)
        if kind.startswith("theta"):
            check_theta(truths[kind][u], sb, gt[b], w)


def branch_of(eng, H, W, B):
    _, vb = eng.lattice_sizes(B)
    return helpers.blur_branch(H, W, vb)


# ---- train41 ----
@pytest.mark.parametrize("kind", ["potts_host", "potts_dev", "theta", "mu"])
def test_train41_every_slot(torch_cuda, device_memory, kind):
    torch = torch_cuda
    H, W, B, sf, U, Tp, Tt, branch = CASES["train41"]
    probs = train41_problems(U)
    grad = "potts" if kind.startswith("potts") else kind
    T = Tp if grad == "potts" else Tt
    truths = problem_truths("train41", ["potts", "theta"] if grad != "mu" else ["mu"], *probs, sf, T)
    pi, s = table("train41-" + kind, B, U)
    p = grad_params(sf, T)
    potts = torch.tensor([p.w1, p.w2], device="cuda") if kind == "potts_dev" else None
    if kind == "potts_dev":
        p.w1, p.w2 = 1.0, 1.0   # the device weights must win over these
    eng = api.Engine(B, H, W, M)
    out = run(torch, eng, grad, *batch(probs, pi, s), p, potts=potts, mus=mus_for() if grad == "mu" else None)
    device_memory()
    assert branch_of(eng, H, W, B) == branch
    check_slots("train41 " + kind, truths, grad, pi, s, out)
    eng.close()


# ---- dsrg321 ----
@pytest.mark.parametrize("kind", ["potts", "theta_mu"])
def test_dsrg321_every_slot(torch_cuda, device_memory, kind):
    torch = torch_cuda
    H, W, B, sf, U, Tp, Tt, branch = CASES["dsrg321"]
    probs = photo_problems(H, W, U)
    T = Tp if kind == "potts" else Tt
    truths = problem_truths("dsrg321", ["potts"] if kind == "potts" else ["mu", "theta_mu"], *probs, sf, T)
    pi, s = table("dsrg321-" + kind, B, U)
    eng = api.Engine(B, H, W, M)
    out = run(torch, eng, kind, *batch(probs, pi, s), grad_params(sf, T), mus=mus_for() if kind != "potts" else None)
    device_memory()
    pred = helpers.predict_tile_paths(probs[0][pi], sf, sm_count(torch))
    assert eng.hybrid_tiles == pred["hybrid_tiles"] > 0
    assert (pred["bi"] == "direct").any() and (pred["bi"] == "smem").any()
    assert branch_of(eng, H, W, B) == branch
    check_slots("dsrg321 " + kind, truths, kind, pi, s, out)
    eng.close()


# ---- gate 2 and the switches ----
@pytest.mark.parametrize("Mg", GATE2_LABELS)
def test_gate2_reverse_blur(torch_cuda, device_memory, Mg):
    torch = torch_cuda
    probs = gate2_problems(Mg)
    B, H, W = probs[0].shape[:3]
    truths = problem_truths("gate2-%d" % Mg, ["potts", "theta"], *probs, 1.0, GATE2_T)
    pi, s = table("gate2-%d" % Mg, B, B)
    eng = api.Engine(B, H, W, Mg)
    out = run(torch, eng, "theta", *batch(probs, pi, s), grad_params(1.0, GATE2_T))
    device_memory()
    assert branch_of(eng, H, W, B) == "gate2"
    check_slots("gate2 M=%d" % Mg, truths, "theta", pi, s, out)
    eng.close()


@pytest.mark.parametrize("name", [c[0] for c in helpers.SWITCH_CASES])
def test_switch_both_sides_reversed(torch_cuda, device_memory, name):
    torch = torch_cuda
    H, W, kinds, branch = switch_case(name)
    probs = switch_problems(name)
    B = len(kinds)
    truths = problem_truths("switch-" + name, ["potts"], *probs, 1.0, SWITCH_T)
    pi, s = table("switch-" + name, B, B)
    eng = api.Engine(B, H, W, M)
    out = run(torch, eng, "potts", *batch(probs, pi, s), grad_params(1.0, SWITCH_T))
    device_memory()
    assert branch_of(eng, H, W, B) == branch
    check_slots("switch " + name, truths, "potts", pi, s, out)
    eng.close()


# ---- batches below the engine's ----
def test_partial_batches_on_one_engine(torch_cuda, device_memory):
    """theta + Potts at B = 3 first (so the theta buffers are allocated at a small batch, hybrid tiles off), then 64,
    37, 1 and 64 again; then theta + mu at 5 and 64: every slot each time, the hybrid-tile count as predicted."""
    torch = torch_cuda
    H, W, Bmax, sf, U, _, T, _ = CASES["dsrg321"]
    probs = photo_problems(H, W, U)
    truths = problem_truths("dsrg321", ["potts", "theta", "mu", "theta_mu"], *probs, sf, T)
    eng = api.Engine(Bmax, H, W, M)
    p = grad_params(sf, T)
    for i, (kind, B) in enumerate(PARTIAL_RUNS):
        pi, s = table("partial-%d" % i, B, U)
        out = run(torch, eng, kind, *batch(probs, pi, s), p, mus=mus_for() if kind == "theta_mu" else None)
        device_memory()
        pred = helpers.predict_tile_paths(probs[0][pi], sf, sm_count(torch))
        assert eng.hybrid_tiles == pred["hybrid_tiles"], (kind, B)
        check_slots("%s B=%d of %d" % (kind, B, Bmax), truths, kind, pi, s, out)
    eng.close()


def test_reshaped_engine(torch_cuda, device_memory):
    """Engine(4, 321, 321, 21) set to 200 x 224 (fewer pixels and tiles than its capacity), then back to 321^2."""
    torch = torch_cuda
    _, _, _, sf, U, _, T, _ = CASES["dsrg321"]
    B = 4
    eng = api.Engine(B, 321, 321, M)
    p = grad_params(sf, T)
    for shape, tag, Us in ((RESHAPE, "reshape", RESHAPE_U), ((321, 321), "dsrg321", U)):
        eng.set_size(*shape)
        probs = photo_problems(shape[0], shape[1], Us)
        truths = problem_truths(tag, ["potts", "theta"], *probs, sf, T)
        pi, s = table("reshape-%s" % tag, B, Us)
        out = run(torch, eng, "theta", *batch(probs, pi, s), p)
        device_memory()
        check_slots("theta %dx%d on a 321x321 engine" % shape, truths, "theta", pi, s, out)
    eng.close()


# ---- nn.dense_crf as a training loop ----
def test_dense_crf_training_loop_with_a_partial_batch(torch_cuda, device_memory):
    """Batches of 20, 20 and 7 through nn.dense_crf with w1, w2 and float64 theta as leaves: per-slot u.grad, the
    batch sums of the w and theta gradients, and the last batch on the cached engine."""
    torch = torch_cuda
    from dsrg_b200 import nn
    H, W, _, sf, U, T, _, _ = CASES["train41"]
    probs = train41_problems(U)
    truths = problem_truths("train41", ["potts", "theta"], *probs, sf, T)
    p = grad_params(sf, T)
    w1 = torch.tensor(float(p.w1), device="cuda", requires_grad=True)
    w2 = torch.tensor(float(p.w2), device="cuda", requires_grad=True)
    th_bi = torch.tensor([p.theta_alpha_x, p.theta_alpha_y, p.theta_beta_r, p.theta_beta_g, p.theta_beta_b],
                         dtype=torch.float64, device="cuda", requires_grad=True)
    th_sp = torch.tensor([p.theta_gamma_x, p.theta_gamma_y], dtype=torch.float64, device="cuda", requires_grad=True)
    engines = []
    for i, B in enumerate(TRAIN_BATCHES):
        pi, s = table("train-loop-%d" % i, B, U)
        images, unary, G = batch(probs, pi, s)
        u = _nchw(torch, unary).requires_grad_(True)
        for t in (w1, w2, th_bi, th_sp):
            t.grad = None
        q = nn.dense_crf(u, torch.from_numpy(images).cuda(), sf, 13, T, w1=w1, w2=w2, theta_bi=th_bi, theta_sp=th_sp)
        (q * _nchw(torch, G)).sum().backward()
        torch.cuda.synchronize()
        device_memory()
        engines.append(nn.cached_engine(M, H, W, torch.cuda.current_device()))
        gU = np.transpose(u.grad.cpu().numpy(), (0, 2, 3, 1))
        for b, (k, sb) in enumerate(zip(pi, s)):
            check_potts(truths["potts"][k], sb, gU[b], None, "batch %d slot %d:" % (i, b))
        pt, tt = [truths["potts"][k] for k in pi], [truths["theta"][k] for k in pi]
        got_w = np.array([float(w1.grad), float(w2.grad)])
        want_w = np.array([sum(sb * t.gw[j] for sb, t in zip(s, pt)) for j in (0, 1)])
        bar_w = np.array([sum(abs(sb) * t.bar_w[j] for sb, t in zip(s, pt)) for j in (0, 1)])
        assert np.all(np.abs(got_w - want_w) <= bar_w), (i, got_w, want_w, bar_w)
        assert th_bi.grad.dtype == torch.float64 and th_bi.grad.device == th_bi.device
        got_t = np.concatenate([th_bi.grad.cpu().numpy(), th_sp.grad.cpu().numpy()])
        want_t = sum(sb * t.want for sb, t in zip(s, tt))
        bar_t = sum(abs(sb) * t.bar for sb, t in zip(s, tt))
        assert np.all(np.abs(got_t - want_t) <= bar_t), (i, got_t, want_t, bar_t)
    assert engines[0] is not None and engines[0].max_batch >= max(TRAIN_BATCHES)
    assert all(e is engines[0] for e in engines), "a batch below the engine's replaced the cached engine"
