"""GPU parity at the sizes the benchmark and the tools run, against the CPU oracles.

bench.py's workloads at their own batch (64 at 321², 16 at 513², 20 at 41²), run as bench.py runs them: on a side
stream, eager, captured into a CUDA graph, then replayed; the replayed pass is checked.  The oracle sees a sample of
each batch; the whole batch is checked for the in-place clamp, normalised finite marginals, seeds that keep every
cue, and against each image run alone on a batch-1 engine.

The bilateral pair blur picks its kernel by lattice size (meanfield.cu: blur_all, k_mf_blur): helpers.blur_branch
names the three branches.  Gate 2 (large scattered lattices) runs at every padded label count here, and both sides
of the device-side row gate and of the host-side capacity switch are compared with the oracle.  The label-chunked
path runs at a COCO image's size with 81 labels and with 255 labels on a lattice above the capacity switch.
tests/test_scale_cpu.py checks on the CPU that every case takes the branch claimed for it.

Tolerances are the suite's: CRF marginals 1e-4 max-abs, seeds bit-exact against the SRG oracle on the float64
renormalisation of the engine's own marginals, the in-place clamp exact, the seed loss rtol 1e-5.  A one-ulp change
of the unary moves the oracle's marginals by less than 1e-5 in every case here (measured on a sample of each bench
batch and on every other case), so none sits where the oracle is chaotic and the unaries need no sharpening.
"""
import numpy as np
import pytest

from helpers import (BENCH_CF, BENCH_M, BENCH_T_ITERS, BENCH_TH, BENCH_WORKLOADS, COCO_M, COCO_SHAPE,
                     GATE2_M, GATE2_SEED, GATE2_SHAPE, SCALE_CASES, SWITCH_CASES, WIDE_BIG_M, WIDE_BIG_SHAPE,
                     bench_sf, bench_unique, blur_branch, crf_both_layouts, log_unary, oracle_batch, renorm64,
                     sample_indices, seeded_images)
from dsrg_b200 import api
from oracle import crf_oracle, loss_oracle, srg_oracle

pytestmark = pytest.mark.gpu
TOL = 1e-4
MIN_PROB = np.float32(1e-4)


def assert_close(got, want, what):
    err = float(np.abs(got - want).max())
    assert err <= TOL, (what, err)


def bench_inputs(torch, workload, variant):
    """bench.py's device inputs: the distinct problems, repeated cyclically to the batch on the device."""
    H, W, B, what = BENCH_WORKLOADS[workload]
    uniq = bench_unique(workload, variant)
    pick = torch.arange(B, device="cuda") % len(uniq["probs"])
    d = {k: torch.from_numpy(uniq[k]).cuda()[pick].contiguous() for k in ("labels", "probs", "cues", "image")}
    return uniq, d


def run_pass(eng, what, d, params, stream=None):
    if what == "crf":
        eng.crf_dev(d["unary"], d["image"], params, d["q"], stream=stream)
        return
    eng.dsrg_forward_dev(d["labels"], d["probs"], d["cues"], d["image"], params, *BENCH_TH, d["seeds"],
                         crf_out=d["q"], stream=stream)
    if "loss" in what:
        eng.seedloss_forward_dev(d["probs"], d["seeds"], d["terms"], stream=stream)


@pytest.mark.parametrize("workload,variant,branch", SCALE_CASES)
def test_bench_workload_at_its_batch(torch_cuda, workload, variant, branch):
    torch = torch_cuda
    H, W, B, what = BENCH_WORKLOADS[workload]
    sf = bench_sf(workload)
    params = api.crf_params(sf, BENCH_CF, BENCH_T_ITERS)
    uniq, d = bench_inputs(torch, workload, variant)
    U = len(uniq["probs"])
    probs0 = d["probs"].clone()
    if what == "crf":
        d["unary"] = d["probs"].permute(0, 2, 3, 1).contiguous()
        d["q"] = torch.empty_like(d["unary"])
    else:
        d["q"] = torch.empty_like(d["probs"])
        d["seeds"] = torch.empty_like(d["probs"])
        d["terms"] = torch.zeros(2, device="cuda")
    eng = api.Engine(B, H, W, BENCH_M)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        for _ in range(3):                        # eager, captured, replayed
            for k in ("q", "seeds", "terms"):     # so that the replay has to write every output again
                if k in d:
                    d[k].fill_(float("nan"))
            run_pass(eng, what, d, params)
    side.synchronize()
    assert eng.graph_replays >= 1
    _, vb = eng.lattice_sizes(B)
    assert blur_branch(H, W, vb) == branch, (list(vb[:U]), branch)
    if variant == "photo":
        assert eng.hybrid_tiles > 0               # the textured batch makes a hybrid pass

    # the whole batch
    q = d["q"] if what == "crf" else d["q"].permute(0, 2, 3, 1)    # NHWC view
    assert bool(torch.isfinite(q).all())
    assert float((q.sum(-1) - 1).abs().max()) <= 1e-5
    if what == "crf":
        assert torch.equal(d["probs"], probs0)
    else:
        assert torch.equal(d["probs"], torch.where(probs0 < MIN_PROB, torch.full_like(probs0, MIN_PROB), probs0))
        assert bool((d["seeds"] >= d["cues"]).all())
    # every image against the same image alone on a batch-1 engine (the batch repeats its U distinct problems)
    one = api.Engine(1, H, W, BENCH_M)
    q1 = []
    for u in range(U):
        d1 = {k: v[u:u + 1].clone() for k, v in d.items() if k != "terms"}
        d1["probs"] = probs0[u:u + 1].clone()
        if what == "crf":
            d1["unary"] = d1["probs"].permute(0, 2, 3, 1).contiguous()
        else:
            d1["terms"] = torch.zeros(2, device="cuda")
        run_pass(one, what, d1, params)
        q1.append(d1["q"])
    q1 = torch.cat(q1)[torch.arange(B, device="cuda") % U]
    err = float((d["q"] - q1).abs().max())
    assert err <= TOL, ("batch vs batch-1", err)
    one.close()

    # a sample against the oracles
    qh = d["q"].cpu().numpy()
    probs_c = d["probs"].cpu().numpy() if what != "crf" else None
    seeds = d["seeds"].cpu().numpy() if what != "crf" else None
    want = {}
    for i in sample_indices(B, seed=B + H):
        u = i % U
        if u not in want:
            p = uniq["probs"][u]
            if what != "crf":
                p = np.where(p < MIN_PROB, MIN_PROB, p)
            want[u] = crf_oracle.CRF(uniq["image"][u], np.ascontiguousarray(np.transpose(p, (1, 2, 0))),
                                     BENCH_T_ITERS, sf, BENCH_CF)
        if what == "crf":
            assert_close(qh[i], want[u], (workload, variant, i))
            continue
        assert_close(np.transpose(qh[i], (1, 2, 0)), want[u], (workload, variant, i))
        r = renorm64(qh[i])
        assert np.array_equal(seeds[i], srg_oracle.srg_closed_form(uniq["labels"][u], uniq["cues"][u], r, *BENCH_TH)), \
            (workload, variant, i)
    if "loss" in what:
        loss = -float(d["terms"].sum()) / B
        want_loss = sum(loss_oracle.balanced_seed_loss(probs_c[b:b + 1], seeds[b:b + 1]) for b in range(B)) / B
        assert abs(loss - want_loss) <= 1e-5 * abs(want_loss), (loss, want_loss)
    eng.close()


@pytest.fixture(scope="module")
def gate2_images():
    return seeded_images(*GATE2_SHAPE, ("noise", "noise"), GATE2_SEED)


@pytest.mark.parametrize("M", GATE2_M)
def test_gate2_blur_every_padded_label_count(torch_cuda, gate2_images, M):
    """k_mf_blur<MP, 2, 4> (gate 2) at one M per MP, tail1 counts included, n_iters 2 and 10, both layouts."""
    image = gate2_images
    B, H, W = image.shape[:3]
    unary = log_unary(B, H, W, M, seed=8000 + M)
    eng = api.Engine(B, H, W, M)
    for n_iters in (2, 10):
        want = oracle_batch(image, unary, 1.0, n_iters)
        nhwc, nchw = crf_both_layouts(torch_cuda, eng, unary, image, api.crf_params(1.0, maxiter=n_iters))
        assert_close(nhwc, want, (M, n_iters, "NHWC"))
        assert_close(nchw, want, (M, n_iters, "NCHW"))
        _, vb = eng.lattice_sizes(B)
        assert blur_branch(H, W, vb) == "gate2", list(vb)
    eng.close()


@pytest.mark.parametrize("name,H,W,kinds,branch", SWITCH_CASES, ids=[c[0] for c in SWITCH_CASES])
def test_blur_switches_both_sides(torch_cuda, name, H, W, kinds, branch):
    """A ~96 k-row noise lattice blurred at full occupancy because its smooth partner keeps the batch's average
    down (gate 1), a noise pair on gate 2, and sizes either side of the host-side capacity switch."""
    image = seeded_images(H, W, kinds, GATE2_SEED)
    B = image.shape[0]
    unary = log_unary(B, H, W, BENCH_M, seed=8100 + H + W)
    want = oracle_batch(image, unary, 1.0)
    eng = api.Engine(B, H, W, BENCH_M)
    nhwc, nchw = crf_both_layouts(torch_cuda, eng, unary, image, api.crf_params(1.0))
    assert_close(nhwc, want, (name, "NHWC"))
    assert_close(nchw, want, (name, "NCHW"))
    _, vb = eng.lattice_sizes(B)
    assert blur_branch(H, W, vb) == branch, list(vb)
    eng.close()


def test_wide_path_coco_size(torch_cuda):
    """DenseCRF(W, H, 81) on a COCO-sized photo-like image as the COCO tool uses it (unary log p, inference and
    map()), and the same problem through crf_dev in NCHW."""
    torch = torch_cuda
    H, W = COCO_SHAPE
    image = seeded_images(H, W, ("photo",), 5)
    unary = log_unary(1, H, W, COCO_M, seed=COCO_M)
    want = oracle_batch(image, unary, 1.0)[0]
    c = api.DenseCRF(W, H, COCO_M)
    c.set_unary_energy(-unary[0].ravel())
    c.add_pairwise_energy(10, 80, 80, 13, 13, 13, 3, 3, 3, image[0].ravel())
    assert_close(c.inference(10).reshape(H, W, COCO_M), want, "DenseCRF.inference")
    top2 = np.sort(want, -1)[..., -2:]
    clear = (top2[..., 1] - top2[..., 0]) > 4 * TOL
    assert np.array_equal(c.map(10).reshape(H, W)[clear], want.argmax(-1)[clear])
    eng = api.Engine(1, H, W, COCO_M)
    d_nchw = torch.from_numpy(np.ascontiguousarray(np.transpose(unary, (0, 3, 1, 2)))).cuda()
    d_out = torch.empty_like(d_nchw)
    eng.crf_dev(d_nchw, torch.from_numpy(image).cuda(), api.crf_params(1.0), d_out, api.LAYOUT_NCHW, api.LAYOUT_NCHW)
    assert_close(np.transpose(d_out.cpu().numpy()[0], (1, 2, 0)), want, "crf_dev NCHW")
    eng.close()


def test_wide_path_most_labels_above_the_capacity_switch(torch_cuda):
    H, W = WIDE_BIG_SHAPE
    image = seeded_images(H, W, ("noise",), 7)
    unary = log_unary(1, H, W, WIDE_BIG_M, seed=WIDE_BIG_M)
    want = oracle_batch(image, unary, 1.0)
    eng = api.Engine(1, H, W, WIDE_BIG_M)
    nhwc, nchw = crf_both_layouts(torch_cuda, eng, unary, image, api.crf_params(1.0))
    assert_close(nhwc, want, "NHWC")
    assert_close(nchw, want, "NCHW")
    eng.close()
