"""Every mean-field pass runs through one helper (csrc/common.cuh: crf_pass).  Whatever its kind, a pass that has to
rebuild the shared spatial lattice is captured with that rebuild, so a caller that alternates image sizes replays its
graphs.  The helper alone writes what the engine holds after a pass: the batch whose marginals the *_last_* entry
points may read."""
import numpy as np
import pytest

from dsrg_b200 import _lib, api, synth

pytestmark = pytest.mark.gpu
B, M, CAP = 3, 21, 48
SIZES = [(40, 48), (48, 40)]   # alternated on one engine: every pass then has to rebuild the spatial lattice
KINDS = ["crf", "crf_map", "forward", "crflayer", "post"]
TOL = 1e-4    # the CRF parity bar (DESIGN.md section 3)
TIES = 1e-3   # share of seed values or labels a threshold or arg-max tie may flip (test_gpu_srg.py's replay test)
TH = (0.99, 0.85)

# Eager launches of one call on a new engine with graphs off: (the first call, which builds the spatial lattice, the
# second).  Taken from the library before crf_pass, on an H100 80GB HBM3; the shapes keep every pass off the hybrid
# tiles, whose use depends on the SM count.  dsrg_forward_host runs three chunks at three images.
LAUNCHES = {"crf_dev": (95, 81), "crf_host": (95, 81), "crf_map_dev": (95, 81),
            "dsrg_forward_dev": (98, 84), "dsrg_forward_host": (263, 249),
            "crflayer_forward_dev": (94, 80), "crflayer_forward_host": (94, 80),
            "predict_mask_batch_dev": (98, 84), "predict_mask_batch_host": (98, 84),
            "predict_mask_dev": (98, 84), "predict_mask_host": (98, 84)}


def params(sigma_scale=12.0):
    return api.crf_params(sigma_scale)


def code(fn, *args):
    try:
        fn(*args)
    except api.DsrgError as ex:
        return ex.code
    return _lib.OK


class Pass(object):
    """One kind of pass at one image size, on fixed buffers (a graph key holds the pointers)."""

    def __init__(self, torch, eng, kind, H, W, seed):
        self.eng, self.kind = eng, kind
        d = synth.make_batch(B, H, W, cues="cam", image="smooth", start=seed)
        d["unary"] = np.log(np.maximum(d["probs"], 1e-5)).transpose(0, 2, 3, 1).copy()
        d["scores"] = np.random.RandomState(seed).standard_normal((B, M, 31, 41)).astype(np.float32)
        self.host = d
        self.dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in d.items()}
        self.probs = self.dev["probs"].clone()
        f = lambda *shape: torch.empty(*shape, device="cuda")
        i = lambda *shape: torch.empty(*shape, dtype=torch.int32, device="cuda")
        self.out = {"crf": {"q": f(B, M, H, W)},
                    "crf_map": {"labels": i(B, H, W)},
                    "forward": {"seeds": f(B, M, H, W), "q": f(B, M, H, W)},
                    "crflayer": {"log": f(B, M, H, W), "result": f(B, M, H, W)},
                    "post": {"labels": i(B, H, W), "q": f(B, H, W, M)}}[kind]
        torch.cuda.synchronize()

    def run(self, p=None):
        """Issues the pass on the current stream and returns copies of its outputs."""
        e, d, o = self.eng, self.dev, self.out
        p = p or params()
        self.probs.copy_(d["probs"])   # forward and crflayer clamp their input in place
        if self.kind == "crf":
            e.crf_dev(d["unary"], d["image"], p, o["q"], out_layout=_lib.LAYOUT_NCHW)
        elif self.kind == "crf_map":
            e.crf_map_dev(d["unary"], d["image"], p, o["labels"])
        elif self.kind == "forward":
            e.dsrg_forward_dev(d["labels"], self.probs, d["cues"], d["image"], p, *TH, o["seeds"], crf_out=o["q"])
        elif self.kind == "crflayer":
            e.crflayer_forward_dev(self.probs, d["image"], p, o["log"], result=o["result"])
        else:
            e.predict_mask_batch_dev([d["scores"]], d["image"], o["labels"], params=p, probs_out=o["q"])
        return {k: v.clone() for k, v in o.items()}


def agree(got, want, what):
    for name in got:
        g, w = got[name].cpu().numpy(), want[name].cpu().numpy()
        if name == "log":
            g, w = np.exp(g), np.exp(w)
        if name in ("seeds", "labels"):
            assert (g != w).sum() <= TIES * g.size, (what, name, int((g != w).sum()))
        else:
            assert np.abs(g - w).max() <= TOL, (what, name, float(np.abs(g - w).max()))


@pytest.mark.parametrize("kind", KINDS)
def test_one_graph_policy_across_sizes(torch_cuda, kind):
    """Two image sizes alternate on one engine on a side stream, four rounds: every call rebuilds the spatial lattice.
    From the second sighting of each key on, every call is one capture or replay, and its outputs agree with a
    graphs-off run."""
    torch = torch_cuda
    eng = api.Engine(B, CAP, CAP, M)
    passes = []
    for i, (H, W) in enumerate(SIZES):
        eng.set_size(H, W)
        passes.append(Pass(torch, eng, kind, H, W, 600 + 10 * i))
    side = torch.cuda.Stream()
    eng.set_graphs(False)
    want = []
    for (H, W), p in zip(SIZES, passes):
        eng.set_size(H, W)
        with torch.cuda.stream(side):
            want.append(p.run())
        side.synchronize()
    eng.set_graphs(True)
    for rnd in range(4):
        for (H, W), p, w in zip(SIZES, passes, want):
            eng.set_size(H, W)
            r0 = eng.graph_replays
            with torch.cuda.stream(side):
                got = p.run()
            side.synchronize()
            assert eng.graph_replays - r0 == (1 if rnd else 0), (kind, rnd, H, W)
            agree(got, w, (kind, rnd, H, W))
    eng.close()


def test_densecrf_objects_across_sizes(torch_cuda, monkeypatch):
    """The DenseCRF kind runs on a pooled engine the caller cannot see, so only its outputs are checked: four rounds
    over two alternating sizes, which capture and replay, against a pooled engine created with graphs off."""
    cases = []
    for i, (H, W) in enumerate(SIZES):
        d = synth.make_problem(650 + i, H, W, image="smooth")
        probs = np.maximum(np.transpose(d["probs"], (1, 2, 0)), 1e-5)
        cases.append((H, W, -np.log(probs).astype(np.float32).ravel(), d["image"].ravel()))

    def run(H, W, costs, im):
        c = api.DenseCRF(W, H, M)
        c.set_unary_energy(costs)
        c.add_pairwise_energy(10.0, 80.0, 80.0, 13.0, 13.0, 13.0, 3.0, 3.0, 3.0, im)
        return c.inference(10), c.map(10)

    _lib.lib().dsrg_densecrf_release_engines()
    monkeypatch.setenv("DSRG_B200_GRAPHS", "0")
    want = [run(*c) for c in cases]
    _lib.lib().dsrg_densecrf_release_engines()
    monkeypatch.delenv("DSRG_B200_GRAPHS")
    try:
        for rnd in range(4):
            for c, (wq, wl) in zip(cases, want):
                q, lab = run(*c)
                assert np.abs(q - wq).max() <= TOL, (rnd, c[:2])
                assert (lab != wl).sum() <= TIES * lab.size, (rnd, c[:2])
    finally:
        _lib.lib().dsrg_densecrf_release_engines()


@pytest.mark.parametrize("kind", KINDS)
def test_notes_after_each_pass(torch_cuda, kind):
    """After each CRF pass over B images, eager, captured or replayed, the engine holds exactly that pass's marginals:
    for B images and no other count.  A refused pass leaves nothing held."""
    torch = torch_cuda
    H, W = SIZES[0]
    eng = api.Engine(B, CAP, CAP, M)
    eng.set_size(H, W)
    p = Pass(torch, eng, kind, H, W, 700)
    labels, cues = p.host["labels"], p.host["cues"]
    side = torch.cuda.Stream()
    r0 = eng.graph_replays
    for i in range(4):   # first sightings with and without the spatial rebuild, then a capture and a replay
        with torch.cuda.stream(side):
            out = p.run()
        side.synchronize()
        held = eng.crf_last_marginals_host(B, _lib.LAYOUT_NHWC if kind == "post" else _lib.LAYOUT_NCHW)
        if "q" in out:
            assert np.array_equal(held, out["q"].cpu().numpy()), (kind, i)
        assert code(eng.srg_last_crf_host, labels[:-1], cues[:-1], *TH) == _lib.E_STATE
        assert code(eng.crf_last_marginals_host, B - 1) == _lib.E_STATE
    assert eng.graph_replays - r0 == 2
    bad = params()
    bad.theta_gamma_x = 0.0
    with torch.cuda.stream(side):
        assert code(p.run, bad) == _lib.E_INVALID
    side.synchronize()
    assert code(eng.srg_last_crf_host, labels, cues, *TH) == _lib.E_STATE
    eng.close()


def test_chunked_host_pass_holds_no_result(torch_cuda, monkeypatch):
    """dsrg_forward_host cuts a batch into chunks that run one after the other on Q0: afterwards Q0 holds the last
    chunk's marginals only, so the engine holds no result.  A batch that runs as one chunk is held."""
    Bh, H, W = 12, 40, 48
    d = synth.make_batch(Bh, H, W, cues="cam", image="smooth", start=720)
    eng = api.Engine(Bh, H, W, M)

    def run():
        q = np.empty_like(d["probs"])
        seeds = eng.dsrg_forward_host(d["labels"], d["probs"].copy(), d["cues"], d["image"], params(), *TH, crf_out=q)
        return seeds, q

    monkeypatch.delenv("DSRG_B200_HOST_SCHEDULE", raising=False)
    run()   # the default schedule at 12 images: 1 | 2 | 2 | 3 | 4
    for n in (4, Bh):
        assert code(eng.srg_last_crf_host, d["labels"][:n], d["cues"][:n], *TH) == _lib.E_STATE, n
        assert code(eng.crf_last_marginals_host, n) == _lib.E_STATE, n
    monkeypatch.setenv("DSRG_B200_HOST_SCHEDULE", str(Bh))
    seeds, q = run()
    assert np.array_equal(eng.crf_last_marginals_host(Bh), q)
    assert np.array_equal(eng.srg_last_crf_host(d["labels"], d["cues"], *TH), seeds)
    eng.close()


def eager_launch_counts(torch):
    """{entry point: LAUNCHES' pair} for every entry point that runs a CRF on a caller-visible engine."""
    H, W = SIZES[0]
    counts = {}
    for kind, entries in [("crf", ["crf_dev", "crf_host"]), ("crf_map", ["crf_map_dev"]),
                          ("forward", ["dsrg_forward_dev", "dsrg_forward_host"]),
                          ("crflayer", ["crflayer_forward_dev", "crflayer_forward_host"]),
                          ("post", ["predict_mask_batch_dev", "predict_mask_batch_host", "predict_mask_dev",
                                    "predict_mask_host"])]:
        for entry in entries:
            eng = api.Engine(B, H, W, M)
            eng.set_graphs(False)
            p = Pass(torch, eng, kind, H, W, 800)
            h, dv = p.host, p.dev
            call = {
                "crf_host": lambda: eng.crf_host(h["unary"], h["image"], params(), out_layout=_lib.LAYOUT_NCHW),
                "dsrg_forward_host": lambda: eng.dsrg_forward_host(h["labels"], h["probs"].copy(), h["cues"],
                                                                   h["image"], params(), *TH),
                "crflayer_forward_host": lambda: eng.crflayer_forward_host(h["probs"].copy(), h["image"], params(),
                                                                           result=np.empty_like(h["probs"])),
                "predict_mask_batch_host": lambda: eng.predict_mask_batch_host([h["scores"]], h["image"], params(),
                                                                               want_probs=True),
                "predict_mask_dev": lambda: eng.predict_mask_dev([dv["scores"][0]], dv["image"][0],
                                                                 p.out["labels"][0], params=params(),
                                                                 probs_out=p.out["q"][0]),
                "predict_mask_host": lambda: eng.predict_mask_host([h["scores"][0]], h["image"][0], params(),
                                                                   want_probs=True),
            }.get(entry, p.run)
            eng.take_launch_count()
            n = []
            for _ in range(2):
                call()
                torch.cuda.synchronize()
                n.append(eng.take_launch_count())
            counts[entry] = tuple(n)
            eng.close()
    return counts


def test_eager_launch_counts_unchanged(torch_cuda, monkeypatch):
    monkeypatch.setenv("DSRG_B200_WIRE", "0")   # the host pipeline's wire format depends on the host's thread count
    monkeypatch.delenv("DSRG_B200_HOST_SCHEDULE", raising=False)
    monkeypatch.delenv("DSRG_B200_HOST_CHUNK", raising=False)
    counts = eager_launch_counts(torch_cuda)
    print("[launches]", counts)
    assert counts == LAUNCHES
