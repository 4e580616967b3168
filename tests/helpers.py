"""Shared helpers of the parity tests (inputs identical to tests/golden/make_golden.py)."""
import hashlib
import importlib.util
import os
import re

import numpy as np

from dsrg_b200 import synth

_spec = importlib.util.spec_from_file_location(
    "make_golden", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_golden.py"))
make_golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(make_golden)


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def renorm64(q_nchw):
    """pylayers.py:328-330 on a float32 (N,C,H,W) array of raw CRF marginals."""
    from oracle import crf_oracle
    return crf_oracle.renormalise(q_nchw)   # the reference's layout decides the float64 summation order


def srg_case_inputs(name):
    for n, H, W, cues, index, tweak in make_golden.SRG_CASES:
        if n == name:
            return make_golden.srg_inputs(H, W, cues, index, tweak)
    raise KeyError(name)


def crf_case_inputs(name):
    for i, (n, H, W, var, sf, kind) in enumerate(make_golden.CRF_CASES):
        if n == name:
            im, unary = make_golden.crf_inputs(H, W, var, kind, i)
            return im, unary, sf
    raise KeyError(name)


# ---- label counts: the cases of test_gpu_label_counts.py (checked on the CPU by test_label_counts_cpu.py) ----
MAX_FUSED = 32                       # DSRG_MAX_LABELS: above it the label-chunked path (meanfield_wide.cu)
FUSED_SHAPES = {"smooth": (37, 45), "noise": (41, 41)}
FUSED_CONFIGS = [("smooth", 1.0), ("noise", 1.0), ("smooth", 12.0)]   # (image, scale factor), B = 2
FUSED_ITER_M = [1, 6, 12, 15, 17, 24, 27, 32]                          # one M per MP for n_iters 1 and 2
HYBRID_M = [1, 6, 9, 16, 18, 24, 25, 32]                               # one M per MP on textured 321x321 images
HYBRID_SHAPE, HYBRID_B, HYBRID_START = (321, 321), 5, 70
WIDE_M = [33, 34, 35, 36, 64, 127, 128, 129, 200, 253, 255]
WIDE_SHAPES = {"smooth": (29, 37), "noise": (19, 23)}
RENORM_M = [1, 7, 8, 9, 16, 17, 21, 32, 33, 127, 128, 129, 136, 255]


def oracle_batch(image, unary, sf, n_iters=10):
    from oracle import crf_oracle
    return np.stack([crf_oracle.CRF(image[b], unary[b], n_iters, sf) for b in range(image.shape[0])])


def crf_both_layouts(torch, eng, unary, image, params):
    """crf_dev on NHWC unaries (init kernel) and on NCHW ones (read in place by the tile kernel); both NHWC out."""
    from dsrg_b200 import api
    d_im = torch.from_numpy(image).cuda()
    d_un = torch.from_numpy(unary).cuda()
    d_out = torch.empty_like(d_un)
    eng.crf_dev(d_un, d_im, params, d_out)
    nhwc = d_out.cpu().numpy()
    d_nchw = d_un.permute(0, 3, 1, 2).contiguous()
    d_out2 = torch.empty_like(d_nchw)
    eng.crf_dev(d_nchw, d_im, params, d_out2, api.LAYOUT_NCHW, api.LAYOUT_NCHW)
    return nhwc, d_out2.permute(0, 2, 3, 1).cpu().numpy()


# ---- scale: the cases of test_gpu_scale.py (checked on the CPU by test_scale_cpu.py) ----
# bench.py's workloads restated, not imported (test_scale_cpu.py pins them to bench.py's literals)
BENCH_WORKLOADS = {
    #            H    W    B   what
    "train41": (41, 41, 20, "crf+srg"),
    "dsrg321": (321, 321, 64, "crf+srg"),
    "crf321": (321, 321, 64, "crf"),
    "full513": (513, 513, 16, "crf+srg+loss"),
}
BENCH_M, BENCH_T_ITERS, BENCH_TH, BENCH_CF, BENCH_UNIQUE = 21, 10, (0.99, 0.85), 13, 8


def bench_sf(workload):
    return 12.0 if workload == "train41" else 1.0


# (workload, image variant, the branch of the bilateral pair blur the batch takes: see blur_branch)
SCALE_CASES = [("dsrg321", "smooth", "gate1"), ("dsrg321", "photo", "gate1"), ("dsrg321", "noise", "gate2"),
               ("crf321", "smooth", "gate1"), ("full513", "smooth", "gate1"), ("train41", "smooth", "ungated")]


def bench_unique(workload, variant):
    """The distinct problems of bench.py's batch: synth_batch repeats the first BENCH_UNIQUE cyclically."""
    H, W, B, _ = BENCH_WORKLOADS[workload]
    return synth.make_batch(min(B, BENCH_UNIQUE), H, W, cues="cam", image=variant)


def sample_indices(B, seed):
    """The images of a batch that are compared with the oracle: both ends, the middle and one seeded draw."""
    return sorted({0, 1, B // 2, B - 2, B - 1, int(np.random.RandomState(seed).randint(2, B - 2))})


# gate 2 of the bilateral pair blur at every padded label count: two noise images of 224 x 224 (~96 k rows each)
GATE2_M = HYBRID_M
GATE2_SHAPE, GATE2_SEED = (224, 224), 60
# (name, H, W, image of each batch entry, branch): both sides of the device-side row gate and of the host-side
# capacity switch
SWITCH_CASES = [("mixed224", 224, 224, ("noise", "smooth"), "gate1"),
                ("noise200", 200, 200, ("noise", "noise"), "gate2"),
                ("noise104x105", 104, 105, ("noise", "noise"), "ungated"),
                ("noise105x105", 105, 105, ("noise", "noise"), "gate1")]
COCO_SHAPE, COCO_M = (427, 640), 81                 # DenseCRF(W, H, 81) of the COCO tool at a COCO image's size
WIDE_BIG_SHAPE, WIDE_BIG_M = (105, 105), 255        # the most labels, on a lattice above the capacity switch


# ---- host-buffer pipeline: the cases of test_gpu_wire.py (checked on the CPU by test_wire_cpu.py) ----
# What crosses PCIe in each wire mode (wire.cu: host_pass_impl): name -> (environment, host threads it runs with)
WIRE_MODES = {
    "bits": ({"DSRG_B200_HOST_THREADS": "8"}, 8),                           # cue bits, seed bits, clamp mask
    "floats": ({"DSRG_B200_HOST_THREADS": "1"}, 1),                         # floats plus the clamp mask
    "raw": ({"DSRG_B200_HOST_THREADS": "8", "DSRG_B200_WIRE": "0"}, 8),     # floats and a full probs D2H
}
# case -> steps; a step is (engine (maxB, Hcap, Wcap, M), image size (H, W), batch B, host chunk cap,
# DSRG_B200_HOST_SCHEDULE or None).  Consecutive steps with the same engine tuple share one engine.
WIRE_CASES = {
    "bench": [((64, 321, 321, 21), (321, 321), 64, 0, None)],
    "mixed_cues": [((12, 45, 52, 21), (45, 52), 12, 0, "3,4,5")],
    "wide": [((6, 37, 45, 81), (37, 45), 6, 2, None)],
    "reshaped": [((8, 64, 80, 21), (41, 41), 5, 0, None), ((8, 64, 80, 21), (64, 80), 8, 0, None),
                 ((4, 2, 3, 21), (1, 1), 4, 0, "1,1,2"), ((4, 2, 3, 21), (2, 3), 4, 0, "1,1,2")],
}
WIRE_SF = {"bench": 1.0, "mixed_cues": 12.0, "wide": 1.0, "reshaped": 12.0}
# cue values that are neither 0 nor 1, as (image, value); each goes on a class the image does not have, so it is
# never grown over and must come back unchanged
WIRE_NONBINARY = {"mixed_cues": [(3, 0.5), (5, 2.0), (6, -1.0)], "wide": [(3, 0.5), (3, 2.0), (3, -1.0)]}
# probs values at the clamp's edge (pylayers.py:312: p[p < 1e-4] = 1e-4), on the last image of the first chunk, the
# first image of the second and the batch's last image
WIRE_EDGE_IMAGES = (4, 5, 63)
WIRE_EDGE_PROBS = np.array([1e-4, np.nextafter(np.float32(1e-4), np.float32(0)), 0.0, -0.0, -1e-3,
                            np.finfo(np.float32).smallest_subnormal], np.float32)


def host_schedule(B, maxB, host_chunk=0, schedule=None):
    """wire.cu:host_pass_impl's chunk sizes for a batch of B: DSRG_B200_HOST_SCHEDULE's sizes (each at most maxB
    and what is left; parsing stops at the first entry atoi reads as < 1) with the rest cut into chunks of
    host_chunk (or one), else five chunks that end at 5/64, 14/64, 27/64, 44/64 and all of the batch, each
    capped at host_chunk."""
    def atoi(s):
        m = re.match(r"\s*([+-]?\d+)", s)
        return int(m.group(1)) if m else 0

    sizes, b = [], 0
    if schedule is not None:
        chunk = host_chunk if host_chunk > 0 else B
        for tok in schedule.split(",") if schedule else []:
            if b >= B:
                break
            v = atoi(tok)
            if v < 1:
                break
            v = min(v, maxB, B - b)
            sizes.append(v)
            b += v
        while b < B:
            sizes.append(min(B - b, chunk))
            b += sizes[-1]
    if sizes:
        return sizes
    cap = host_chunk if host_chunk > 0 else B
    edges = (5.0 / 64, 14.0 / 64, 27.0 / 64, 44.0 / 64, 1.0)
    k = 0
    while b < B:
        end = int(edges[k] * B + 0.5) if k < 5 else B
        k += 1
        if end <= b:
            continue
        if end > B or k >= 5:
            end = B
        while b < end:
            sizes.append(min(end - b, cap))
            b += sizes[-1]
    return sizes


def wire_inputs(case, step):
    """labels (B, M), probs and cues (B, M, H, W), image (B, H, W, 3) of one step of a WIRE_CASES case.  "bench" is
    bench.py's batch (bench_unique repeated to 64) with WIRE_EDGE_PROBS on WIRE_EDGE_IMAGES; the others are seeded
    synth batches with the case's WIRE_NONBINARY cue values."""
    _, (H, W), B, _, _ = WIRE_CASES[case][step]
    M = WIRE_CASES[case][step][0][3]
    if case == "bench":
        uniq = bench_unique("dsrg321", "smooth")
        pick = np.arange(B) % len(uniq["probs"])
        d = {k: uniq[k][pick] for k in ("labels", "probs", "cues", "image")}
        for b in WIRE_EDGE_IMAGES:
            d["probs"][b, 2, 10, 10:10 + WIRE_EDGE_PROBS.size] = WIRE_EDGE_PROBS
        return d
    tiny = H * W < 64
    d = synth.make_batch(B, H, W, C=M, cues="random" if tiny else "cam", image="noise" if tiny else "smooth",
                         start=700 + 10 * step)
    d = {k: np.ascontiguousarray(d[k]) for k in ("labels", "probs", "cues", "image")}
    used = {}
    for b, v in WIRE_NONBINARY.get(case, []):
        k = used[b] = used.get(b, -1) + 1
        c = np.nonzero(d["labels"][b] == 0)[0][k]
        d["cues"][b, c, 1 + k, 2 + 2 * k] = v
    return d


def chunk_of(sizes, b):
    """Index of the chunk that holds image b."""
    return int(np.searchsorted(np.cumsum(sizes), b, side="right"))


def wire_call_marker(B, maxB, host_chunk, schedule):
    """The line the worker writes to stderr before each host-buffer call: what the call's schedule derives from."""
    return "[wire call] B=%d maxB=%d chunk=%d schedule=%s" % (B, maxB, host_chunk, schedule or "")


def parse_wire_log(text):
    """Host-buffer calls in a worker's stderr: one dict per wire_call_marker line, with the B / maxB / chunk /
    schedule it states and what the library's DSRG_B200_DEBUG_TIMING lines that follow it report -- the chunk
    sizes of the timeline ("[n img: ...]") and the totals line's "(threads N, chunks K)"."""
    calls = []
    for line in text.splitlines():
        m = re.match(r"\[wire call\] B=(\d+) maxB=(\d+) chunk=(\d+) schedule=(\S*)$", line.strip())
        if m:
            calls.append({"B": int(m.group(1)), "maxB": int(m.group(2)), "chunk": int(m.group(3)),
                          "schedule": m.group(4) or None, "sizes": None, "threads": None, "chunks": None})
            continue
        if not calls:
            continue
        if line.startswith("[dsrg host pass] timeline"):
            calls[-1]["sizes"] = [int(v) for v in re.findall(r"\[(\d+) img:", line)]
        m = re.match(r"\[dsrg host pass\] total .*\(threads (\d+), chunks (\d+)\)\s*$", line)
        if m:
            calls[-1]["threads"], calls[-1]["chunks"] = int(m.group(1)), int(m.group(2))
    return calls


def as_params(params, cf=13, n_iters=10):
    """A copy of a dsrg_crf_params, or api.crf_params(sf, cf, n_iters) for a scale factor sf."""
    from dsrg_b200 import api
    if isinstance(params, api.CrfParams):
        return api.CrfParams.from_buffer_copy(params)
    return api.crf_params(params, cf, n_iters)


def pairwise_args(params):
    """The nine pairwise values of a dsrg_crf_params in add_pairwise_energy's order (wrapper.pyx)."""
    p = params
    return (p.w1, p.theta_alpha_x, p.theta_alpha_y, p.theta_beta_r, p.theta_beta_g, p.theta_beta_b, p.w2,
            p.theta_gamma_x, p.theta_gamma_y)


def oracle_lattices(image, params):
    """The oracle's DenseCRF of one (H,W,3) image under `params` (sf or dsrg_crf_params); .lattice(k) and .norm(k)."""
    from oracle import crf_oracle
    H, W = image.shape[:2]
    c = crf_oracle.DenseCRF(W, H, 1)
    c.set_unary_energy(np.zeros(H * W, np.float32))
    c.add_pairwise_energy(*pairwise_args(as_params(params)), np.ascontiguousarray(image).ravel())
    return c


def mf64_problem_params(sf, zero=None, n_iters=10):
    """api.crf_params(sf) (or a copy of the dsrg_crf_params `sf`) for an n_iters run, with w1 ("w1") or w2 ("w2") set
    to 0 to isolate one lattice."""
    p = as_params(sf)
    p.n_iters = n_iters
    if zero:
        setattr(p, zero, 0.0)
    return p


# ---- float64 mean field: the cases of test_gpu_meanfield64.py (checked on the CPU by test_meanfield64_cpu.py) ----
MF64_ITERS = (1, 2, 3, 10)
MF64_GATE2_M = [6, 24, 32]
MF64_WIDE_M = [M for M in WIDE_M if M in (33, 81, 128, 255)]
# (H, W, image): N % 4 = 0, 1, 2, 3, so the last 4-pixel block of the lattice build has 0..3 phantom lanes
MF64_TINY = [(4, 4, "noise"), (3, 7, "noise"), (5, 6, "noise"), (3, 5, "noise")]
MF64_TINY_M, MF64_TINY_SEED = 5, 90
# (path, zeroed weight): each case runs on one lattice only, so a failure names the lattice
MF64_ZERO_W = [(path, w) for path in ("smem", "bi_direct", "sp_direct", "hybrid", "wide") for w in ("w1", "w2")]
MF64_ZERO_W_M = {"smem": 6, "bi_direct": 6, "sp_direct": 6, "hybrid": 24, "wide": 33}
MF64_PATH_CONFIG = {"smem": ("smooth", 1.0), "bi_direct": ("noise", 1.0), "sp_direct": ("smooth", 12.0)}

# The bar of a case after n iterations: BAR_K times the largest max|Q32 - Q64| over the float32 models, at least
# BAR_FLOOR.  The models are the oracle's sequential splat, three shuffled splat orders (the device's float atomics
# add in no fixed order) and two draws of the device's own operation order (meanfield64 arith="device": folded
# weights, an fma slice, exp with a seeded 2^-22 relative error, a reciprocal); each is one draw of float32 rounding
# noise, and the device is one more draw of the same size.  After ten iterations on noise images that noise is
# heavy-tailed (over 40 draws of the device model the largest error was up to 3x the median), so BAR_K = 4 leaves
# room for the device's draw to land beyond the largest of the six we sampled without letting through an error that
# is itself several times the float32 noise.  A bar belongs to one image.  BAR_FLOOR covers the
# exp of ex2.approx where the models agree exactly (M = 1, where Q is 1): a 2^-22 relative error in the numerator and
# in the sum of the soft-max, on a Q of at most 1, is at most 2^-21; the floor is twice that.
BAR_K = 4.0
BAR_FLOOR = 2.0 ** -20
BAR_MODELS = [dict(splat_order=None), dict(splat_order=1), dict(splat_order=2), dict(splat_order=3),
              dict(splat_order=4, arith="device"), dict(splat_order=5, arith="device", exp_seed=1)]


def mf64_truth_and_bar(problem, unary, iters=MF64_ITERS, extra=()):
    """(Q64 after every n of `iters`, {n: bar}, {n: largest model error}) for one image's (H, W, M) unary; `extra`
    are more float32 runs (meanfield64.Problem.run keywords) returned as a list of {n: Q}.  The float64 run and the
    models run on threads (numpy's gathers and scipy's sparse products release the GIL)."""
    import numpy as np
    from concurrent.futures import ThreadPoolExecutor
    T = max(iters)
    problem.norms(np.float64)
    jobs = [dict(dtype=np.float64)] + [dict(dtype=np.float32, **m) for m in BAR_MODELS] + \
        [dict(dtype=np.float32, **e) for e in extra]
    for j in jobs:
        problem.norms(j["dtype"], j.get("splat_order"))
    with ThreadPoolExecutor(min(len(jobs), os.cpu_count() or 1)) as ex:
        runs = list(ex.map(lambda kw: problem.run(unary, T, **kw), jobs))
    q64 = {n: runs[0][n] for n in iters}
    spread = {n: max(float(np.abs(r[n] - q64[n]).max()) for r in runs[1:1 + len(BAR_MODELS)]) for n in iters}
    bar = {n: max(BAR_K * spread[n], BAR_FLOOR) for n in iters}
    return q64, bar, spread, [{n: r[n] for n in iters} for r in runs[1 + len(BAR_MODELS):]]



class Truth(object):
    """The float64 marginals and the bar of the compared images of a batch, each image's lattices built once."""

    def __init__(self, image, params, images):
        from oracle import meanfield64
        self.images = list(images)
        self.problems = {b: meanfield64.Problem(image[b], params) for b in self.images}

    def __call__(self, unary):
        q64, bars = {}, {}
        for b in self.images:
            q64[b], bars[b], _, _ = mf64_truth_and_bar(self.problems[b], unary[b])
        return q64, bars

def seeded_images(H, W, kinds, seed):
    return np.stack([synth.make_image(np.random.RandomState(seed + b), H, W, k) for b, k in enumerate(kinds)])


def blur_cached_rows():
    """meanfield.cu's default kBlurCachedRows (DSRG_BLUR_CACHED_ROWS)."""
    import re
    src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "dsrg_b200", "csrc",
                            "meanfield.cu")).read()
    return int(re.search(r"#define\s+DSRG_BLUR_CACHED_ROWS\s+(\d+)\s*$", src, re.M).group(1))


def blur_branch(H, W, vb):
    """Which kernel runs the bilateral pair passes (meanfield.cu: blur_all, k_mf_blur) for a batch of H x W images
    whose bilateral lattices have vb[b] vertices: "ungated" when no image of this size can have more than
    kBlurCachedRows rows (capv = (N + P) * 6, P the phantom lanes of api.cu:lattice_shape), else "gate1" (full
    occupancy) when the batch has at most kBlurCachedRows rows per image on average (a row per vertex plus each
    image's zero row), "gate2" (4 CTAs per SM) when it has more."""
    rows = blur_cached_rows()
    N = H * W
    if (N + (4 - N % 4) % 4) * 6 <= rows:
        return "ungated"
    return "gate2" if sum(int(v) + 1 for v in vb) > rows * len(vb) else "gate1"


def bilateral_vertices(image, sf=1.0, cf=13):
    """The oracle's bilateral lattice size of one (H,W,3) image (phantom lanes included, as the engine counts) under
    crf_params(sf, cf) or the dsrg_crf_params `sf`."""
    return int(oracle_lattices(image, as_params(sf, cf)).lattice(1).M)


def padded(M):
    """MP: the label count rounded up to the lane width of the value rows (api.cu)."""
    return (M + 3) // 4 * 4


def tail1(M):
    """The fused kernels' last label quad holds one real label (meanfield.cu: tile_slice_smem)."""
    return M == padded(M) - 3


def small_image(rng, H, W, img):
    """synth's images at a small shape.  "smooth" is the corner of an image eight times larger: synth blurs in
    proportion to the size, and at 40 pixels its smooth image already overflows every bilateral tile."""
    if img == "smooth":
        return np.ascontiguousarray(synth.make_image(rng, 8 * H, 8 * W, img)[:H, :W])
    return synth.make_image(rng, H, W, img)


def fused_images(img, B=2):
    H, W = FUSED_SHAPES[img]
    return np.stack([small_image(np.random.RandomState(17 + b), H, W, img) for b in range(B)])


def wide_images(img, B=2):
    H, W = WIDE_SHAPES[img]
    return np.stack([small_image(np.random.RandomState(29 + b), H, W, img) for b in range(B)])


def hybrid_images():
    return synth.make_batch(HYBRID_B, *HYBRID_SHAPE, image="photo", start=HYBRID_START)["image"]


def log_unary(B, H, W, M, seed, scale=2.0):
    """(B,H,W,M) float32 log-probabilities with a few confident regions (label 0 and label M-1 win a block each)."""
    rng = np.random.RandomState(seed)
    logits = rng.randn(B, H, W, M) * scale
    logits[:, : H // 3, : W // 2, 0] += 4
    logits[:, H // 2:, W // 3:, M - 1] += 4
    pr = np.exp(logits - logits.max(-1, keepdims=True))
    pr /= pr.sum(-1, keepdims=True)
    return np.log(np.maximum(pr, 1e-5)).astype(np.float32)


_CONSTS = None


def csrc_constants():
    """The compile-time defaults of the tile geometry and the tile-path thresholds, read from csrc/common.cuh."""
    global _CONSTS
    if _CONSTS is None:
        import re
        src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "dsrg_b200", "csrc",
                                "common.cuh")).read()
        c = {k: int(v) for k, v in re.findall(r"#define\s+(DSRG_\w+)\s+(\d+)\s*$", src, re.M)}
        m = re.search(r"constexpr int kTileW = (\d+), kTileH = (\d+);", src)
        c["kTileW"], c["kTileH"] = int(m.group(1)), int(m.group(2))
        _CONSTS = c
    return _CONSTS


def tile_geometry(H, W):
    """api.cu:engine_shape: tiles of tile_w x kTileH pixels, the width split evenly."""
    k = csrc_constants()
    tiles_x = -(-W // k["kTileW"])
    tile_w = -(-W // tiles_x)
    tiles_y = -(-H // k["kTileH"])
    return tiles_x, tile_w, tiles_y


def _hybrid_cover_ok(counts, npix, k):
    """k_tile_build's rule for an overflow tile (tiles.cu): the smallest incidence count c >= 2 whose vertices (those
    touched c times or more) fit into DSRG_MAXLOC_HY, plus the first `extra` vertices of the next bucket, must cover
    DSRG_HY_MIN_COVER percent of the tile's incidences."""
    maxloc = k["DSRG_MAXLOC_HY"]
    threads = k["kTileW"] * k["kTileH"]
    hist = np.bincount(counts, minlength=threads + 2)
    nv_ge = np.cumsum(hist[::-1])[::-1]                          # vertices with >= c incidences
    ni_ge = np.cumsum((hist * np.arange(hist.size))[::-1])[::-1]  # their incidences
    c = next(c for c in range(2, threads + 1) if nv_ge[c] <= maxloc)
    extra = maxloc - nv_ge[c] if c - 1 >= 2 else 0
    covered = ni_ge[c] + extra * (c - 1)
    return covered * 100 >= npix * 6 * k["DSRG_HY_MIN_COVER"]


def tile_of_pixels(H, W):
    """The tile index and the thread index in the tile of every pixel (row-major), tiles.cu's geometry."""
    k = csrc_constants()
    tiles_x, tile_w, _ = tile_geometry(H, W)
    ys, xs = np.mgrid[0:H, 0:W]
    ty, tx = ys // k["kTileH"], xs // tile_w
    return (ty * tiles_x + tx).ravel(), ((ys - ty * k["kTileH"]) * k["kTileW"] + xs - tx * tile_w).ravel()


def lattice_tile_kinds(off, H, W, which, hybrid_on):
    """k_tile_build's kind of every tile of one lattice (before k_tile_demote), from the oracle's offsets (N, d+1)."""
    k = csrc_constants()
    tiles_x, _, tiles_y = tile_geometry(H, W)
    ntiles = tiles_x * tiles_y
    tile_of, _ = tile_of_pixels(H, W)
    npix = np.bincount(tile_of, minlength=ntiles)
    maxa = k["DSRG_MAXLOC_SP"] if which == 0 else k["DSRG_MAXLOC_BI"]
    off = off.astype(np.int64)
    keys = tile_of[:, None] * (int(off.max()) + 1) + off
    uniq, cnt = np.unique(keys.ravel(), return_counts=True)
    utile = uniq // (int(off.max()) + 1)
    nvert = np.bincount(utile, minlength=ntiles)
    kinds = np.where(nvert > maxa, "direct", "smem").astype(object)
    if which == 1 and hybrid_on:
        for t in np.nonzero(nvert > maxa)[0]:
            if _hybrid_cover_ok(cnt[utile == t], npix[t], k):
                kinds[t] = "hybrid"
    return kinds


def hybrid_tiles_on(H, W, B, sm_count):
    """common.cuh: hybrid_tiles_on (for label counts of the fused path)."""
    tiles_x, _, tiles_y = tile_geometry(H, W)
    return tiles_x * tiles_y * B >= 16 * sm_count


def demote_hybrid_tiles(bi_kinds, sm_count):
    """k_tile_demote on the bilateral kinds (B, ntiles), in place; returns the hybrid-tile count the engine reports."""
    nhy = int((bi_kinds == "hybrid").sum())
    if nhy < csrc_constants()["DSRG_HY_MIN_TILES"] * sm_count:
        bi_kinds[bi_kinds == "hybrid"] = "direct"
        nhy = 0
    return nhy


def predict_tile_paths(images, sf, sm_count, cf=13):
    """What tiles.cu does to each tile of a mean-field pass over `images` (B,H,W,3) with crf_params(sf, cf) or the
    dsrg_crf_params `sf`, from the oracle's own lattices.  Returns {"sp": kinds (ntiles,), "bi": kinds (B, ntiles),
    "hybrid_tiles": n}; a kind is "smem" (the tile's distinct vertices fit the shared-memory list), "direct" (overflow
    tile on k_mf_tile's direct path) or "hybrid" (k_mf_tile_hy).  Only the bilateral lattice has hybrid tiles;
    `hybrid_tiles` is the count the engine reports after k_tile_demote.  A batch that repeats an image builds its
    lattices once."""
    B, H, W = images.shape[:3]
    params = as_params(sf, cf)
    gate = hybrid_tiles_on(H, W, B, sm_count)
    sp_kinds, bi_kinds = None, np.empty((B, tile_geometry(H, W)[0] * tile_geometry(H, W)[2]), object)
    seen = {}
    for b in range(B):
        key = digest(images[b])
        if key not in seen:
            c = oracle_lattices(images[b], params)
            if b == 0:                                             # one spatial lattice serves the batch
                sp_kinds = lattice_tile_kinds(c.lattice(0).offset, H, W, 0, gate)
            seen[key] = lattice_tile_kinds(c.lattice(1).offset, H, W, 1, gate)
        bi_kinds[b] = seen[key]
    nhy = demote_hybrid_tiles(bi_kinds, sm_count)
    return {"sp": sp_kinds, "bi": bi_kinds, "hybrid_tiles": nhy}


# ---- the lattice build, table by table: the cases of test_gpu_lattice_exact.py (checked on the CPU by
# test_lattice_exact_cpu.py) ----
def tile_major_pos(H, W):
    """Position of every pixel (row-major order) in tile-major order: tile index, then thread index in the tile."""
    k = csrc_constants()
    tile_of, tid = tile_of_pixels(H, W)
    return tile_of * k["kTileW"] * k["kTileH"] + tid


def check_order(off, H, W):
    """ids follow the first tile-major incidence; vertices without one (the phantom lanes') come last.
    Returns the number of vertices that pixels touch."""
    dp1 = off.shape[0]
    ids = off - 1
    key = tile_major_pos(H, W)[None, :] * dp1 + np.arange(dp1)[:, None]
    V_pix = int(ids.max()) + 1
    first = np.full(V_pix, np.iinfo(np.int64).max)
    np.minimum.at(first, ids.ravel(), key.ravel())
    assert (first < np.iinfo(np.int64).max).all(), "ids touched by pixels are not contiguous from 0"
    assert (np.diff(first) > 0).all(), "ids do not increase with the first tile-major incidence"
    return V_pix


def check_against_oracle(off, nbr, lat, V_pix):
    """The engine's tables are the oracle's lattice renamed: one-to-one vertex mapping, same neighbours.  Returns the
    mapping (oracle id -> engine id, -1 for the vertices only the phantom lanes touch)."""
    dp1, V = off.shape[0], nbr.shape[1] - 1
    assert V == lat.M
    o = lat.offset.T                                   # (d+1, N) oracle ids
    m = np.full(lat.M, -1, np.int64)
    m[o.ravel()] = off.ravel() - 1
    assert np.array_equal(m[o], off - 1), "a vertex maps to two ids"
    seen = m >= 0
    assert np.unique(m[seen]).size == seen.sum() == V_pix
    assert (nbr[:, 0] == 0).all(), "the zero row must point at itself"
    for j in range(dp1):
        for on, col in ((lat.n1[j], 0), (lat.n2[j], 1)):
            got = nbr[j, m[seen] + 1, col]
            tgt = on[seen]
            want = np.where(tgt < 0, 0, m[np.maximum(tgt, 0)] + 1)
            mapped = (tgt < 0) | (m[np.maximum(tgt, 0)] >= 0)
            assert np.array_equal(got[mapped], want[mapped]), "axis %d neighbour %d" % (j, col)
            # a neighbour that no pixel touches is one of the phantom lanes' vertices, numbered last
            assert (got[~mapped] > V_pix).all()
    return m


def phantom_lanes(N):
    """api.cu:lattice_shape: the tail of the last 4-pixel block (permutohedral.cpp:196)."""
    return (4 - N % 4) % 4


def lattice_scales(d):
    """api.cu:lattice_scales (permutohedral.cpp:179-182)."""
    inv_std_dev = np.float32(np.sqrt(2.0 / 3.0) * (d + 1))
    return np.array([1.0 / np.sqrt((i + 2) * (i + 1)) * np.float64(inv_std_dev) for i in range(d)], np.float32)


def key_range_ok(sigma, H, W):
    """api.cu:key_range_ok for a lattice with the feature sigmas `sigma` (x, y[, c0, c1, c2], float32 values)."""
    d = len(sigma)
    sig = [float(np.float32(s)) for s in sigma]
    scale = lattice_scales(d)
    fmax = [(W - 1) / sig[0], (H - 1) / sig[1]] + [255.0 / sig[i] for i in range(2, d)]
    total = big = 0.0
    for i in range(d):
        cf = abs(fmax[i]) * float(scale[i])
        total += cf
        if (i + 1) * cf > big:
            big = (i + 1) * cf
    bound = total + big + 3.0 * (d + 1) + 2
    return bool(bound < float((1 << ((16 if d == 2 else 12) - 1)) - 1) and np.isfinite(bound))


def lattice_sigmas(params, which):
    """The feature sigmas of lattice `which` (0 spatial, 1 bilateral) under a dsrg_crf_params."""
    if which == 0:
        return [params.theta_gamma_x, params.theta_gamma_y]
    return [params.theta_alpha_x, params.theta_alpha_y, params.theta_beta_r, params.theta_beta_g, params.theta_beta_b]


def lattice_features(image, sigma):
    """(N + phantom lanes, d) float32 features of an (H, W, 3) image, as k_lattice_insert forms them (x / sigma_x,
    y / sigma_y, colour / sigma_c, each one float32 division); the phantom lanes' rows are 0."""
    H, W = image.shape[:2]
    d = len(sigma)
    ys, xs = np.mgrid[0:H, 0:W]
    cols = [xs.ravel().astype(np.float32) / np.float32(sigma[0]), ys.ravel().astype(np.float32) / np.float32(sigma[1])]
    px = image.reshape(-1, 3)
    cols += [px[:, c].astype(np.float32) / np.float32(sigma[2 + c]) for c in range(d - 2)]
    f = np.stack(cols, 1)
    return np.concatenate([f, np.zeros((phantom_lanes(H * W), d), np.float32)])


def lattice_insert(f):
    """k_lattice_insert's arithmetic restated in float32 (one rounding per operation, no contraction) on features
    (n, d): elevate, the closest 0-coloured simplex, the rank, the barycentric weights and the d+1 vertex keys.
    Returns keys (n, d+1, d) int64 and bary (n, d+1) float32."""
    f32 = np.float32
    n, d = f.shape
    dp1 = f32(d + 1)
    scale = lattice_scales(d)
    el = np.zeros((n, d + 1), f32)
    sm = np.zeros(n, f32)
    for j in range(d, 0, -1):
        cf = f[:, j - 1] * scale[j - 1]
        el[:, j] = sm - f32(j) * cf
        sm = sm + cf
    el[:, 0] = sm
    inv = f32(1.0) / dp1
    v = np.rint(inv * el)
    rem0 = v * dp1
    isum = v.astype(np.int64).sum(1)
    rank = np.zeros((n, d + 1), np.int64)
    for k in range(d):
        di = el[:, k] - rem0[:, k]
        for j in range(k + 1, d + 1):
            lt = di < (el[:, j] - rem0[:, j])
            rank[:, k] += lt
            rank[:, j] += ~lt
    rank += isum[:, None]
    low, high = rank < 0, rank >= d + 1
    rank[low] += d + 1
    rem0[low] = rem0[low] + dp1
    rank[high] -= d + 1
    rem0[high] = rem0[high] - dp1
    bc = np.zeros((n, d + 2), f32)
    ar = np.arange(n)
    for k in range(d + 1):
        val = (el[:, k] - rem0[:, k]) * inv
        p = d - rank[:, k]
        bc[ar, p] = bc[ar, p] + val
        bc[ar, p + 1] = bc[ar, p + 1] - val
    bc[:, 0] = bc[:, 0] + (f32(1.0) + bc[:, d + 1])
    keys = np.empty((n, d + 1, d), np.int64)
    for r in range(d + 1):
        canon = np.where(rank[:, :d] <= d - r, r, r - (d + 1))
        keys[:, r] = rem0[:, :d].astype(np.int64) + canon
    return keys, bc[:, :d + 1]


def max_abs_key(image, sigma):
    return int(np.abs(lattice_insert(lattice_features(image, sigma))[0]).max())


def renum_key_limit(H, W):
    """The largest renumbering key of an engine of H x W (lattice.cu: pos * (d+1) + r of the bilateral lattice, pos
    up to the phantom lanes' ntiles * kTileThreads), which api.cu keeps below kNoKey."""
    k = csrc_constants()
    tiles_x, _, tiles_y = tile_geometry(H, W)
    return tiles_x * tiles_y * k["kTileW"] * k["kTileH"] * 6 + 5


K_NO_KEY = 0x7F7F7F7F                                  # common.cuh: kNoKey
RENUM_MAX_H_W1 = 11140944                              # the tallest one-pixel-wide engine whose keys stay below it

# A float32 sigma at which api.cu:key_range_ok only just passes: the smallest one (the others fixed), so that the next
# float32 below it is refused
EDGE_SHAPE, EDGE_B = (96, 128), 2
# bilateral: per-axis sigmas that give each feature about the share of the bound that maximises the largest key
# (cf_i ~ 1/(i+1)); alpha_x is the one at the edge
EDGE_BI = (0.71240306, 0.616, 1.753, 1.81, 1.848)
EDGE_SP = (0.016331082, 0.016331082)                   # spatial: both at the edge
EDGE_MAX_KEY = {0: 19287, 1: 1412}                     # the largest |key| coordinate the edge images reach


def edge_params(spatial=EDGE_SP, bilateral=EDGE_BI):
    from dsrg_b200 import api
    p = api.crf_params(1.0, maxiter=1)
    p.theta_gamma_x, p.theta_gamma_y = spatial
    (p.theta_alpha_x, p.theta_alpha_y, p.theta_beta_r, p.theta_beta_g, p.theta_beta_b) = bilateral
    return p


def check_restatement(image, params):
    """The restated insert gives the oracle's barycentric weights bit for bit and its vertices one to one (real
    pixels and phantom lanes); returns the largest |key| per lattice."""
    c = oracle_lattices(image, params)
    N = image.shape[0] * image.shape[1]
    out = {}
    for which in (0, 1):
        lat = c.lattice(which)
        keys, bary = lattice_insert(lattice_features(image, lattice_sigmas(params, which)))
        assert np.array_equal(bary[:N].view(np.uint32), lat.bary.view(np.uint32)), which
        d = keys.shape[2]
        _, ids = np.unique(keys.reshape(-1, d), axis=0, return_inverse=True)
        ids = ids.reshape(-1, d + 1)[:N]
        pairs = np.unique(np.stack([ids.ravel(), lat.offset.ravel()]), axis=1)
        assert pairs.shape[1] == np.unique(ids).size == np.unique(lat.offset).size, which
        assert np.unique(keys.reshape(-1, d), axis=0).shape[0] == lat.M, which     # phantom lanes' vertices too
        out[which] = int(np.abs(keys).max())
    return out


def extreme_image(rng, H, W):
    """Colours 0 and 255 only; the first and last eight pixels of the first and last rows run through all eight
    colour corners, so the largest features meet at the image's corners."""
    im = (rng.randint(0, 2, (H, W, 3)) * 255).astype(np.uint8)
    corners = ((np.arange(8)[:, None] >> np.arange(3)) & 1).astype(np.uint8) * 255
    n = min(8, W)
    for y in {0, H - 1}:
        im[y, :n] = corners[:n]
        im[y, W - n:] = corners[8 - n:]
    return im


# name -> (H, W, B, image kind, sf, M, phantom lanes, tile_w).  Kinds: synth's, "constant", "binary" (0 and 255 only),
# "repeat" (one synth photo B times).  M > 32 takes the label-chunked path.
EXACT_CASES = {
    "1x1": (1, 1, 2, "noise", 1.0, 21, 3, 1),
    "1x38": (1, 38, 2, "noise", 1.0, 21, 2, 19),
    "39x1": (39, 1, 2, "noise", 1.0, 21, 1, 1),
    "2x2": (2, 2, 2, "noise", 1.0, 21, 0, 2),
    "21x33": (21, 33, 2, "photo", 1.0, 21, 3, 17),
    "constant": (41, 41, 2, "constant", 1.0, 21, 3, 21),
    "binary": (45, 52, 2, "binary", 1.0, 21, 0, 26),
    "repeat": (37, 45, 4, "repeat", 12.0, 21, 3, 23),
    "513x513": (513, 513, 2, "smooth", 1.0, 21, 3, 31),
    "coco481x640": (481, 640, 1, "photo", 1.0, 81, 0, 32),
}
EXACT_BENCH = (321, 321, 64)                           # bench.py's batch, distinct images
EXACT_BENCH_CONFIGS = [(img, sf) for img in ("smooth", "photo", "noise") for sf in (12.0, 1.0)]
EXACT_BENCH_FULL = (0, 31, 63)                         # images whose full tables are compared
EXACT_SEED = 500


def exact_images(kind, H, W, B, seed=EXACT_SEED):
    rng = np.random.RandomState(seed)
    if kind == "constant":
        return np.broadcast_to(np.array([90, 140, 200], np.uint8), (B, H, W, 3)).copy()
    if kind == "binary":
        return np.stack([extreme_image(rng, H, W) for _ in range(B)])
    if kind == "repeat":
        return np.stack([synth.make_image(rng, H, W, "photo")] * B)
    return np.stack([small_image(rng, H, W, kind) if H * W < 4096 else synth.make_image(rng, H, W, kind)
                     for _ in range(B)])


# ---- pairwise parameters other than CRF()'s: the cases of test_gpu_crf_params.py (checked on the CPU by
# test_crf_params_cpu.py) ----
# name -> ((w1, theta_alpha x, y, theta_beta r, g, b, w2, theta_gamma x, y), n_iters, image kind, (H, W), B, the
# tile paths the pass must reach as (spatial, bilateral), or None).  Every image is non-square, so an x / y mix-up
# cannot hide behind symmetry.  Kinds: "smooth" and "photo" are synth's, "channels" a smooth red, a textured green and
# a constant blue channel, "binary" helpers.extreme_image.
PARAM_SETS = {
    "aniso_xy": ((10, 50, 120, 13, 13, 13, 3, 2, 5), 10, "smooth", (37, 53), 2, None),
    "aniso_xy_inv": ((10, 120, 50, 13, 13, 13, 3, 5, 2), 10, "smooth", (37, 53), 2, None),   # same images
    "aniso_rgb": ((10, 80, 80, 7, 13, 31, 3, 3, 3), 10, "channels", (37, 53), 2, None),
    "weights": ((4.5, 80, 80, 13, 13, 13, 7, 3, 3), 10, "smooth", (37, 53), 2, None),
    "weights_neg": ((10, 80, 80, 13, 13, 13, -1.5, 3, 3), 10, "smooth", (37, 53), 2, None),
    "decoupled_sp_direct_bi_smem": ((10, 80, 80, 13, 13, 13, 3, 1.0, 1.2), 10, "smooth", (37, 53), 2,
                                    ("direct", "smem")),
    "decoupled_sp_smem_bi_direct": ((10, 3, 4, 2, 2, 2, 3, 3, 3), 10, "smooth", (37, 53), 2, ("smem", "direct")),
    "decoupled_sp_direct_bi_hybrid": ((10, 80, 80, 13, 13, 13, 3, 0.5, 0.6), 10, "photo", (321, 353), 5,
                                      ("direct", "hybrid")),
    "degenerate_x": ((10, 1e4, 80, 13, 13, 13, 3, 1e4, 3), 10, "smooth", (37, 53), 2, None),
    "degenerate_g": ((10, 80, 80, 13, 1e4, 13, 3, 3, 3), 10, "channels", (37, 53), 2, None),
}
PARAM_M, PARAM_WIDE_M = 21, 81
PARAM_WIDE_SETS = ("aniso_xy", "aniso_rgb")            # also run on the label-chunked path
PARAM_TINY = (3, 7)                                    # N % 4 = 1: three phantom lanes
PARAM_SEED = 300
# A strip on which the x terms of both lattices sit at the packed-key limit: the smallest float32 theta_gamma_x
# (theta_alpha_x) that api.cu:key_range_ok passes with theta_gamma_y (theta_alpha_y) fixed.  y is smaller than x,
# so with the two swapped the x term is (W-1)/y and the set is refused.
KEY_EDGE_SHAPE, KEY_EDGE_B = (31, 700), 2
KEY_EDGE_SP = (0.07747016102075577, 0.02)
KEY_EDGE_BI = (2.5485446453094482, 1.0, 13.0, 13.0, 13.0)
KEY_EDGE_MAX_KEY = {0: 17129, 1: 1079}                 # the largest |key| coordinate the strip's images reach


def make_params(values, n_iters=10):
    """A dsrg_crf_params from the nine pairwise values (add_pairwise_energy's order) and n_iters."""
    from dsrg_b200 import api
    p = api.CrfParams()
    (p.w1, p.theta_alpha_x, p.theta_alpha_y, p.theta_beta_r, p.theta_beta_g, p.theta_beta_b, p.w2, p.theta_gamma_x,
     p.theta_gamma_y) = values
    p.n_iters = n_iters
    return p


def set_params(name):
    values, n_iters = PARAM_SETS[name][:2]
    return make_params(values, n_iters)


def set_images(kind, H, W, B, seed=PARAM_SEED):
    if kind == "channels":
        out = []
        for b in range(B):
            rng = np.random.RandomState(seed + b)
            im = small_image(rng, H, W, "smooth").copy()
            im[..., 1] = synth.make_image(rng, H, W, "noise")[..., 1]
            im[..., 2] = 90
            out.append(im)
        return np.stack(out)
    if kind == "photo":
        return synth.make_batch(B, H, W, image="photo", start=seed)["image"]
    if kind == "binary":
        return exact_images("binary", H, W, B, seed)
    return np.stack([small_image(np.random.RandomState(seed + b), H, W, kind) for b in range(B)])


def param_set_images(name):
    _, _, kind, (H, W), B, _ = PARAM_SETS[name]
    return set_images(kind, H, W, B)


def tile_pairing(pred):
    """(spatial, bilateral) path of a predict_tile_paths result: "direct" when a tile overflows, "hybrid" when the
    engine runs hybrid tiles, else "smem"."""
    sp = "direct" if (pred["sp"] == "direct").any() else "smem"
    bi = "hybrid" if pred["hybrid_tiles"] else "direct" if (pred["bi"] == "direct").any() else "smem"
    return sp, bi
