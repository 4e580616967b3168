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


def mf64_problem_params(sf, zero=None, n_iters=10):
    """api.crf_params(sf) for an n_iters run, with w1 ("w1") or w2 ("w2") set to 0 to isolate one lattice."""
    from dsrg_b200 import api
    p = api.crf_params(sf, maxiter=n_iters)
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
    """The oracle's bilateral lattice size of one (H,W,3) image (phantom lanes included, as the engine counts)."""
    from oracle import crf_oracle
    H, W = image.shape[:2]
    c = crf_oracle.DenseCRF(W, H, 1)
    c.set_unary_energy(np.zeros(H * W, np.float32))
    c.add_pairwise_energy(10, 80 / sf, 80 / sf, cf, cf, cf, 3, 3 / sf, 3 / sf, image.ravel())
    return int(c.lattice(1).M)


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


def predict_tile_paths(images, sf, sm_count, cf=13):
    """What tiles.cu does to each tile of a mean-field pass over `images` (B,H,W,3) with crf_params(sf, cf), from the
    oracle's own lattices.  Returns {"sp": kinds (ntiles,), "bi": kinds (B, ntiles), "hybrid_tiles": n}; a kind is
    "smem" (the tile's distinct vertices fit the shared-memory list), "direct" (overflow tile on k_mf_tile's direct
    path) or "hybrid" (k_mf_tile_hy).  Only the bilateral lattice has hybrid tiles; `hybrid_tiles` is the count the
    engine reports after k_tile_demote."""
    from oracle import crf_oracle
    k = csrc_constants()
    B, H, W = images.shape[:3]
    tiles_x, tile_w, tiles_y = tile_geometry(H, W)
    ntiles = tiles_x * tiles_y
    ys, xs = np.mgrid[0:H, 0:W]
    tile_of = ((ys // k["kTileH"]) * tiles_x + xs // tile_w).ravel()
    npix = np.bincount(tile_of, minlength=ntiles)
    gate = ntiles * B >= 16 * sm_count                             # common.cuh: hybrid_tiles_on
    sp_kinds, bi_kinds = None, np.empty((B, ntiles), object)
    for b in range(B):
        c = crf_oracle.DenseCRF(W, H, 1)
        c.set_unary_energy(np.zeros(H * W, np.float32))
        c.add_pairwise_energy(10, 80 / sf, 80 / sf, cf, cf, cf, 3, 3 / sf, 3 / sf, images[b].ravel())
        for lat, maxa in ((0, k["DSRG_MAXLOC_SP"]), (1, k["DSRG_MAXLOC_BI"])):
            if lat == 0 and b > 0:
                continue                                           # one spatial lattice serves the batch
            off = c.lattice(lat).offset.astype(np.int64)          # (N, d+1): the vertex of every (pixel, r)
            keys = tile_of[:, None] * (int(off.max()) + 1) + off
            uniq, cnt = np.unique(keys.ravel(), return_counts=True)
            utile = uniq // (int(off.max()) + 1)
            nvert = np.bincount(utile, minlength=ntiles)
            kinds = np.where(nvert > maxa, "direct", "smem").astype(object)
            if lat == 1 and gate:
                for t in np.nonzero(nvert > maxa)[0]:
                    if _hybrid_cover_ok(cnt[utile == t], npix[t], k):
                        kinds[t] = "hybrid"
            if lat == 0:
                sp_kinds = kinds
            else:
                bi_kinds[b] = kinds
    nhy = int((bi_kinds == "hybrid").sum())
    if nhy < k["DSRG_HY_MIN_TILES"] * sm_count:                    # k_tile_demote
        bi_kinds[bi_kinds == "hybrid"] = "direct"
        nhy = 0
    return {"sp": sp_kinds, "bi": bi_kinds, "hybrid_tiles": nhy}
