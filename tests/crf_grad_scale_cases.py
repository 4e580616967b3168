"""Cases of the CRF gradient tests at the training and benchmark batch sizes and on large lattices
(test_gpu_crf_grad_scale.py, checked on the CPU by test_crf_grad_scale_cpu.py).

Every slot of a batch is checked, at the cost of a few truths.  A batch holds U distinct problems (image, unary, G):
slot b holds problem pi(b) from a seeded table in which each problem fills several slots and neighbouring slots hold
different problems, and its upstream gradient is s_b * G_pi(b) with s_b in SCALES.  Every gradient (dL/dU, dL/dw,
dL/dmu, dL/dtheta) is linear in G, and a power-of-two scale or a sign is exact in float32, so slot b's truth is s_b
times its problem's truth and its bar |s_b| times that truth's bar (crf_grad_cases.GradTruth,
crf_compat_cases.CompatTruth, crf_kgrad_cases.KgradTruth).  A slot that reads another slot's G, Q_t or lattice rows
misses either through the scale or through the image.

The truths are computed once per problem, on threads (numpy's gathers and scipy's sparse products release the GIL),
and kept for the module's life.
"""
import os
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

import helpers
from crf_compat_cases import CompatTruth, compat_mats
from crf_grad_cases import GradTruth, grad_params, upstream
from crf_kgrad_cases import KgradTruth
from dsrg_b200 import synth
from oracle import meanfield64

SCALES = (0.5, -1.0, 2.0, -0.5, 1.0, -2.0)
M = helpers.BENCH_M                      # 21 labels everywhere
SM_H100 = 132                            # H100 SXM
MU_KIND = "nonsym"

# name -> (H, W, B, sf, U, T of the Potts gradient, T of the theta / mu gradients, the bilateral pair blur's branch
# (helpers.blur_branch)).  train41 runs bench.py's train41 problems, dsrg321 U seeded synth photos.
CASES = {
    "train41": (41, 41, 20, 12.0, 8, 10, 10, "ungated"),
    "dsrg321": (321, 321, 64, 1.0, 4, 10, 3, "gate1"),
}
GATE2_LABELS = helpers.MF64_GATE2_M      # 6, 24, 32: the gate-2 label counts of the float64 forward's tests
GATE2_T = 2
SWITCH_T = 2
PHOTO_START = 90                         # synth.make_batch start of the dsrg321 photos
NOISE_PATCH = (16, 64)                   # the last photo's noise patch: four direct bilateral tiles at 321^2
RESHAPE = (200, 224)                     # the re-shaped engine's smaller size
RESHAPE_U = 2
# (gradient, batch) in order on one Engine(64, 321, 321, 21): theta + Potts first at B = 3, so that the theta buffers
# are allocated at a small batch, then theta + mu
PARTIAL_RUNS = [("theta", 3), ("theta", 64), ("theta", 37), ("theta", 1), ("theta", 64), ("theta_mu", 5),
                ("theta_mu", 64)]
TRAIN_BATCHES = (20, 20, 7)              # nn.dense_crf as a training loop at train41
TABLE_SEED = 1000


def slot_table(B, U, seed):
    """(pi (B,) problem of each slot, s (B,) its scale): the problems in seeded rounds of a permutation each, no round
    starting with the last round's final problem (so neighbouring slots differ when U > 1), and the scales likewise
    in rounds of SCALES."""
    rng = np.random.RandomState(seed)

    def rounds(n, k):
        out = []
        while len(out) < n:
            r = list(rng.permutation(k))
            if out and k > 1 and r[0] == out[-1]:
                r[0], r[-1] = r[-1], r[0]
            out += r
        return np.array(out[:n])
    pi = rounds(B, U)
    s = np.array(SCALES)[rounds(B, len(SCALES))]
    return pi, s


def table(tag, B, U):
    """The slot table of the batch `tag` (a stable name: the CPU tests rebuild the GPU tests' tables)."""
    return slot_table(B, U, TABLE_SEED + zlib.crc32(tag.encode()) % 100000)


def _log_unary(probs):
    """(M, H, W) probabilities -> (H, W, M) float32 log-probabilities, the values CRF() takes."""
    return np.log(np.maximum(np.transpose(probs, (1, 2, 0)), 1e-5)).astype(np.float32)


def train41_problems(U):
    """(images (U, 41, 41, 3) uint8, unaries (U, 41, 41, M), G (U, 41, 41, M)): bench.py's train41 problems, the
    log of their probabilities as unaries."""
    d = helpers.bench_unique("train41", "smooth")
    unary = np.stack([_log_unary(p) for p in d["probs"][:U]])
    return np.ascontiguousarray(d["image"][:U]), unary, _upstreams(unary, 41)


def photo_problems(H, W, U):
    """U seeded synth photos with log_unary unaries.  Every overflowing bilateral tile of synth's photos qualifies as
    hybrid, so the last photo carries a patch of noise in its top-left corner: the few tiles under it overflow
    without a hybrid cover and take the direct path."""
    images = synth.make_batch(U, H, W, image="photo", start=PHOTO_START)["image"].copy()
    images[-1, :NOISE_PATCH[0], :NOISE_PATCH[1]] = synth.make_image(np.random.RandomState(3), *NOISE_PATCH, "noise")
    unary = helpers.log_unary(U, H, W, M, seed=H + W, scale=1.0)
    return np.ascontiguousarray(images), unary, _upstreams(unary, H)


def gate2_problems(Mg):
    """test_gpu_scale.py's two gate-2 noise images, with unaries and G for Mg labels."""
    H, W = helpers.GATE2_SHAPE
    images = helpers.seeded_images(H, W, ("noise", "noise"), helpers.GATE2_SEED)
    unary = helpers.log_unary(2, H, W, Mg, seed=8000 + Mg, scale=1.0)
    return images, unary, _upstreams(unary, Mg)


def switch_problems(name):
    """test_gpu_scale.py's images of a helpers.SWITCH_CASES entry, with unaries and G."""
    H, W, kinds, _ = switch_case(name)
    images = helpers.seeded_images(H, W, kinds, helpers.GATE2_SEED)
    unary = helpers.log_unary(len(kinds), H, W, M, seed=8100 + H + W, scale=1.0)
    return images, unary, _upstreams(unary, H + W)


def _upstreams(unary, seed):
    U, H, W, Mu = unary.shape
    return np.stack([upstream(H, W, Mu, seed + u) for u in range(U)])


def switch_case(name):
    """(H, W, kinds, branch) of a helpers.SWITCH_CASES entry."""
    return next(c[1:] for c in helpers.SWITCH_CASES if c[0] == name)


# ---- truths ----
_TRUTHS = {}


def _truth(kind, image, unary, G, p, mus):
    if kind == "potts":
        return GradTruth(meanfield64.Problem(image, p), unary, G, int(p.n_iters))
    if kind == "mu":
        return CompatTruth(meanfield64.Problem(image, p), unary, G, int(p.n_iters), mus)
    return KgradTruth(image, p, unary, G, mus)


def mus_for(Mg=M):
    return compat_mats(MU_KIND, Mg, 7)


def problem_truths(tag, kinds, images, unary, G, sf, T):
    """{kind: [truth of each problem]} for the U problems (images, unary, G) at crf_params(sf) with T iterations.
    Kinds: "potts" (GradTruth), "mu" (CompatTruth with mus_for()), "theta" and "theta_mu" (KgradTruth with Potts
    weights and with mus_for()).  `tag` names the problems; what is missing is computed together on threads."""
    p = grad_params(sf, T)
    reqs = [((tag, kind, T, u), kind, u) for kind in kinds for u in range(len(images))]
    todo = [r for r in reqs if r[0] not in _TRUTHS]
    if todo:
        mus = mus_for(unary.shape[-1])
        with ThreadPoolExecutor(max(1, min(len(todo), os.cpu_count() or 1))) as ex:
            jobs = [(kind, images[u], unary[u], G[u], p, mus if kind in ("mu", "theta_mu") else None)
                    for _, kind, u in todo]
            for r, t in zip(todo, ex.map(lambda j: _truth(*j), jobs)):
                _TRUTHS[r[0]] = t
    return {kind: [_TRUTHS[(tag, kind, T, u)] for u in range(len(images))] for kind in kinds}


# ---- per-slot checks: the truth times s, the bar times |s| ----
def _close(what, got, want, bar, s):
    got = np.asarray(got, np.float64)
    assert np.all(np.isfinite(got)), "%s: not finite" % what
    err = np.abs(got - s * np.asarray(want, np.float64))
    lim = abs(s) * np.asarray(bar, np.float64)
    i = np.unravel_index(int(np.argmax(err - lim)), err.shape) if err.ndim else ()
    assert np.all(err <= lim), "%s off by %.3g > bar %.3g at %s (got %.9g, want %.9g)" % (
        what, err[i], lim[i] if np.ndim(lim) else lim, i, got[i], s * np.asarray(want)[i])


def check_potts(truth, s, gU, gw, what):
    """GradTruth: dL/dU (H, W, M) and, unless None, the Potts pair (2,)."""
    _close(what + " dL/dunary", gU, truth.gU, truth.bar_u, s)
    if gw is not None:
        for i, n in ((0, "w1"), (1, "w2")):
            _close(what + " dL/d" + n, gw[i], truth.gw[i], truth.bar_w[i], s)


def check_mu(truth, s, gU, gmu, what):
    """CompatTruth: dL/dU and dL/dmu (2, M, M)."""
    _close(what + " dL/dunary", gU, truth.gU, truth.bar_u, s)
    _close(what + " dL/dmu", gmu, truth.gmu, truth.bar_mu, s)


def check_theta(truth, s, gt, what):
    """KgradTruth: dL/dtheta (7,)."""
    _close(what + " dL/dtheta", gt, truth.want, truth.bar, s)


def over_potts(truth, s, gU, gw):
    """The largest error over its bar (> 1: outside) of a slot's dL/dU and Potts pair: the check's margin."""
    r = [float(np.abs(np.asarray(gU, np.float64) - s * truth.gU).max()) / (abs(s) * truth.bar_u)]
    return max(r + [abs(float(gw[i]) - s * truth.gw[i]) / (abs(s) * truth.bar_w[i]) for i in (0, 1)])


# ---- which paths each case takes (from the oracle's lattices) ----
def batch_branch(images, pi, sf):
    """helpers.blur_branch of the batch images[pi] (the bilateral lattice of each distinct image built once)."""
    H, W = images.shape[1:3]
    vb = [helpers.bilateral_vertices(images[u], sf) for u in range(images.shape[0])]
    return helpers.blur_branch(H, W, [vb[int(u)] for u in pi])

