"""The claims of test_gpu_crf_grad_scale.py, checked without a GPU: every case takes the blur branch and the tile
paths it is there for; the slot tables put each problem in several slots, never the same one twice in a row, with
negative and non-unit scales, and a slot given its neighbour's result falls outside its bar; the float32 models'
backward is exactly linear in G at every scale; and every mutant of the three backward restatements falls outside the
bars at 321^2 and on a gate-2 image."""
import numpy as np
import pytest

import helpers
from crf_compat_cases import CompatTruth
from crf_grad_cases import GradTruth, grad_params, upstream
from crf_grad_scale_cases import (CASES, GATE2_LABELS, GATE2_T, PARTIAL_RUNS, SCALES, SM_H100, TRAIN_BATCHES,
                                  batch_branch, gate2_problems, mus_for, over_potts, photo_problems,
                                  problem_truths, switch_case, switch_problems, table, train41_problems)
from crf_kgrad_cases import KgradTruth
from oracle import crf_compat_oracle, crf_grad_oracle, meanfield64
from oracle import crf_kgrad_oracle as K


def _case_problems(name):
    H, W, _, _, U = CASES[name][:5]
    return train41_problems(U) if name == "train41" else photo_problems(H, W, U)


@pytest.mark.parametrize("name", sorted(CASES))
def test_cases_take_their_blur_branch(name):
    H, W, B, sf, U, _, _, branch = CASES[name]
    images = _case_problems(name)[0]
    for kind in (["potts_host", "potts_dev", "theta", "mu"] if name == "train41" else ["potts", "theta_mu"]):
        assert batch_branch(images, table("%s-%s" % (name, kind), B, U)[0], sf) == branch, kind


def test_gate2_and_switch_cases_take_their_blur_branch():
    images = gate2_problems(GATE2_LABELS[0])[0]
    for Mg in GATE2_LABELS:
        assert batch_branch(images, table("gate2-%d" % Mg, 2, 2)[0], 1.0) == "gate2"
    seen = set()
    for name in [c[0] for c in helpers.SWITCH_CASES]:
        branch = switch_case(name)[3]
        assert batch_branch(switch_problems(name)[0], table("switch-" + name, 2, 2)[0], 1.0) == branch, name
        seen.add(branch)
    assert seen == {"ungated", "gate1", "gate2"}


def test_dsrg321_tile_paths_and_partial_batches():
    """At 132 SMs the B = 64 batch runs hybrid, direct and shared-memory bilateral tiles after demotion; of the
    partial batches on the same engine B = 1, 3 have hybrid tiles off and 37, 64 on (and kept by k_tile_demote)."""
    H, W, B, sf, U = CASES["dsrg321"][:5]
    images = photo_problems(H, W, U)[0]
    pred = helpers.predict_tile_paths(images[table("dsrg321-potts", B, U)[0]], sf, SM_H100)
    assert pred["hybrid_tiles"] > 0
    assert (pred["bi"] == "direct").any() and (pred["bi"] == "smem").any() and (pred["bi"] == "hybrid").any()
    assert PARTIAL_RUNS[0] == ("theta", 3)            # the theta buffers are first allocated at a small batch
    for i, (kind, Bp) in enumerate(PARTIAL_RUNS):
        on = helpers.hybrid_tiles_on(H, W, Bp, SM_H100)
        nhy = helpers.predict_tile_paths(images[table("partial-%d" % i, Bp, U)[0]], sf, SM_H100)["hybrid_tiles"]
        if Bp in (1, 3):
            assert not on and nhy == 0, Bp
        if Bp in (37, 64):
            assert on and nhy > 0, Bp


def _all_tables():
    out = [("%s-%s" % (n, k), CASES[n][2], CASES[n][4]) for n in CASES
           for k in (["potts_host", "potts_dev", "theta", "mu"] if n == "train41" else ["potts", "theta_mu"])]
    out += [("partial-%d" % i, B, CASES["dsrg321"][4]) for i, (_, B) in enumerate(PARTIAL_RUNS)]
    out += [("train-loop-%d" % i, B, CASES["train41"][4]) for i, B in enumerate(TRAIN_BATCHES)]
    out += [("gate2-%d" % Mg, 2, 2) for Mg in GATE2_LABELS]
    return out


@pytest.mark.parametrize("tag,B,U", _all_tables())
def test_slot_tables(tag, B, U):
    pi, s = table(tag, B, U)
    assert pi.shape == s.shape == (B,)
    assert set(pi) <= set(range(U)) and set(s) <= set(SCALES)
    if U > 1:
        assert (pi[1:] != pi[:-1]).all(), "neighbouring slots hold one problem"
    if B >= 2 * U:
        assert np.bincount(pi, minlength=U).min() >= 2, "a problem fills fewer than two slots"
    if B >= len(SCALES):
        assert (s < 0).any() and (np.abs(s) != 1).any()


def test_neighbouring_slots_fall_outside_each_others_bars():
    """On train41 (every gradient kind): slot b given slot b+1's result, as a mixed-up slot offset would give it, is
    outside slot b's bar."""
    H, W, B, sf, U, T, _, _ = CASES["train41"]
    probs = train41_problems(U)
    tr = problem_truths("train41", ["potts", "theta"], *probs, sf, T)
    tr.update(problem_truths("train41", ["mu"], *probs, sf, T))
    for kind in ("potts_host", "theta", "mu"):
        pi, s = table("train41-" + kind, B, U)
        for b in range(B - 1):
            a, c = pi[b], pi[b + 1]
            if kind == "mu":
                t, n = tr["mu"][a], tr["mu"][c]
                over = max(float(np.abs(s[b + 1] * n.gU - s[b] * t.gU).max()) / (abs(s[b]) * t.bar_u),
                           float((np.abs(s[b + 1] * n.gmu - s[b] * t.gmu) / (abs(s[b]) * t.bar_mu)).max()))
            else:
                t, n = tr["potts"][a], tr["potts"][c]
                over = over_potts(t, s[b], s[b + 1] * n.gU, [s[b + 1] * w for w in n.gw])
                if kind == "theta":
                    tt, nt = tr["theta"][a], tr["theta"][c]
                    over = max(over, float((np.abs(s[b + 1] * nt.want - s[b] * tt.want) / (abs(s[b]) * tt.bar)).max()))
            assert over > 1.0, (kind, b, over)


def test_float32_backward_is_linear_in_the_upstream_gradient():
    """Every float32 model of the three backwards, with s G in place of G, gives s times its result bit for bit, so
    the scaled truths and bars of the slots add no error of their own."""
    H, W, Ms, T = 9, 11, 6, 3
    image = helpers.small_image(np.random.RandomState(5), H, W, "noise")
    unary = helpers.log_unary(1, H, W, Ms, 5, scale=1.0)[0]
    G = upstream(H, W, Ms, 6)
    p = grad_params(1.0, T)
    P = meanfield64.Problem(image, p)
    mus = mus_for(Ms)
    frozen = K.Frozen(meanfield64.Problem(image, p), image, p)
    for m in helpers.BAR_MODELS:
        kw = dict(m)
        es = kw.pop("exp_seed", 0)
        q32 = P.run(unary, T, np.float32, exp_seed=es, **kw)
        qc = crf_compat_oracle.run(P, unary, mus, T, np.float32, exp_seed=es, **kw)

        def run(g):
            gu, gw, _ = crf_grad_oracle.backward(P, q32, g, np.float32, **kw)
            cu, cm, _ = crf_compat_oracle.backward(P, qc, g, mus, np.float32, **kw)
            th = [K.theta_grad(frozen, frozen.theta0, unary, g, T, mu, dtype=np.float32, exp_seed=es, **kw)[0]
                  for mu in (None, mus)]
            return [gu, np.array(gw), cu, cm] + th
        base = run(G)
        for sc in SCALES:
            for i, (a, b) in enumerate(zip(run((np.float32(sc) * G).astype(np.float32)), base)):
                assert np.array_equal(np.asarray(a), (sc * np.asarray(b)).astype(np.asarray(a).dtype)), (m, sc, i)


def _mutant_problems():
    """(name, image, unary, G, sf, T of the Potts case, T of the theta / mu case) of dsrg321's first problem and of
    the first gate-2 image at the fewest labels."""
    H, W, _, sf, U, Tp, Tt, _ = CASES["dsrg321"]
    im, un, G = photo_problems(H, W, U)
    gi, gu, gG = gate2_problems(GATE2_LABELS[0])
    return [("dsrg321", im[0], un[0], G[0], sf, Tp, Tt), ("gate2", gi[0], gu[0], gG[0], 1.0, GATE2_T, GATE2_T)]


@pytest.mark.parametrize("which", [0, 1], ids=["dsrg321", "gate2"])
def test_mutants_outside_the_bars_at_scale(which):
    """transpose_forward_order (the Potts backward), the compatibility backward's three mutants and every kernel
    bandwidth mutant fall outside the bars the GPU tests hold the device to, on one large problem each."""
    from concurrent.futures import ThreadPoolExecutor
    name, image, unary, G, sf, Tp, Tt = _mutant_problems()[which]
    mus = mus_for(unary.shape[-1])
    pp, pt = grad_params(sf, Tp), grad_params(sf, Tt)
    jobs = [lambda: GradTruth(meanfield64.Problem(image, pp), unary, G, Tp, mutant="transpose_forward_order"),
            lambda: CompatTruth(meanfield64.Problem(image, pt), unary, G, Tt, mus,
                                mutants=sorted(crf_compat_oracle.MUTANTS)),
            lambda: KgradTruth(image, pt, unary, G, mus if name == "dsrg321" else None)]
    with ThreadPoolExecutor(len(jobs)) as ex:
        grad, compat, kgrad = list(ex.map(lambda f: f(), jobs))
    mu, mw = grad.mutant
    assert over_potts(grad, 1.0, mu, mw) > 1.0, "transpose_forward_order"
    for m, (u, g) in compat.mutants.items():
        assert max(compat.over(u, g)) > 1.0, m
    for m in sorted(K.MUTANTS):
        assert kgrad.mutant_excess(m) > 1.0, m
