"""The case table of test_gpu_scale.py reaches what it claims to (no GPU needed): the restated workloads are
bench.py's, every case takes the bilateral blur branch the GPU test asserts (from the oracle's own lattices and
meanfield.cu's threshold), and gate 2 meets every fused instantiation MP = 4..32."""
import ast
import os

import pytest

import helpers
from helpers import (BENCH_CF, BENCH_M, BENCH_T_ITERS, BENCH_TH, BENCH_UNIQUE, BENCH_WORKLOADS, GATE2_M, GATE2_SEED,
                     GATE2_SHAPE, MAX_FUSED, SCALE_CASES, SWITCH_CASES, WIDE_BIG_SHAPE, bench_sf, bench_unique,
                     bilateral_vertices, blur_branch, padded, seeded_images, tail1)

BENCH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "bench.py")


@pytest.fixture(scope="module")
def bench_ast():
    return ast.parse(open(BENCH).read())


def _assigned(tree, name):
    for node in tree.body:
        if isinstance(node, ast.Assign):
            for t in node.targets:
                if isinstance(t, ast.Name) and t.id == name:
                    return ast.literal_eval(node.value)
                if isinstance(t, ast.Tuple) and name in [e.id for e in t.elts]:
                    return ast.literal_eval(node.value)[[e.id for e in t.elts].index(name)]
    raise KeyError(name)


def _function(tree, name):
    return next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == name)


def test_workload_table_is_bench_py(bench_ast):
    workloads = _assigned(bench_ast, "WORKLOADS")
    for k, v in BENCH_WORKLOADS.items():
        assert workloads[k] == v, k
    assert _assigned(bench_ast, "M") == BENCH_M
    assert _assigned(bench_ast, "T_ITERS") == BENCH_T_ITERS
    assert (_assigned(bench_ast, "TH1"), _assigned(bench_ast, "TH2")) == BENCH_TH
    # synth_batch(H, W, B, unique=8): synth.make_batch(B, H, W, cues="cam", image=IMAGE_VARIANT, unique=unique)
    f = _function(bench_ast, "synth_batch")
    assert [a.arg for a in f.args.args] == ["H", "W", "B", "unique"]
    assert ast.literal_eval(f.args.defaults[0]) == BENCH_UNIQUE
    call = next(n for n in ast.walk(f) if isinstance(n, ast.Call) and getattr(n.func, "attr", "") == "make_batch")
    assert [a.id for a in call.args] == ["B", "H", "W"]
    kw = {k.arg: k.value for k in call.keywords}
    assert ast.literal_eval(kw["cues"]) == "cam" and kw["image"].id == "IMAGE_VARIANT" and kw["unique"].id == "unique"
    # run_b200 calls synth_batch(H, W, B) and api.crf_params(12.0 if args.workload == "train41" else 1.0, 13, T_ITERS)
    run = _function(bench_ast, "run_b200")
    sb = [n for n in ast.walk(run) if isinstance(n, ast.Call) and getattr(n.func, "id", "") == "synth_batch"]
    assert len(sb) == 1 and [a.id for a in sb[0].args] == ["H", "W", "B"] and not sb[0].keywords
    cp = [n for n in ast.walk(run) if isinstance(n, ast.Call) and getattr(n.func, "attr", "") == "crf_params"]
    assert len(cp) == 1
    sf, cf, it = cp[0].args
    assert isinstance(sf, ast.IfExp) and ast.literal_eval(sf.test.comparators[0]) == "train41"
    assert (ast.literal_eval(sf.body), ast.literal_eval(sf.orelse)) == (bench_sf("train41"), bench_sf("dsrg321"))
    assert ast.literal_eval(cf) == BENCH_CF and it.id == "T_ITERS"
    # the image variants the benchmark measures
    images = next(n for n in ast.walk(bench_ast) if isinstance(n, ast.Call) and n.args and
                  isinstance(n.args[0], ast.Constant) and n.args[0].value == "--images")
    choices = ast.literal_eval(next(k.value for k in images.keywords if k.arg == "choices"))
    assert {v for w, v, _ in SCALE_CASES if w == "dsrg321"} == set(choices)
    assert {w for w, _, _ in SCALE_CASES} == set(BENCH_WORKLOADS)


def test_blur_branch_rule():
    rows = helpers.blur_cached_rows()
    assert rows == 65536
    # capv = (N + P) * 6: 104 x 105 = 10920 pixels fit 65536 rows, 105 x 105 (+ 3 phantom lanes) do not
    assert blur_branch(104, 105, [10 ** 6]) == "ungated"
    assert blur_branch(105, 105, [0]) == "gate1"
    assert blur_branch(321, 321, [rows - 1, rows - 1]) == "gate1"      # rows per image = V + 1
    assert blur_branch(321, 321, [rows, rows - 1]) == "gate2"


@pytest.mark.parametrize("workload,variant,branch", SCALE_CASES)
def test_bench_cases_take_their_branch(workload, variant, branch):
    H, W, B, _ = BENCH_WORKLOADS[workload]
    uniq = bench_unique(workload, variant)["image"]
    vb = [bilateral_vertices(im, bench_sf(workload)) for im in uniq]
    assert blur_branch(H, W, [vb[i % len(vb)] for i in range(B)]) == branch, vb


def test_gate2_cases_cover_every_instantiation():
    image = seeded_images(*GATE2_SHAPE, ("noise", "noise"), GATE2_SEED)
    assert blur_branch(*GATE2_SHAPE, [bilateral_vertices(im) for im in image]) == "gate2"
    assert {padded(M) for M in GATE2_M} == set(range(4, MAX_FUSED + 1, 4))
    assert {tail1(M) for M in GATE2_M} == {True, False}


@pytest.mark.parametrize("name,H,W,kinds,branch", SWITCH_CASES, ids=[c[0] for c in SWITCH_CASES])
def test_switch_cases_take_their_branch(name, H, W, kinds, branch):
    image = seeded_images(H, W, kinds, GATE2_SEED)
    assert blur_branch(H, W, [bilateral_vertices(im) for im in image]) == branch


def test_switch_cases_cover_both_sides():
    assert {c[-1] for c in SWITCH_CASES} == {"ungated", "gate1", "gate2"}
    branch = {(H, W): b for _, H, W, _, b in SWITCH_CASES}
    assert branch[(104, 105)] == "ungated" and branch[(105, 105)] == "gate1"   # one pixel row apart
    N = WIDE_BIG_SHAPE[0] * WIDE_BIG_SHAPE[1]
    assert (N + (4 - N % 4) % 4) * 6 > helpers.blur_cached_rows()             # the 255-label case's lattice
