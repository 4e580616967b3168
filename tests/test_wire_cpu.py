"""The host-buffer pipeline's chunk schedule restated (helpers.host_schedule, wire.cu:host_pass_impl) and the claims
of test_gpu_wire.py's case table, without a GPU."""
import numpy as np
import pytest

from helpers import (WIRE_CASES, WIRE_EDGE_IMAGES, WIRE_EDGE_PROBS, WIRE_MODES, WIRE_NONBINARY, chunk_of,
                     host_schedule, parse_wire_log, wire_call_marker, wire_inputs)


@pytest.mark.parametrize("B,maxB,chunk,schedule,want", [
    (64, 64, 0, None, [5, 9, 13, 17, 20]),        # bench.py's batch
    (5, 8, 0, None, [1, 1, 1, 2]),
    (12, 12, 0, "3,4,5", [3, 4, 5]),
    (6, 6, 2, None, [1, 2, 1, 2]),                # host_chunk caps every chunk
    (8, 8, 0, None, [1, 1, 1, 3, 2]),
    (1, 1, 0, None, [1]),
    (64, 64, 8, None, [5, 8, 1, 8, 5, 8, 8, 1, 8, 8, 4]),
    (4, 4, 0, "1,1,2", [1, 1, 2]),
    (12, 8, 0, "4,40", [4, 8]),                   # an entry is cut to maxB and to what is left
    (12, 12, 0, "2", [2, 10]),                    # the rest of the batch is one chunk ...
    (12, 12, 3, "2", [2, 3, 3, 3, 1]),            # ... or chunks of host_chunk
    (12, 12, 0, "2,0,5", [2, 10]),                # parsing stops at an entry below 1
    (12, 12, 0, "2,x,5", [2, 10]),
    (12, 12, 0, "3,4,", [3, 4, 5]),
    (12, 12, 0, "", [12]),
    (12, 12, 0, "5,5,5,5", [5, 5, 2]),
])
def test_host_schedule(B, maxB, chunk, schedule, want):
    got = host_schedule(B, maxB, chunk, schedule)
    assert got == want
    assert sum(got) == B and all(1 <= n <= maxB for n in got)


def test_default_schedule_covers_every_batch():
    for B in range(1, 129):
        for chunk in (0, 1, 3, 16):
            s = host_schedule(B, B, chunk)
            assert sum(s) == B and min(s) >= 1
            assert max(s) <= (chunk or B)
            assert len(s) <= 5 or chunk


def test_modes_differ_in_what_crosses_pcie():
    assert WIRE_MODES["bits"][1] >= 6 > WIRE_MODES["floats"][1]       # wire.cu: wire_worthwhile()
    assert WIRE_MODES["raw"][0].get("DSRG_B200_WIRE") == "0" and WIRE_MODES["raw"][1] >= 6
    assert all("DSRG_B200_WIRE" not in env for m, (env, _) in WIRE_MODES.items() if m != "raw")


def _sizes(case, step=0):
    (maxB, _, _, _), _, B, chunk, schedule = WIRE_CASES[case][step]
    return host_schedule(B, maxB, chunk, schedule)


def test_bench_case_is_bench_py_batch():
    (maxB, H, W, M), size, B, chunk, schedule = WIRE_CASES["bench"][0]
    assert (maxB, H, W, M, B) == (64, 321, 321, 21, 64) and size == (H, W) and not chunk and schedule is None
    sizes = _sizes("bench")
    assert sizes == [5, 9, 13, 17, 20]
    a, b, last = WIRE_EDGE_IMAGES
    assert chunk_of(sizes, a) == 0 and chunk_of(sizes, a + 1) == 1 and a + 1 == b and last == B - 1
    assert (M * H * W) % 32 != 0
    # image b's seeds_out starts b * M * N floats into a page-aligned buffer: every 16-byte phase occurs, so the host
    # unpack peels 0, 1, 2 and 3 floats before its aligned stores
    assert {(b * M * H * W * 4) % 16 for b in range(B)} == {0, 4, 8, 12}


def test_edge_probs():
    v = WIRE_EDGE_PROBS
    lo = np.float32(1e-4)
    assert v[0] == lo and v[1] == np.nextafter(lo, np.float32(0)) and v[1] < lo
    assert v[2] == 0 and not np.signbit(v[2]) and v[3] == 0 and np.signbit(v[3]) and v[4] < 0
    assert v[5] == np.finfo(np.float32).smallest_subnormal and v[5] > 0
    c = v.copy()
    c[c < 1e-4] = 1e-4
    assert c[0] == lo and (c[1:] == lo).all()


@pytest.mark.parametrize("case", ["mixed_cues", "wide"])
def test_nonbinary_cues_in_exactly_one_chunk(case):
    sizes = _sizes(case)
    assert len({chunk_of(sizes, b) for b, _ in WIRE_NONBINARY[case]}) == 1
    assert 0 < chunk_of(sizes, WIRE_NONBINARY[case][0][0]) < len(sizes) - 1    # binary chunks on both sides
    d = wire_inputs(case, 0)
    nonbin = {b for b in range(len(d["cues"])) if not np.isin(d["cues"][b], (0.0, 1.0)).all()}
    assert nonbin == {b for b, _ in WIRE_NONBINARY[case]}
    for b, v in WIRE_NONBINARY[case]:
        ys, xs = np.nonzero(d["cues"][b] == v)[1:]
        cls = np.nonzero((d["cues"][b] == v).any((1, 2)))[0]
        assert len(cls) == 1 and len(ys) == 1 and d["labels"][b, cls[0]] == 0   # a class the image lacks
    assert {v for _, v in WIRE_NONBINARY[case]} == {0.5, 2.0, -1.0}


def test_mixed_case_mixes_both_decisions():
    sizes = _sizes("mixed_cues")
    assert sizes == [3, 4, 5]
    assert {chunk_of(sizes, b) for b, _ in WIRE_NONBINARY["mixed_cues"]} == {1}     # chunks 0 and 2 stay binary


def test_wide_case_runs_the_generic_kernels():
    (maxB, H, W, M), _, B, chunk, _ = WIRE_CASES["wide"][0]
    assert M == 81 and M != 21 and _sizes("wide") == [1, 2, 1, 2]      # srg.cu instantiates MT = 21 and MT = 0


@pytest.mark.parametrize("case,step", [("bench", 0), ("mixed_cues", 0), ("wide", 0), ("reshaped", 2), ("reshaped", 3)])
def test_ragged_cases(case, step):
    (_, _, _, M), (H, W), _, _, _ = WIRE_CASES[case][step]
    assert (M * H * W) % 32 != 0
    want = {"mixed_cues": 20, "wide": 17}.get(case)
    assert want is None or (M * H * W) % 32 == want


def test_reshaped_case():
    steps = WIRE_CASES["reshaped"]
    (cap, size, B, _, _), (cap1, size1, B1, _, _) = steps[:2]
    assert cap == cap1 == (8, 64, 80, 21) and size == (41, 41) and B < cap[0] and size1 == cap[1:3] and B1 == cap[0]
    wpi = lambda H, W, M: -(-(M * H * W) // 32)   # noqa: E731
    assert wpi(41, 41, 21) < wpi(64, 80, 21)
    assert [s[1] for s in steps[2:]] == [(1, 1), (2, 3)]
    for s in steps[2:]:
        (_, _, _, M), (H, W) = s[0], s[1]
        assert wpi(H, W, M) * 32 - M * H * W > 0       # one ragged word per plane
        assert host_schedule(s[2], s[0][0], s[3], s[4]) == [1, 1, 2]
    for k in range(len(steps)):
        d = wire_inputs("reshaped", k)
        assert np.isin(d["cues"], (0.0, 1.0)).all() and np.isfinite(d["probs"]).all()
        assert d["image"].dtype == np.uint8 and d["image"].shape[1:3] == steps[k][1]


def test_parse_wire_log():
    text = "\n".join([
        "some other line",
        wire_call_marker(12, 12, 0, "3,4,5"),
        "[dsrg host pass] timeline (ms from the first H2D; chunk: h2d begin-end | kernels begin-end | d2h end):"
        "  [3 img: 0.00-0.31 | 0.32-1.90 | 2.10]  [4 img: 0.31-0.70 | 1.90-3.80 | 4.00]  [5 img: 0.70-1.20 | "
        "3.80-6.10 | 6.40]",
        "[dsrg host pass] total 7.02 ms: pack 0.40 issue 0.20 unpack 0.30 wait 5.10 (threads 8, chunks 3)",
        wire_call_marker(5, 8, 2, None),
        "[dsrg host pass] timeline (ms from the first H2D; chunk: h2d begin-end | kernels begin-end | d2h end):"
        "  [1 img: 0.00-0.10 | 0.10-0.50 | 0.60]",
        "[dsrg host pass] total 1.00 ms: pack 0.00 issue 0.10 unpack 0.00 wait 0.80 (threads 1, chunks 1)",
    ])
    calls = parse_wire_log(text)
    assert calls == [
        {"B": 12, "maxB": 12, "chunk": 0, "schedule": "3,4,5", "sizes": [3, 4, 5], "threads": 8, "chunks": 3},
        {"B": 5, "maxB": 8, "chunk": 2, "schedule": None, "sizes": [1], "threads": 1, "chunks": 1}]
    # a call the library did not log stays incomplete
    assert parse_wire_log(wire_call_marker(4, 4, 0, "1,1,2"))[0]["threads"] is None


def test_restatement_matches_wire_cu():
    """The edges, the debug lines the parser reads and the schedule variable are wire.cu's."""
    import os
    import re
    src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "dsrg_b200", "csrc", "wire.cu")).read()
    edges = re.search(r"const double edge\[5\] = \{([^}]*)\};", src).group(1)
    assert [eval(e) for e in edges.split(",")] == [5 / 64, 14 / 64, 27 / 64, 44 / 64, 1.0]
    assert '"  [%d img: ' in src and "(threads %d, chunks %d)\\n" in src and "[dsrg host pass] timeline" in src
    assert 'getenv("DSRG_B200_HOST_SCHEDULE")' in src and "static bool wire_worthwhile() { return host_threads() >= 6; }" in src
