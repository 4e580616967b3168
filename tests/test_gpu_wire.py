"""The host-buffer entry points (dsrg_forward_host, srg_host: csrc/wire.cu) in every wire mode, against the oracles.

Per chunk the pipeline decides what crosses PCIe as 1 bit per value: the cues when they are all exactly 0 or 1 and
the host has enough threads to pack them, the seeds under the same condition, the in-place clamp as a mask on full
passes.  Which of these a run takes depends on the host's thread count, read once per process, so each case of
helpers.WIRE_CASES runs in one subprocess per mode of helpers.WIRE_MODES (tests/wire_worker.py does the checks), one
after the other.  From the worker's stderr this test checks that every host-buffer call ran with the mode's thread
count and with the chunk schedule helpers.host_schedule derives for it, and it compares the SRG-only outputs across
the modes bit for bit.  tests/test_wire_cpu.py checks the schedule and the case table without a GPU."""
import json
import os
import subprocess
import sys
import time

import pytest

from helpers import WIRE_CASES, WIRE_MODES, host_schedule, parse_wire_log

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "wire_worker.py")
TIMEOUT = {"bench": 1500}   # seconds per worker; the others take 600


def run_worker(case, mode, out_json):
    env = {k: v for k, v in os.environ.items()
           if k not in ("DSRG_B200_HOST_THREADS", "DSRG_B200_WIRE", "DSRG_B200_HOST_SCHEDULE", "DSRG_B200_HOST_CHUNK")}
    env.update(WIRE_MODES[mode][0], DSRG_B200_DEBUG_TIMING="1", WIRE_MODE=mode)
    t = time.time()
    r = subprocess.run([sys.executable, WORKER, case, mode, out_json], capture_output=True, text=True, env=env,
                       timeout=TIMEOUT.get(case, 600), cwd=ROOT)
    return r, time.time() - t


def schedule_problems(stderr, threads):
    calls = parse_wire_log(stderr)
    if not calls:
        return ["no host-buffer call was logged"]
    out = []
    for i, c in enumerate(calls):
        want = host_schedule(c["B"], c["maxB"], c["chunk"], c["schedule"])
        got = (c["threads"], c["chunks"], c["sizes"])
        if got != (threads, len(want), want):
            out.append("call %d (%s): (threads, chunks, sizes) %s, expected %s" % (i, c, got, (threads, len(want), want)))
    return out


@pytest.mark.parametrize("case", list(WIRE_CASES))
def test_host_buffer_pipeline_every_wire_mode(torch_cuda, tmp_path, case):
    failures, digests = [], {}
    for mode, (_, threads) in WIRE_MODES.items():
        out_json = str(tmp_path / ("%s.json" % mode))
        r, dt = run_worker(case, mode, out_json)
        print("[wire] %-10s %-6s %6.1f s  exit %d" % (case, mode, dt, r.returncode))
        if r.returncode != 0 or "WIRE-OK case=%s mode=%s" % (case, mode) not in r.stdout:
            failures.append("%s: exit %d\n%s%s" % (mode, r.returncode, r.stdout[-1500:], r.stderr[-3000:]))
            continue
        failures += ["%s: %s" % (mode, p) for p in schedule_problems(r.stderr, threads)]
        with open(out_json) as f:
            digests[mode] = json.load(f)
    assert not failures, "\n\n".join(failures)
    first = digests["bits"]
    for mode, d in digests.items():
        assert d == first, ("SRG-only outputs differ between the bits and %s modes" % mode,
                            sorted(k for k in d if d[k] != first.get(k)))
