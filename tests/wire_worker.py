"""Worker of tests/test_gpu_wire.py: one WIRE_CASES case through the host-buffer entry points (dsrg_forward_host,
srg_host) in one wire mode.  The mode is the process's environment (the host thread count is read once per process,
DSRG_B200_WIRE when an engine is created), so every (case, mode) pair runs in a process of its own.

Before every host-buffer call the worker writes helpers.wire_call_marker to stderr; the library's
DSRG_B200_DEBUG_TIMING lines follow it, and the parent checks them against helpers.host_schedule.  Every check runs
here; a failure exits nonzero with its message.  On success the worker prints "WIRE-OK ..." and writes the SHA-256
digests of its SRG-only outputs to argv[3] (JSON), which the parent compares across the modes.

Per full-pass call:
  * the probs buffer equals numpy's float32 p[p < 1e-4] = 1e-4 bit for bit;
  * seeds equal srg_closed_form(labels, cues, renorm64(crf_out)) bit for bit on this call's own marginals (every
    image; for "bench" a sample plus the edge images, and the whole batch against srg_dev(renorm=True) run on the
    device over crf_out);
  * crf_out within 1e-4 of crf_oracle.CRF (same images) and of dsrg_forward_dev on the same inputs (all images);
  * a call without crf_out differs from the call with it in at most 1e-3 of the seed values (float atomics);
  * a profiled call (graphs off) counts one wire_bits launch per chunk where the clamp travels as a mask.
SRG-only calls (renorm off and on, label map out): seeds and label maps bit-exact against the oracle."""
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import helpers  # noqa: E402
from oracle import crf_oracle, srg_oracle  # noqa: E402
from helpers import (BENCH_CF, BENCH_T_ITERS, BENCH_TH, WIRE_CASES, WIRE_EDGE_IMAGES, WIRE_MODES,  # noqa: E402
                     WIRE_NONBINARY, WIRE_SF, host_schedule, renorm64, sample_indices, wire_call_marker, wire_inputs)

TOL = 1e-4
MIN_PROB = np.float32(1e-4)


def log(msg):
    sys.stderr.write(msg + "\n")
    sys.stderr.flush()


def first_diff(got, want):
    bad = np.argwhere(got != want)
    i = tuple(bad[0])
    return "%d values differ, first at %s: got %r want %r" % (len(bad), i, float(got[i]), float(want[i]))


def clamped(p):
    c = p.copy()
    c[c < MIN_PROB] = MIN_PROB
    return c


class Step(object):
    def __init__(self, case, k, eng, pinned):
        self.case, self.k, self.eng, self.pinned = case, k, eng, pinned
        (self.maxB, _, _, self.M), (self.H, self.W), self.B, self.chunk, self.schedule = WIRE_CASES[case][k]
        self.d = wire_inputs(case, k)
        self.params = self.crf_params()
        self.sizes = host_schedule(self.B, self.maxB, self.chunk, self.schedule)

    def crf_params(self):
        from dsrg_b200 import api
        return api.crf_params(WIRE_SF[self.case], BENCH_CF, BENCH_T_ITERS)

    def buf(self, a=None, shape=None):
        from dsrg_b200 import api
        shape = a.shape if a is not None else shape
        out = api.pinned_empty(shape, np.float32) if self.pinned else np.empty(shape, np.float32)
        if a is not None:
            out[...] = a
        return out

    def host_call(self, fn, *args, **kw):
        if self.schedule is None:
            os.environ.pop("DSRG_B200_HOST_SCHEDULE", None)
        else:
            os.environ["DSRG_B200_HOST_SCHEDULE"] = self.schedule
        log(wire_call_marker(self.B, self.maxB, self.chunk, self.schedule))
        return fn(*args, **kw)

    def tag(self, what):
        return "%s step %d (%s, %s): %s" % (self.case, self.k, "pinned" if self.pinned else "pageable",
                                            os.environ.get("WIRE_MODE"), what)


def check_seeds(st, seeds, q, images):
    """seeds of `images` == the SRG oracle on the float64 renormalisation of this call's own marginals."""
    d = st.d
    for b in images:
        want = srg_oracle.srg_closed_form(d["labels"][b], d["cues"][b], renorm64(q[b]), *BENCH_TH)
        assert np.array_equal(seeds[b], want), st.tag("seeds of image %d: %s" % (b, first_diff(seeds[b], want)))


def check_marginals(st, q, images, oracle_cache):
    d = st.d
    probs_c = clamped(d["probs"])
    for b in images:
        key = helpers.digest(probs_c[b], d["image"][b])
        if key not in oracle_cache:
            oracle_cache[key] = crf_oracle.CRF(d["image"][b], np.ascontiguousarray(np.transpose(probs_c[b], (1, 2, 0))),
                                               BENCH_T_ITERS, WIRE_SF[st.case], BENCH_CF)
        err = float(np.abs(np.transpose(q[b], (1, 2, 0)) - oracle_cache[key]).max())
        assert err <= TOL, st.tag("marginals of image %d off the oracle by %g" % (b, err))


def full_pass(st, torch, oracle_cache, calls=1):
    """Host-buffer full pass(es) with crf_out and every check on the last one's outputs."""
    eng, d, B = st.eng, st.d, st.B
    want_probs = clamped(d["probs"])
    labels, cues, image = st.buf(d["labels"]), st.buf(d["cues"]), d["image"]
    if st.pinned:
        from dsrg_b200 import api
        image = api.pinned_empty(d["image"].shape, np.uint8)
        image[...] = d["image"]
    probs = st.buf(d["probs"])
    seeds, q = st.buf(shape=d["probs"].shape), st.buf(shape=d["probs"].shape)
    if st.pinned:   # page-aligned: image b's seeds start at byte b * M * N * 4 mod 16 of a 16-byte boundary
        assert seeds.ctypes.data % 16 == 0
    for _ in range(calls):   # bench.py re-sends the same (now clamped) probs buffer
        seeds.fill(np.nan)
        q.fill(np.nan)
        st.host_call(eng.dsrg_forward_host, labels, probs, cues, image, st.params, *BENCH_TH, seeds_out=seeds,
                     crf_out=q)
        assert np.array_equal(probs.view(np.uint32), want_probs.view(np.uint32)), \
            st.tag("in-place clamp: " + first_diff(probs, want_probs))
    if st.case == "bench":
        images = sorted(set(sample_indices(B, seed=B + st.H)) | set(WIRE_EDGE_IMAGES))
        # the whole batch: SRG on the device over this call's own marginals
        d_q = torch.from_numpy(q).cuda()
        d_s = torch.empty_like(d_q)
        eng.srg_dev(torch.from_numpy(d["labels"]).cuda(), d_q, torch.from_numpy(d["cues"]).cuda(), *BENCH_TH, d_s,
                    renorm=True)
        torch.cuda.synchronize()
        n = int((d_s != torch.from_numpy(seeds).cuda()).sum())
        assert n == 0, st.tag("seeds differ from srg_dev(renorm) on crf_out in %d values" % n)
        del d_q, d_s
    else:
        images = range(B)
    check_seeds(st, seeds, q, images)
    check_marginals(st, q, images, oracle_cache)
    # the device entry point on the same inputs
    dev = {k: torch.from_numpy(np.ascontiguousarray(d[k])).cuda() for k in ("labels", "probs", "cues", "image")}
    d_seeds, d_q = torch.empty_like(dev["probs"]), torch.empty_like(dev["probs"])
    eng.dsrg_forward_dev(dev["labels"], dev["probs"], dev["cues"], dev["image"], st.params, *BENCH_TH, d_seeds,
                         crf_out=d_q)
    torch.cuda.synchronize()
    err = float((d_q - torch.from_numpy(q).cuda()).abs().max())
    assert err <= TOL, st.tag("crf_out off dsrg_forward_dev's by %g" % err)
    del dev, d_seeds, d_q
    return labels, cues, image, seeds


def no_crf_out_and_profiled(st, labels, cues, image, seeds, mode):
    eng, d = st.eng, st.d
    probs = st.buf(d["probs"])
    s2 = st.host_call(eng.dsrg_forward_host, labels, probs, cues, image, st.params, *BENCH_TH,
                      seeds_out=st.buf(shape=d["probs"].shape))
    n = int((s2 != seeds).sum())
    assert n <= 1e-3 * seeds.size, st.tag("seeds without crf_out differ in %d of %d values" % (n, seeds.size))
    eng.profile(True)
    eng.profile_read()
    probs[...] = d["probs"]
    st.host_call(eng.dsrg_forward_host, labels, probs, cues, image, st.params, *BENCH_TH,
                 seeds_out=st.buf(shape=d["probs"].shape))
    prof = eng.profile_read()
    eng.profile(False)
    want = 0 if mode == "raw" else len(st.sizes)
    got = prof.get("wire_bits", (0.0, 0))[1]
    assert got == want, st.tag("wire_bits launches %d, expected %d" % (got, want))


def srg_only(st, digests):
    eng, d = st.eng, st.d
    labels, probs, cues = st.buf(d["labels"]), st.buf(d["probs"]), st.buf(d["cues"])
    images = sorted(set(sample_indices(st.B, seed=st.B)) | set(WIRE_EDGE_IMAGES)) if st.case == "bench" \
        else range(st.B)
    for renorm in (False, True):
        seeds = st.buf(shape=d["probs"].shape)
        lmap = np.full((st.B, st.H, st.W), -7, np.int32)
        st.host_call(eng.srg_host, labels, probs, cues, *BENCH_TH, renorm=renorm, seeds_out=seeds, label_map_out=lmap)
        assert np.array_equal(probs, d["probs"]), st.tag("srg_host wrote to its probs")
        p = renorm64(d["probs"][list(images)]) if renorm else d["probs"][list(images)]
        for i, b in enumerate(images):
            want, wlm = srg_oracle.srg_closed_form(d["labels"][b], d["cues"][b], p[i], *BENCH_TH,
                                                           return_label_map=True)
            assert np.array_equal(lmap[b], wlm), st.tag("srg_host(renorm=%d) label map of image %d: %s"
                                                        % (renorm, b, first_diff(lmap[b], wlm)))
            assert np.array_equal(seeds[b], want), st.tag("srg_host(renorm=%d) seeds of image %d: %s"
                                                          % (renorm, b, first_diff(seeds[b], want)))
        digests["step%d_%s_renorm%d" % (st.k, "pinned" if st.pinned else "pageable", renorm)] = helpers.digest(seeds, lmap)


def check_case_inputs(st):
    """What the case claims about its inputs: non-binary cues in one chunk only, on classes the image lacks."""
    nonbin = [b for b in range(st.B) if not np.isin(st.d["cues"][b], (0.0, 1.0)).all()]
    want = sorted({b for b, _ in WIRE_NONBINARY.get(st.case, [])})
    assert nonbin == want, (nonbin, want)


def main():
    case, mode, out_json = sys.argv[1], sys.argv[2], sys.argv[3]
    assert os.environ.get("DSRG_B200_DEBUG_TIMING") and os.environ.get("WIRE_MODE") == mode
    for k, v in WIRE_MODES[mode][0].items():
        assert os.environ.get(k) == v, (k, os.environ.get(k))
    import torch
    from dsrg_b200 import api
    t0 = time.time()
    digests, oracle_cache = {}, {}
    eng, eng_key = None, None
    for k, step in enumerate(WIRE_CASES[case]):
        if step[0] != eng_key:
            if eng is not None:
                eng.close()
            eng, eng_key = api.Engine(*step[0]), step[0]
        eng.set_size(*step[1])
        eng.set_host_chunk(step[3])
        for pinned in ((True, False) if case == "mixed_cues" else (True,)):
            st = Step(case, k, eng, pinned)
            check_case_inputs(st)
            calls = 2 if case == "bench" else 1
            before = eng.graph_replays
            labels, cues, image, seeds = full_pass(st, torch, oracle_cache, calls)
            if case == "bench":
                assert eng.graph_replays > before, st.tag("the second call replayed no graph")
            no_crf_out_and_profiled(st, labels, cues, image, seeds, mode)
            srg_only(st, digests)
        log("[wire worker] %s step %d done at %.1f s" % (case, k, time.time() - t0))
    eng.close()
    with open(out_json, "w") as f:
        json.dump(digests, f)
    print("WIRE-OK case=%s mode=%s steps=%d %.1f s" % (case, mode, len(WIRE_CASES[case]), time.time() - t0),
          flush=True)


if __name__ == "__main__":
    main()
