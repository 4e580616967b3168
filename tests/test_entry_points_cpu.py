"""CPU tests of the engine entry points' first check: every function of include/dsrg_b200.h that takes the engine
as its first parameter refuses a NULL engine before it touches CUDA, so no GPU is needed."""
import os
import re

import pytest

from conftest import ROOT
from dsrg_b200 import _lib


def engine_functions():
    """Names of the header's functions whose first parameter is `dsrg_engine *` or `const dsrg_engine *`."""
    src = open(os.path.join(ROOT, "include", "dsrg_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dsrg_[a-z0-9_]+)\s*\(\s*(?:const\s+)?dsrg_engine\s*\*", src)))


def test_header_has_engine_entry_points():
    names = engine_functions()
    assert len(names) >= 50
    for n in ("dsrg_engine_destroy", "dsrg_engine_get_size", "dsrg_crf_batch_dev", "dsrg_predict_mask_host"):
        assert n in names


def _zero_args(argtypes):
    return [0.0 if t in (_lib.C.c_float, _lib.C.c_double) else (None if t in (_lib._vp, _lib._pp) else 0)
            for t in argtypes]


# the non-int getters answer a NULL engine with a sentinel and leave no message
SENTINELS = {"dsrg_engine_device_bytes": 0, "dsrg_engine_graph_replays": 0, "dsrg_engine_take_launch_count": 0,
             "dsrg_engine_hybrid_tiles": -1}


@pytest.mark.parametrize("name", engine_functions())
def test_null_engine_is_refused(name):
    L = _lib.lib()
    res, args = _lib.SIGNATURES[name]
    # leave a different message behind first, so that the call must set its own
    assert L.dsrg_densecrf_create(0, 0, 0) is None
    rc = getattr(L, name)(*_zero_args(args))
    if res is None:   # dsrg_engine_destroy: a no-op
        return
    if name in SENTINELS:
        assert rc == SENTINELS[name]
        return
    assert rc == _lib.E_INVALID
    assert L.dsrg_last_error().decode() == "engine is NULL"
