"""GPU tests (-m gpu): k_intra's small-TU prediction plans on the engine.  The coverage pictures of intra_plan_cases.py, which
reach every reachable plan class (test_cpu_intra_plans.py proves it from the records and checks the table itself against the
oracle), run through a fresh engine per test against the CPU oracle: at 8, 10 and 12 bit and with 12-bit luma / 9-bit chroma,
after reconstruction and after the loop filters; with 8x8 regions, with the planes of a region merged into one task (plan words
carried from one segment into the next) and in CTB anti-diagonal order; and through submit_async.  A mismatch names the TU
under the first differing sample and its plan class."""
import pytest

import intra_plan_cases as ipc
from libde265_b200 import capi
from libde265_b200.engine import Engine
from test_gpu_range_edges import _read_async

pytestmark = pytest.mark.gpu

DEPTHS = {"8": (8, None), "10": (10, None), "12": (12, None), "12_9": (12, 9)}
_pictures = {}


def pictures(depth):
    if depth not in _pictures:
        _pictures[depth] = ipc.coverage_pictures(*DEPTHS[depth])
    return _pictures[depth]


def check(pic, got, want, tag):
    msg = ipc.first_mismatch_class(pic, got, want)
    assert msg is None, f"{tag} {pic.params.width}x{pic.params.height} seed {pic.params.poc}: {msg}"


def run_against_oracle(oracle_mod, depth, stages, tag):
    e, orc = Engine(0), oracle_mod.Oracle()
    try:
        for p in pictures(depth):
            ipc.upload_references((e, orc), p)
            for st in stages:
                p.c.params.stop_after_stage = st
                e.submit(p)
                orc.reconstruct(p)
                check(p, e.read_slot(ipc.DST_SLOT, p.params), orc.read_slot(ipc.DST_SLOT, p.params), f"{tag} stage {st}")
            p.c.params.stop_after_stage = 0
    finally:
        orc.close()
        e.close()


@pytest.mark.parametrize("depth", list(DEPTHS))
def test_coverage_pictures_match_the_oracle(oracle_mod, depth):
    run_against_oracle(oracle_mod, depth, (capi.STAGE_RECON, capi.STAGE_ALL), f"{depth} bit")


@pytest.mark.parametrize("env", [{"B200_REGION": "8"}, {"B200_INTRA_SPLIT": "0"}, {"B200_INTRA_ORDER": "diag"}],
                         ids=lambda e: ",".join(f"{k}={v}" for k, v in e.items()))
@pytest.mark.parametrize("depth", ["10", "12_9"])
def test_other_intra_task_shapes(oracle_mod, monkeypatch, env, depth):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    run_against_oracle(oracle_mod, depth, (capi.STAGE_RECON,), f"{env} {depth} bit")


def test_submit_async(oracle_mod):
    """The 10-bit pictures queued with submit_async and queued reads (a sync before each new set of reference slots)."""
    pics = pictures("10")
    want = ipc.oracle_outputs(oracle_mod, pics, capi.STAGE_ALL)
    e = Engine(0)
    try:
        bufs = []
        for p in pics:
            if p.c.n_pu:
                e.sync()
                ipc.upload_references((e,), p)
            e.submit_async(p)
            bufs.append(_read_async(e, p))
        e.sync()
        for p, b, w in zip(pics, bufs, want):
            check(p, b, w, "submit_async")
    finally:
        e.close()
