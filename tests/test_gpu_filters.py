"""GPU tests (-m gpu) of the in-loop filters branch by branch (filter_cases.py): the engine against the CPU oracle at
STAGE_RECON, STAGE_DEBLOCK and STAGE_ALL, sample for sample, on every case and on each SAO kernel: k_sao8 (8 bit, CTB 32 /
64, the default), k_sao<u8> (B200_SAO_LEGACY=1, and CTB 16) and k_sao<u16> (above 8 bit).  The oracle is pinned to the
reference on the same cases, and its filter decisions to a classifier that proves every branch is taken, by
test_cpu_filters.py."""
import pytest

import filter_cases
from libde265_b200 import capi
from libde265_b200.engine import Engine
from test_gpu_parity import assert_same

pytestmark = pytest.mark.gpu

STAGES = ((capi.STAGE_RECON, "recon"), (capi.STAGE_DEBLOCK, "deblock"), (capi.STAGE_ALL, "all"))


def sao_kernel(case, legacy):
    """The SAO kernel the engine runs on the case's pictures."""
    if case.bd > 8 or case.kw.get("bit_depth_chroma", case.bd) > 8:
        return "k_sao<u16>"
    return "k_sao<u8>" if legacy or case.kw.get("log2_ctb", 6) < 5 else "k_sao8"


# every case on the default engine, and the cases that run k_sao8 by default once more with the legacy kernel
RUNS = [(c.id, False) for c in filter_cases.CASES] + [(c.id, True) for c in filter_cases.CASES if sao_kernel(c, False) == "k_sao8"]


@pytest.fixture(scope="module")
def engines():
    made = {}

    def get(legacy):
        if legacy not in made:
            with pytest.MonkeyPatch.context() as mp:  # the engine reads its switches when it is created
                if legacy:
                    mp.setenv("B200_SAO_LEGACY", "1")
                else:
                    mp.delenv("B200_SAO_LEGACY", raising=False)
                made[legacy] = Engine(0)
        return made[legacy]
    yield get
    for e in made.values():
        e.close()


@pytest.mark.parametrize("case,legacy", RUNS, ids=[f"{c}-{'legacy' if l else 'default'}" for c, l in RUNS])
def test_engine_matches_oracle_on_the_filter_cases(engines, oracle_mod, case, legacy):
    c = filter_cases.BY_ID[case]
    kernel = sao_kernel(c, legacy)
    eng = engines(legacy)
    planes, pics = filter_cases.make_sequence(c.W, c.H, c.bd, **c.kw)
    orc = oracle_mod.Oracle()
    for e in (eng, orc):
        e.upload_slot(5, pics[0].params, planes)
    for i, p in enumerate(pics):
        for st, name in STAGES:
            p.c.params.stop_after_stage = st
            eng.submit(p)
            orc.reconstruct(p)
            assert_same(eng.read_slot(p.params.dst_slot, p.params), orc.read_slot(p.params.dst_slot, p.params),
                        f"{case} [{kernel}] pic {i} stage {name}")
        p.c.params.stop_after_stage = 0
    orc.close()
