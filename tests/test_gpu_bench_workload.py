"""Every picture bench.py decodes, on every path it times and under the engine switches its sweeps flip (-m gpu).

The workloads are bench.py's own (bench_workloads.build: its functions, rank 0's seeds); the oracle chain decodes them in
bench order on the CPU (pinned to the reference on the headline's first step by test_cpu_bench_workload_oracle.py).  Each
test runs a fresh engine the way a bench leg does and compares the md5 of every picture it decoded, or of every DPB slot at
the end, with the chain; a mismatch names the picture and reports its first differing sample."""
import filecmp
import importlib
import os

import numpy as np
import pytest
import torch

import bench
import bench_workloads as bw
from libde265_b200 import capi
from libde265_b200.engine import Engine
from test_gpu_parity import assert_same

pytestmark = pytest.mark.gpu

HEADLINE_STEPS = 4  # steps 2 and 3 replay the records of steps 0 and 1 on new reference content
LEG_STEPS = 2
MATRIX_STEPS = 2


def chain_fixture(name, steps):
    @pytest.fixture(scope="module")
    def fx():
        wl = bw.build(name)
        chain = bw.Chain(wl, steps)
        yield wl, chain
        chain.close()
    return fx


headline = chain_fixture("main_ra_4k", HEADLINE_STEPS)
main10_4k = chain_fixture("main10_4k", LEG_STEPS)
intra1080 = chain_fixture("intra1080", LEG_STEPS)


@pytest.fixture(scope="module")
def tight_dpb():
    """The headline workload under B200_TIGHT_DPB=1: 7 slots, every slot reused as early as the GOP allows.  It names the same
    reference POCs as the default workload (test_cpu_bench_workload.py), so it must decode to the same pictures."""
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("B200_TIGHT_DPB", "1")
        tight = importlib.reload(bench)
        try:
            assert (tight.KEY_SLOTS, tight.REFB_SLOTS, tight.NONREF_SLOTS) == (2, 3, 2)
            wl = bw.build("main_ra_4k", bench_mod=tight)
        finally:
            mp.delenv("B200_TIGHT_DPB")
            importlib.reload(bench)
    return wl


class PinnedPictures:
    """Page-locked host buffers, one per decoded picture (pageable destinations would make every read a host synchronisation and
    change the schedule under test).  Refilled with a pattern before every use, so that a read that never happened shows."""

    def __init__(self):
        self.buf = None

    def get(self, params, n):
        bps = 2 if params.bit_depth_luma > 8 else 1
        w, h = params.width, params.height
        shapes = [(h, w), (h // 2, w // 2), (h // 2, w // 2)]
        per = sum(a * b for a, b in shapes) * bps
        if self.buf is None or self.buf.numel() < per * n:
            self.buf = None
            self.buf = torch.empty(per * n, dtype=torch.uint8, pin_memory=True)
        self.buf.fill_(0xA5)
        arr = self.buf.numpy()
        dt = np.uint16 if bps == 2 else np.uint8
        out = []
        for k in range(n):
            off, planes = k * per, []
            for a, b in shapes:
                planes.append(arr[off:off + a * b * bps].view(dt).reshape(a, b))
                off += a * b * bps
            out.append(planes)
        return out


@pytest.fixture(scope="module")
def pinned():
    p = PinnedPictures()
    yield p
    p.buf = None


def queue_read(eng, slot, planes):
    capi.check(eng.lib.b200_engine_read_slot_async(eng.handle, slot, capi.PlaneArray(*[x.ctypes.data for x in planes]),
                                                   capi.StrideArray(*[x.strides[0] for x in planes])), "read_slot_async")


def upload_reference(eng, wl):
    if wl.ref0 is not None:  # the POC 0 reference, as bench.run_config uploads it
        eng.upload_slot(wl.key_slot, wl.seq[0].params, wl.ref0)


def run_value(eng, wl, steps, bufs=None):
    """bench's `value` leg: all 64 pictures prepared (records resident in HBM), then `steps` steps of run_prepared back to
    back as step_resident issues them; bufs: a read of every picture queued right behind it (None: no read in between)."""
    upload_reference(eng, wl)
    prepared = [eng.prepare(p) for p in wl.seq]
    try:
        for n, (_, _, j) in enumerate(bw.schedule(wl, steps)):
            eng.run_prepared(prepared[j])
            if bufs is not None:
                queue_read(eng, wl.seq[j].params.dst_slot, bufs[n])
        eng.sync()
    finally:
        for h in prepared:
            eng.free_prepared(h)


def run_e2e(eng, wl, steps, bufs, submit):
    """bench's `e2e` leg: host records submitted picture by picture, a read queued behind each."""
    upload_reference(eng, wl)
    for n, (_, _, j) in enumerate(bw.schedule(wl, steps)):
        p = wl.seq[j]
        submit(p)
        queue_read(eng, p.params.dst_slot, bufs[n])
    eng.sync()


def check_pictures(got_planes, want_md5, wl, steps, what, oracle_wl=None):
    """Every picture against the chain; on a mismatch the first differing sample of the first bad picture (the chain is re-run
    up to it on oracle_wl: the workload with the same pictures, when wl only differs in its slot assignment)."""
    got = [bw.md5_planes(b) for b in got_planes]
    assert len(got) == len(want_md5) == bw.PER_STEP * steps
    bad = [n for n, (g, w) in enumerate(zip(got, want_md5)) if g != w]
    if not bad:
        return
    n = bad[0]
    try:
        assert_same(got_planes[n], bw.oracle_picture(oracle_wl or wl, steps, n), "")
        detail = "(equal to the re-run oracle: the chain is not reproducible)"
    except AssertionError as e:
        detail = str(e).strip()
    pytest.fail(f"{what}: {len(bad)} of {len(got)} pictures differ from the oracle chain; first: {bw.describe(wl, steps, n)}:{detail}; "
                f"all: {', '.join(bw.describe(wl, steps, k) for k in bad[:8])}{' ...' if len(bad) > 8 else ''}")


def check_dpb(eng, wl, chain, what):
    """Every slot the chain left filled, read back from the engine after the run."""
    got = {s: eng.read_slot(s, prm) for s, prm in chain.params_of.items()}
    bad = [s for s in sorted(got) if bw.md5_planes(got[s]) != chain.dpb[s]]
    if not bad:
        return
    try:
        assert_same(got[bad[0]], bw.oracle_slot(wl, chain.steps, bad[0]), "")
        detail = "(equal to the re-run oracle: the chain is not reproducible)"
    except AssertionError as e:
        detail = str(e).strip()
    pytest.fail(f"{what}: DPB slots {bad} differ from the oracle chain after {chain.steps} steps; slot {bad[0]}:{detail}")


# ---- the headline (main_ra_4k), every path bench.py times ------------------------------------------------------------------
def test_value_as_timed_final_dpb_and_dump_outputs(headline, tmp_path):
    """`value` exactly as timed: 4 steps of run_prepared, no read in between; then every slot, and what --dump-outputs writes
    for the last step against the same dump of the oracle's final state."""
    wl, chain = headline
    eng = Engine(0)
    try:
        run_value(eng, wl, HEADLINE_STEPS)
        check_dpb(eng, wl, chain, "value")
        v = (HEADLINE_STEPS - 1) % bench.STEP_VARIANTS
        last_step = wl.seq[bw.PER_STEP * v:bw.PER_STEP * (v + 1)]
        bench.dump_outputs(str(tmp_path / "gpu"), eng, last_step)
    finally:
        eng.close()
    bench.dump_outputs(str(tmp_path / "orc"), chain.orc, last_step)
    names = ["luma.npy", "cb.npy", "cr.npy", "plane_sums.npy", "poc.npy"]
    assert sorted(os.listdir(tmp_path / "gpu")) == sorted(names)
    match, mismatch, errors = filecmp.cmpfiles(tmp_path / "gpu", tmp_path / "orc", names, shallow=False)
    assert not mismatch and not errors, f"--dump-outputs differs from the oracle's in {mismatch + errors}"


def test_value_every_picture(headline, pinned):
    wl, chain = headline
    bufs = pinned.get(wl.seq[0].params, bw.PER_STEP * HEADLINE_STEPS)
    eng = Engine(0)
    try:
        run_value(eng, wl, HEADLINE_STEPS, bufs)
    finally:
        eng.close()
    check_pictures(bufs, chain.pic_md5, wl, HEADLINE_STEPS, "value")


def test_stage_timing_pass_every_picture(headline, pinned):
    """The one-stream pass behind `stages` / `roofline` (timing on: no renaming, stream 0 only)."""
    wl, chain = headline
    bufs = pinned.get(wl.seq[0].params, bw.PER_STEP * HEADLINE_STEPS)
    eng = Engine(0)
    try:
        eng.enable_timing(True)
        run_value(eng, wl, HEADLINE_STEPS, bufs)
        stage_ms, n_timed = eng.timing_sum(reset=True)
    finally:
        eng.close()
    check_pictures(bufs, chain.pic_md5, wl, HEADLINE_STEPS, "stage timing pass")
    assert n_timed == bw.PER_STEP * HEADLINE_STEPS
    assert all(stage_ms[k] > 0 for k in ("inter_pred", "recon", "deblock", "sao", "total")), stage_ms


@pytest.mark.parametrize("mode", ["pinned_async", "pageable_async", "pageable_sync"])
def test_e2e_every_picture(headline, pinned, mode):
    """`e2e`: host records through submit_async from page-locked arrays (bench.pin_records), from pageable arrays
    (B200_E2E_PAGEABLE) and through the synchronous submit (B200_E2E_SYNC), a read queued behind every picture."""
    wl, chain = headline
    bufs = pinned.get(wl.seq[0].params, bw.PER_STEP * HEADLINE_STEPS)
    eng = Engine(0)
    try:
        if mode == "pinned_async":
            assert bench.pin_records(wl.seq, torch), "cudaHostRegister of the records failed"
        run_e2e(eng, wl, HEADLINE_STEPS, bufs, eng.submit if mode == "pageable_sync" else eng.submit_async)
    finally:
        if mode == "pinned_async":
            bench.unpin_records(wl.seq, torch)
        eng.close()
    check_pictures(bufs, chain.pic_md5, wl, HEADLINE_STEPS, f"e2e {mode}")


# ---- the legs ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("leg", ["main10_4k", "intra1080"])
def test_leg_value_final_dpb(request, leg):
    wl, chain = request.getfixturevalue(leg)
    eng = Engine(0)
    try:
        run_value(eng, wl, LEG_STEPS)
        check_dpb(eng, wl, chain, f"{leg} value")
    finally:
        eng.close()


@pytest.mark.parametrize("leg", ["main10_4k", "intra1080"])
def test_leg_value_every_picture(request, pinned, leg):
    wl, chain = request.getfixturevalue(leg)
    bufs = pinned.get(wl.seq[0].params, bw.PER_STEP * LEG_STEPS)
    eng = Engine(0)
    try:
        run_value(eng, wl, LEG_STEPS, bufs)
    finally:
        eng.close()
    check_pictures(bufs, chain.pic_md5, wl, LEG_STEPS, f"{leg} value")


# ---- the engine switches the sweeps flip (tools/sweep_bench.py, RESULTS.md), on the headline -----------------------------------
SWITCHES = [
    {"B200_MC_LEGACY": "1"}, {"B200_SAO_LEGACY": "1"},  # other kernels: k_inter_pred8, k_sao<u8> at CTB 64
    {"B200_MC_CTAS": "2"}, {"B200_MC_CTAS": "4"}, {"B200_INTRA_CTAS": "2"}, {"B200_INTRA_CTAS": "4"},
    {"B200_INTRA_I_GRID": "0"}, {"B200_INTRA_I_GRID": "48"}, {"B200_INTRA_I_GRID": "96"}, {"B200_IND_STREAMS": "1"}, {"B200_IND_STREAMS": "3"},
    {"B200_RENAME": "0"}, {"B200_SCHED": "rr"}, {"B200_REGION": "8"}, {"B200_INTRA_ORDER": "level_i"}, {"B200_INTRA_SPLIT": "0"},
    {"B200_INTRA_WIDTH_PCT": "100"}, {"B200_STREAMS": "1"}, {"B200_STREAMS": "12"}, {"B200_HOST_THREADS": "0"},
]


@pytest.mark.parametrize("env", SWITCHES, ids=lambda e: "-".join(f"{k[5:]}={v}" for k, v in e.items()))
def test_switch_every_picture(headline, pinned, monkeypatch, env):
    wl, chain = headline
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    bufs = pinned.get(wl.seq[0].params, bw.PER_STEP * MATRIX_STEPS)
    eng = Engine(0)
    try:
        run_value(eng, wl, MATRIX_STEPS, bufs)
    finally:
        eng.close()
    check_pictures(bufs, chain.pic_md5[:bw.PER_STEP * MATRIX_STEPS], wl, MATRIX_STEPS, f"value with {env}")


@pytest.mark.parametrize("rename", ["1", "0"])
def test_tight_dpb_every_picture(headline, tight_dpb, pinned, monkeypatch, rename):
    """The smallest DPB the GOP allows, where every WAR / WAW hazard between pictures is real: with slot renaming (what it
    exists for) and with renaming off (in-place writes ordered behind the readers)."""
    _, chain = headline
    monkeypatch.setenv("B200_RENAME", rename)
    bufs = pinned.get(tight_dpb.seq[0].params, bw.PER_STEP * MATRIX_STEPS)
    eng = Engine(0)
    try:
        run_value(eng, tight_dpb, MATRIX_STEPS, bufs)
    finally:
        eng.close()
    check_pictures(bufs, chain.pic_md5[:bw.PER_STEP * MATRIX_STEPS], tight_dpb, MATRIX_STEPS, f"tight DPB, B200_RENAME={rename}",
                   oracle_wl=headline[0])
