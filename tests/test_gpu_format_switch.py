"""GPU tests (-m gpu) of one engine across format changes (format_cases.py): a new picture size, chroma format, bit depth or CTB
size between pictures, through every way pictures reach the engine -- submit() stage by stage, the asynchronous call with
read-backs queued on either side of a switch, prepared pictures of two formats interleaved, the benchmark's workload at two
formats on one engine, the utility calls between queued pictures, the kernel switches -- and real streams that switch format
through the drop-in path.  Every picture and every name read back is compared with the CPU oracle sample for sample; the oracle is
pinned to the reference on the same cases by test_cpu_format_switch.py.  A fresh engine per test: nothing of an earlier test's
format may leak into a case."""
import functools
import hashlib
import os

import numpy as np
import pytest

import bench
import format_cases
import oracle_lib
from libde265_b200 import capi, de265, synth
from libde265_b200.engine import Engine
from test_cpu_oracle import GOLDEN
from test_gpu_parity import assert_same

pytestmark = pytest.mark.gpu


def md5_planes(planes):
    return hashlib.md5(b"".join(p.tobytes() for p in planes)).hexdigest()


def buffers(params):
    dt = np.uint16 if params.bit_depth_luma > 8 else np.uint8
    W, H = params.width, params.height
    return [np.empty((H, W), dt)] + ([np.empty((H // 2, W // 2), dt) for _ in range(2)] if params.chroma_format_idc else [])


def read_async(e, slot, params):
    """Queues a read of `slot` (holding a picture of format `params`) into fresh arrays; valid after e.sync()."""
    bufs = buffers(params)
    capi.check(e.lib.b200_engine_read_slot_async(e.handle, slot, capi.PlaneArray(*[x.ctypes.data for x in bufs] + [None] * (3 - len(bufs))),
                                                 capi.StrideArray(*[x.strides[0] for x in bufs] + [0] * (3 - len(bufs)))), "read_slot_async")
    return bufs


def other_format_names(case, i):
    """After picture i: [(slot, index of the picture it holds)] for every name that holds a picture of another format."""
    held = {}
    for j, (_, _, dst, _) in enumerate(case.steps[:i + 1]):
        held[dst] = j
    f = case.steps[i][0]
    return [(s, j) for s, j in sorted(held.items()) if case.steps[j][0] != f]


@functools.lru_cache(maxsize=None)
def oracle_trace(case_id):
    """The oracle decoding the case once: (planes of every picture, {i: [(slot, planes)] of the other-format names after a
    switch picture i}, {slot: (params, planes)} at the end)."""
    c = format_cases.BY_ID[case_id]
    pics = format_cases.make_sequence(case_id)
    orc = oracle_lib.Oracle()
    out, old, end = [], {}, {}
    for i, p in enumerate(pics):
        orc.reconstruct(p)
        out.append(orc.read_slot(p.params.dst_slot, p.params))
        if i and c.steps[i][0] != c.steps[i - 1][0]:
            old[i] = [(s, orc.read_slot(s, pics[j].params)) for s, j in other_format_names(c, i)]
        end[p.params.dst_slot] = p.params
    end = {s: (prm, orc.read_slot(s, prm)) for s, prm in end.items()}
    orc.close()
    return out, old, end


def check_end(e, case_id):
    """Every name of the engine against the oracle at the end, the names that still hold an earlier format's picture included."""
    _, _, end = oracle_trace(case_id)
    for s, (prm, want) in sorted(end.items()):
        assert_same(e.read_slot(s, prm), want, f"{case_id} slot {s} at the end")


# ---- (a) synchronous submit, stage by stage ----
@pytest.mark.parametrize("case", format_cases.CASE_IDS)
def test_submit_every_stage_across_switches(oracle_mod, case):
    """Each picture first in full (it writes its name in its own format, over whatever the name held), then stage by stage.  The
    full pass comes first so that at STAGE_INTER_PRED the samples of intra CUs, which that stage leaves alone, hold the same
    picture in the engine and in the oracle."""
    pics = format_cases.make_sequence(case)
    stages = (capi.STAGE_ALL, capi.STAGE_INTER_PRED, capi.STAGE_RECON, capi.STAGE_DEBLOCK, capi.STAGE_ALL)
    e, orc = Engine(0), oracle_mod.Oracle()
    try:
        for i, p in enumerate(pics):
            for st in stages:
                p.c.params.stop_after_stage = st
                e.submit(p)
                orc.reconstruct(p)
                assert_same(e.read_slot(p.params.dst_slot, p.params), orc.read_slot(p.params.dst_slot, p.params), f"{case} pic {i} stage {st}")
            p.c.params.stop_after_stage = 0
        check_end(e, case)
    finally:
        for p in pics:
            p.c.params.stop_after_stage = 0
        orc.close()
        e.close()


# ---- (b) queued, with read-backs on either side of every switch; (f) under the kernel switches ----
def run_queued(case, streams=None):
    """Every picture through submit_async with a read of its name queued behind it; after the first picture of each new format
    also reads of the names that still hold the previous formats' pictures (what the drop-in does when it fetches one call
    late).  Then every name at the end."""
    c = format_cases.BY_ID[case]
    pics = format_cases.make_sequence(case)
    out, old, _ = oracle_trace(case)
    e = Engine(0)
    try:
        if streams is not None:
            e.set_streams(streams)
        got, got_old = [], {}
        for i, p in enumerate(pics):
            e.submit_async(p)
            got.append(read_async(e, p.params.dst_slot, p.params))
            if i in old:
                got_old[i] = [(s, read_async(e, s, pics[j].params)) for s, j in other_format_names(c, i)]
        e.sync()
        for i, (g, w) in enumerate(zip(got, out)):
            assert_same(g, w, f"{case} pic {i}")
        for i, reads in got_old.items():
            for (s, g), (s2, w) in zip(reads, old[i]):
                assert s == s2
                assert_same(g, w, f"{case}: slot {s} read after the switch at pic {i}")
        check_end(e, case)
    finally:
        e.close()


@pytest.mark.parametrize("config", ["1", "4", "8", "8_no_rename"])
@pytest.mark.parametrize("case", format_cases.CASE_IDS)
def test_queued_across_switches(monkeypatch, case, config):
    if config.endswith("no_rename"):
        monkeypatch.setenv("B200_RENAME", "0")
    run_queued(case, streams=int(config.split("_")[0]))


@pytest.mark.parametrize("env", ["B200_MC_LEGACY", "B200_SAO_LEGACY", "B200_STREAMS"])
@pytest.mark.parametrize("case", format_cases.CASE_IDS)
def test_queued_across_switches_kernel_variants(monkeypatch, case, env):
    """k_inter_pred8 instead of the TMA-staged MC kernel, k_sao on every 8-bit picture, one stream."""
    monkeypatch.setenv(env, "1")
    run_queued(case)


# ---- (c) prepared pictures of two formats, interleaved ----
PAIRS = {
    "bytes": (format_cases.S8, format_cases.S10),
    "depth": (format_cases.D9, format_cases.D10),
    "size_chroma": (format_cases.A, format_cases.fmt(200, 136, cf=0)),
}


def pair_pictures(name):
    """Three pictures of each format, A on names 0-2 and B on names 3-5; B's P and B pictures also reference A's names."""
    a, b = PAIRS[name]
    mk = lambda f, t, seed, dst, refs=(): synth.make_picture(f.W, f.H, t, seed=seed, dst_slot=dst, ref_slots=refs, bit_depth=f.bd,
                                                             bit_depth_chroma=f.bdc, chroma_format_idc=f.cf, log2_ctb=f.ctb)
    A = [mk(a, "I", 901, 0), mk(a, "P", 902, 1, (0, 4)), mk(a, "B", 903, 2, (0, 1, 3))]
    B = [mk(b, "I", 911, 3), mk(b, "P", 912, 4, (3, 0)), mk(b, "B", 913, 5, (3, 4, 1))]
    return [p for ab in zip(A, B) for p in ab]  # A B A B A B


@pytest.mark.parametrize("pair", sorted(PAIRS))
def test_prepared_two_formats_interleaved(oracle_mod, pair):
    """The pictures of two formats prepared up front, run A B A B ... twice over with reads queued behind each and no sync in
    between; the handles are freed after the switches."""
    order = pair_pictures(pair)
    orc = oracle_mod.Oracle()
    want = []
    for _ in range(2):
        for p in order:
            orc.reconstruct(p)
            want.append(orc.read_slot(p.params.dst_slot, p.params))
    end = {p.params.dst_slot: (p.params, orc.read_slot(p.params.dst_slot, p.params)) for p in order}
    orc.close()
    e = Engine(0)
    try:
        hs = [e.prepare(p) for p in order]
        got = []
        for _ in range(2):
            for p, h in zip(order, hs):
                e.run_prepared(h)
                got.append(read_async(e, p.params.dst_slot, p.params))
        for h in hs:
            e.free_prepared(h)
        e.sync()
        for n, (g, w) in enumerate(zip(got, want)):
            assert_same(g, w, f"{pair}: round {n // len(order)} pic {n % len(order)}")
        for s, (prm, w) in sorted(end.items()):
            assert_same(e.read_slot(s, prm), w, f"{pair} slot {s} at the end")
    finally:
        e.close()


# ---- (d) the benchmark's workload at two formats on one engine ----
BENCH_FORMATS = ((640, 368, 8), (416, 240, 10))


def test_bench_workload_two_formats_one_engine(oracle_mod):
    """bench.build_workload at 640x368 8-bit (A) and 416x240 10-bit (B), prepared and run on one engine with the default streams
    and renaming as tools/format_switch.py does: A for 2 steps, B for 2 steps, A for 2 steps, each phase starting with its key
    picture uploaded.  The oracle replays the same interleaved schedule: when A comes back some of its names hold B pictures,
    which its pictures then predict from as from missing references."""
    wls = []
    for w, h, bd in BENCH_FORMATS:
        seq, key_slot, _ = bench.build_workload(w, h, bd, seed0=1000 + bd)
        wls.append((seq, key_slot, synth.random_planes(w, h, bd, 7 + bd)))
    phases = [0, 1, 0]
    sched = [(ph, 32 * (s % bench.STEP_VARIANTS) + i) for ph in phases for s in range(2) for i in range(32)]
    orc = oracle_mod.Oracle()
    want, n = [], 0
    for ph in phases:
        seq, key, ref0 = wls[ph]
        orc.upload_slot(key, seq[0].params, ref0)
        for _ in range(64):
            p = seq[sched[n][1]]
            orc.reconstruct(p)
            want.append(md5_planes(orc.read_slot(p.params.dst_slot, p.params)))
            n += 1
    held = {}
    for ph, j in sched:
        held[wls[ph][0][j].params.dst_slot] = wls[ph][0][j].params
    end = {s: md5_planes(orc.read_slot(s, prm)) for s, prm in held.items()}
    orc.close()
    e = Engine(0)
    try:
        got, n = [], 0
        for ph in phases:
            seq, key, ref0 = wls[ph]
            e.upload_slot(key, seq[0].params, ref0)
            hs = [e.prepare(p) for p in seq]
            for s in range(2):
                v = s % bench.STEP_VARIANTS
                for i in range(32):
                    e.run_prepared(hs[32 * v + i])
                    got.append(read_async(e, seq[32 * v + i].params.dst_slot, seq[32 * v + i].params))
                    n += 1
            e.sync()
            for h in hs:
                e.free_prepared(h)
        bad = [k for k, (g, w) in enumerate(zip(got, want)) if md5_planes(g) != w]
        assert not bad, f"{len(bad)} of {len(got)} pictures differ, first: phase {bad[0] // 64} step {bad[0] % 64 // 32} index {bad[0] % 32}"
        bad = [s for s, prm in sorted(held.items()) if md5_planes(e.read_slot(s, prm)) != end[s]]
        assert not bad, f"slots {bad} differ at the end"
    finally:
        e.close()


# ---- (e) the utility calls between queued pictures of another format ----
def test_upload_and_fill_between_queued_pictures_of_another_format(oracle_mod):
    """8-bit pictures queued with submit_async, then upload_slot and fill_slot of 10-bit pictures (one onto a name the queued
    pictures write and read), 10-bit pictures that reference them and the 8-bit names, and 8-bit pictures again."""
    S8, S10 = format_cases.S8, format_cases.S10
    mk = lambda f, t, seed, dst, refs=(): synth.make_picture(f.W, f.H, t, seed=seed, dst_slot=dst, ref_slots=refs, bit_depth=f.bd)
    first = [mk(S8, "I", 921, 0), mk(S8, "P", 922, 1, (0,)), mk(S8, "B", 923, 2, (0, 1))]
    second = [mk(S10, "B", 924, 4, (3, 1, 0)), mk(S10, "P", 925, 5, (4, 3))]
    third = [mk(S8, "P", 926, 6, (0, 2, 1)), mk(S8, "B", 927, 1, (6, 2, 4))]
    planes10 = synth.random_planes(S10.W, S10.H, 10, 928)
    p10 = second[0].params
    orc = oracle_mod.Oracle()
    want = []

    def utility(x):
        x.upload_slot(3, p10, planes10)
        x.fill_slot(1, p10, 300, 700)

    for p in first:
        orc.reconstruct(p)
        want.append(orc.read_slot(p.params.dst_slot, p.params))
    utility(orc)
    for p in second + third:
        orc.reconstruct(p)
        want.append(orc.read_slot(p.params.dst_slot, p.params))
    end = {s: (prm, orc.read_slot(s, prm)) for s, prm in ((0, first[0].params), (2, first[2].params), (3, p10), (4, p10), (5, p10),
                                                          (6, third[0].params), (1, third[1].params))}
    orc.close()
    e = Engine(0)
    try:
        e.set_streams(4)
        got = []
        for p in first:
            e.submit_async(p)
            got.append(read_async(e, p.params.dst_slot, p.params))
        utility(e)
        for p in second + third:
            e.submit_async(p)
            got.append(read_async(e, p.params.dst_slot, p.params))
        e.sync()
        for i, (g, w) in enumerate(zip(got, want)):
            assert_same(g, w, f"pic {i}")
        for s, (prm, w) in sorted(end.items()):
            assert_same(e.read_slot(s, prm), w, f"slot {s} at the end")
    finally:
        e.close()


# ---- the drop-in path on real streams that switch format ----
PARTS = ("girlshy", "intra1080", "intra4k", "girlshy")
HAVE_DROPIN = oracle_lib.ref_path("libde265_hooked.so") is not None and oracle_lib.ref_path("libde265_ref.so") is not None


def concatenated():
    return b"".join(open(os.path.join(GOLDEN, n + ".h265"), "rb").read() for n in PARTS)


@functools.lru_cache(maxsize=None)
def reference_md5s():
    """What the unmodified reference decoder outputs from the concatenated bytes: one md5 per picture."""
    out = []
    ref = de265.Decoder(oracle_lib.ref_path("libde265_ref.so"))
    ref.decode_stream(concatenated(), lambda img: out.append(hashlib.md5(b"".join(img.plane_bytes(c) for c in range(3))).hexdigest()))
    ref.close()
    return out


EXPECTED_PICTURES = 75 + 2 + 1 + 75  # girlshy, intra1080, intra4k, girlshy


@pytest.mark.parametrize("lag,queued", [(0, False), (1, False), (0, True), (1, True)])
@pytest.mark.skipif(not HAVE_DROPIN, reason="oracle/_ref not shipped")
def test_dropin_streams_that_switch_format(b200lib, monkeypatch, lag, queued):
    """316x240 -> 1920x1080 -> 3840x2160 -> 316x240, each part with its own parameter sets and an IDR picture, decoded by one
    libde265 decoder with the B200 backend selected: every picture as the unmodified reference decodes the same bytes."""
    if queued:
        monkeypatch.setenv("B200_HOOK_ASYNC", "1")
    want = reference_md5s()
    assert len(want) == EXPECTED_PICTURES
    got = []
    dec = de265.Decoder(oracle_lib.ref_path("libde265_hooked.so"))
    dec.select_b200()
    dec.decode_stream(concatenated(), lambda img: got.append(hashlib.md5(b"".join(img.plane_bytes(c) for c in range(3))).hexdigest()), lag=lag)
    dec.close()
    assert len(got) == len(want), f"{len(got)} pictures, the reference outputs {len(want)}"
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert not bad, f"pictures {bad[:10]} differ ({len(bad)} in all)"


@pytest.mark.skipif(not HAVE_DROPIN, reason="oracle/_ref not shipped")
def test_sink_streams_that_switch_format(b200lib):
    """The same bytes through the sink path: one engine reconstructs every picture the hooked parser records."""
    want = reference_md5s()
    eng = Engine(0)
    dec = de265.Decoder(oracle_lib.ref_path("libde265_hooked.so"))

    def sink(pic, planes, strides):
        eng.submit(pic)
        eng.read_slot_into(pic.params.dst_slot, [planes[0], planes[1], planes[2]], [strides[0], strides[1], strides[2]])
        return 0

    dec.attach(sink)
    got = []
    dec.decode_stream(concatenated(), lambda img: got.append(hashlib.md5(b"".join(img.plane_bytes(c) for c in range(3))).hexdigest()))
    dec.close()
    eng.close()
    assert len(got) == len(want) == EXPECTED_PICTURES
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert not bad, f"pictures {bad[:10]} differ ({len(bad)} in all)"
