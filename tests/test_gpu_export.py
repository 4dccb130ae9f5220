"""GPU tests (-m gpu) of b200_engine_export_slot through Engine.export: cropped YUV and planar RGB in CUDA memory, enqueued on
the caller's stream.  YUV exports equal read_slot cropped; RGB exports equal export_ref's restatement of the integer formula
applied to read_slot (or to the oracle at full size).  The ordering cases each decide their result by themselves and run once: a
bounded torch.cuda._sleep holds the caller's stream so that a missing wait would let the engine overwrite the surface first."""
import ctypes as C
import time

import numpy as np
import pytest
import torch

import export_ref
from libde265_b200 import capi, synth
from libde265_b200.engine import Engine
from test_gpu_parity import assert_same, md5_planes

pytestmark = pytest.mark.gpu

INVALID = -1  # B200_ERR_INVALID
SLEEP_CYCLES = 200_000_000  # about 0.1 s at the H100's clock: longer than any picture these tests submit behind it
RGB = list(export_ref.RGB_NAMES)


def to_np(t):
    t = t.cpu()
    return t.view(torch.int16).numpy().view(np.uint16) if t.dtype == torch.uint16 else t.numpy()


def crop_planes(planes, crop, mono):
    x, y, w, h = crop
    out = [planes[0][y:y + h, x:x + w]]
    if not mono:
        out += [p[y // 2:(y + h) // 2, x // 2:(x + w) // 2] for p in planes[1:]]
    return out


def check_export(eng, slot, params, planes, crops, stream=None):
    """Every crop as YUV and as every RGB matrix and range, against `planes` (the picture as read_slot / the oracle gives it)."""
    mono = params.chroma_format_idc == 0
    got = []
    for crop in crops:
        got.append((crop, None, False, eng.export(slot, params, crop=crop, stream=stream)))
        for rgb in RGB:
            for full in (False, True):
                got.append((crop, rgb, full, eng.export(slot, params, crop=crop, rgb=rgb, full_range=full, stream=stream)))
    torch.cuda.synchronize()
    for crop, rgb, full, out in got:
        c = crop if crop is not None else (0, 0, params.width, params.height)
        tag = f"{params.width}x{params.height} {params.bit_depth_luma}/{params.bit_depth_chroma} crop {c} {rgb or 'yuv'}{' full' if full else ''}"
        if rgb is None:
            assert len(out) == (1 if mono else 3), tag
            assert_same([to_np(t) for t in out], crop_planes(planes, c, mono), tag)
        else:
            assert out.shape == (3, c[3], c[2]) and out.dtype == torch.uint8, tag
            want = export_ref.rgb_planes(export_ref.RGB_NAMES[rgb], full, params.bit_depth_luma, params.bit_depth_chroma, planes, c)
            assert_same(list(to_np(out)), list(want), tag)


# (id, W, H, luma depth, chroma depth, chroma format, log2 CTB)
FORMATS = [("8bit", 200, 136, 8, 8, 1, 6), ("10bit", 208, 120, 10, 10, 1, 4), ("12bit", 136, 72, 12, 12, 1, 6),
           ("10_12", 200, 136, 10, 12, 1, 5), ("12_9", 72, 40, 12, 9, 1, 4), ("mono8", 200, 136, 8, 8, 0, 6), ("mono10", 136, 72, 10, 10, 0, 4)]


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


@pytest.mark.parametrize("fmt", FORMATS, ids=[f[0] for f in FORMATS])
def test_yuv_and_rgb_exports_equal_read_slot(eng, fmt):
    _, W, H, bd, bdc, chroma, log2_ctb = fmt
    p = synth.make_picture(W, H, "I", seed=61, dst_slot=4, bit_depth=bd, bit_depth_chroma=bdc, chroma_format_idc=chroma, log2_ctb=log2_ctb)
    eng.submit(p)
    planes = eng.read_slot(4, p.params)
    crops = [None, (2, 2, W - 8, H - 4), (14, 6, 34, 18), (W - 10, H - 8, 10, 8), (6, 0, 2, 2)]
    if not chroma:
        crops += [(3, 5, 41, 27), (W - 1, H - 1, 1, 1)]  # 4:0:0 takes odd windows
    check_export(eng, 4, p.params, planes, crops)
    # on a side stream, into outputs allocated there
    s = torch.cuda.Stream()
    check_export(eng, 4, p.params, planes, [(10, 2, W - 20, H - 4)], stream=s)


@pytest.mark.parametrize("bd", [8, 10])
def test_4k_b_picture_exports_equal_the_oracle(oracle_mod, bd):
    """3840x2160 B pictures (8 bit, and Main10 with explicit weights), exported right after submission, against the oracle's planes."""
    W, H = 3840, 2160
    e = Engine(0)
    orc = oracle_mod.Oracle()
    b = synth.make_picture(W, H, "B", seed=62 + bd, dst_slot=2, ref_slots=(0, 1), bit_depth=bd, weighted=bd > 8)
    for s in (0, 1):
        r = synth.random_planes(W, H, bd, 70 + s)
        e.upload_slot(s, b.params, r)
        orc.upload_slot(s, b.params, r)
    e.submit(b)
    yuv = e.export(2, b.params)
    rgb = e.export(2, b.params, rgb="bt709" if bd == 8 else "bt2020")
    crop = (1918, 2, 1024, 1000)
    yuv_c = e.export(2, b.params, crop=crop)
    orc.reconstruct(b)
    want = orc.read_slot(2, b.params)
    torch.cuda.synchronize()
    assert_same([to_np(t) for t in yuv], want, f"4K {bd}-bit YUV")
    assert_same([to_np(t) for t in yuv_c], crop_planes(want, crop, False), f"4K {bd}-bit YUV crop")
    assert_same(list(to_np(rgb)), list(export_ref.rgb_planes(2 if bd == 8 else 3, False, bd, bd, want)), f"4K {bd}-bit RGB")
    orc.close()
    e.close()


@pytest.mark.parametrize("queued", [False, True], ids=["submit", "submit_async"])
def test_export_right_after_submit_of_a_4k_intra_picture(queued):
    """The export waits for the picture that writes the slot, through the asynchronous queue too."""
    W, H = 3840, 2160
    e = Engine(0)
    p = synth.make_picture(W, H, "I", seed=63, dst_slot=3)
    e.fill_slot(3, p.params, 0, 0)
    (e.submit_async if queued else e.submit)(p)
    yuv = e.export(3, p.params)
    rgb = e.export(3, p.params, rgb="bt601")
    torch.cuda.current_stream().synchronize()
    got_yuv, got_rgb = [to_np(t) for t in yuv], to_np(rgb)
    want = e.read_slot(3, p.params)
    assert_same(got_yuv, want, "4K I YUV")
    assert_same(list(got_rgb), list(export_ref.rgb_planes(1, False, 8, 8, want)), "4K I RGB")
    e.close()


def small_pair(W=416, H=240, bd=8):
    a = synth.make_picture(W, H, "I", seed=64, dst_slot=0, bit_depth=bd)
    b = synth.make_picture(W, H, "I", seed=65, dst_slot=0, bit_depth=bd)
    return a, b


def delayed_exports(e, slot, params, stream):
    """A YUV and an RGB export of `slot` on `stream`, held back by a sleep enqueued in front of them."""
    with torch.cuda.stream(stream):
        torch.cuda._sleep(SLEEP_CYCLES)
    return e.export(slot, params, stream=stream), e.export(slot, params, rgb="bt709", stream=stream)


def assert_old_picture(exported, old, params, tag):
    yuv, rgb = exported
    assert_same([to_np(t) for t in yuv], old, tag + " YUV")
    assert_same(list(to_np(rgb)), list(export_ref.rgb_planes(2, False, params.bit_depth_luma, params.bit_depth_chroma, old)), tag + " RGB")


@pytest.mark.parametrize("mode", ["rename", "no_rename", "one_stream"])
def test_delayed_export_then_a_picture_that_writes_the_same_name(oracle_mod, monkeypatch, mode):
    monkeypatch.setenv("B200_RENAME", "0" if mode == "no_rename" else "1")
    e = Engine(0)
    if mode == "one_stream":
        e.set_streams(1)
    orc = oracle_mod.Oracle()
    a, b = small_pair()
    e.submit(a)
    old = e.read_slot(0, a.params)
    s = torch.cuda.Stream()
    exported = delayed_exports(e, 0, a.params, s)
    e.submit(b)
    s.synchronize()
    assert_old_picture(exported, old, a.params, mode)
    orc.reconstruct(b)
    assert_same(e.read_slot(0, b.params), orc.read_slot(0, b.params), mode + ": the later picture")
    orc.close()
    e.close()


@pytest.mark.parametrize("kind", ["fill_slot", "upload_slot", "format_change"])
def test_delayed_export_then_a_utility_write_or_a_format_change(kind):
    e = Engine(0)
    a, b = small_pair()
    e.submit(a)
    old = e.read_slot(0, a.params)
    s = torch.cuda.Stream()
    exported = delayed_exports(e, 0, a.params, s)
    if kind == "fill_slot":
        e.fill_slot(0, a.params, 1, 2)
        after = [np.full_like(p, v) for p, v in zip(old, (1, 2, 2))]
    elif kind == "upload_slot":
        after = synth.random_planes(a.params.width, a.params.height, 8, 66)
        e.upload_slot(0, a.params, after)
    else:  # the name moves off the exported surface, then a picture of another size frees every unnamed surface
        e.submit(b)
        c = synth.make_picture(256, 128, "I", seed=67, dst_slot=1)
        e.submit(c)
        after = None
    s.synchronize()
    assert_old_picture(exported, old, a.params, kind)
    if after is not None:
        assert_same(e.read_slot(0, a.params), after, kind + ": the write")
    e.sync()
    e.close()


def test_exports_of_one_surface_from_two_streams(monkeypatch):
    """The second export's stream waits for the first export before it records the surface's external read, so a picture that
    writes the surface in place waits for both."""
    monkeypatch.setenv("B200_RENAME", "0")
    e = Engine(0)
    a, b = small_pair()
    e.submit(a)
    old = e.read_slot(0, a.params)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    first = delayed_exports(e, 0, a.params, s1)
    second = e.export(0, a.params, stream=s2), e.export(0, a.params, rgb="bt709", stream=s2)
    e.submit(b)
    s1.synchronize()
    s2.synchronize()
    assert_old_picture(first, old, a.params, "delayed stream")
    assert_old_picture(second, old, a.params, "second stream")
    e.close()


@pytest.mark.parametrize("how", ["wait_slot", "sync"])
def test_wait_slot_and_sync_wait_for_exports(how):
    e = Engine(0)
    a, _ = small_pair()
    e.submit(a)
    old = e.read_slot(0, a.params)
    s = torch.cuda.Stream()
    exported = delayed_exports(e, 0, a.params, s)
    behind = torch.cuda.Event()
    behind.record(s)
    e.wait_slot(0) if how == "wait_slot" else e.sync()
    deadline = time.monotonic() + 0.005  # the event is recorded right behind the export: it completes a moment after it
    while not behind.query() and time.monotonic() < deadline:
        pass
    assert behind.query(), f"{how} returned while the export was still held back"
    assert_old_picture(exported, old, a.params, how)
    e.close()


def test_pipelined_hierarchical_b_exports_through_the_queue(oracle_mod):
    """test_gpu_parity's hierarchical-B sequence with a ring of 10 slots on 8 streams through submit_async, every picture exported
    right after its submission (later pictures rename or overwrite the slots the exports read), twice over."""
    W, H = 256, 128
    order = [("I", 0, ()), ("P", 8, (0,)), ("B", 4, (0, 8)), ("B", 2, (0, 4)), ("B", 1, (0, 2)), ("B", 3, (2, 4)), ("B", 6, (4, 8)),
             ("B", 5, (4, 6)), ("B", 7, (6, 8)), ("P", 16, (8,)), ("B", 12, (8, 16)), ("B", 10, (8, 12)), ("B", 9, (8, 10)),
             ("B", 11, (10, 12)), ("B", 14, (12, 16)), ("B", 13, (12, 14)), ("B", 15, (14, 16)), ("I", 24, ())]
    ring = 10
    pics = [synth.make_picture(W, H, t, seed=500 + poc, dst_slot=poc % ring, ref_slots=tuple(r % ring for r in refs)) for t, poc, refs in order]
    orc = oracle_mod.Oracle()
    expect = []
    for p in pics:
        orc.reconstruct(p)
        expect.append(md5_planes(orc.read_slot(p.params.dst_slot, p.params)))
    orc.close()
    e = Engine(0)
    e.set_streams(8)
    for rep in range(2):
        outs = []
        for p in pics:
            e.submit_async(p)
            outs.append(e.export(p.params.dst_slot, p.params))
        torch.cuda.current_stream().synchronize()
        got = [md5_planes([to_np(t) for t in o]) for o in outs]
        assert got == expect, f"round {rep}: pictures {[i for i, (g, x) in enumerate(zip(got, expect)) if g != x]} differ"
    e.sync()
    e.close()


def raw_export(e, slot, ex, ptrs, pitches):
    return e.lib.b200_engine_export_slot(e.handle, slot, C.byref(ex), capi.PlaneArray(*ptrs), capi.StrideArray(*pitches),
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream))


def test_every_invalid_export_is_rejected_and_the_engine_stays_usable(oracle_mod):
    e = Engine(0)
    orc = oracle_mod.Oracle()
    W, H = 64, 48
    p = synth.make_picture(W, H, "I", seed=68, dst_slot=0)
    p10 = synth.make_picture(W, H, "I", seed=69, dst_slot=1, bit_depth=10)
    e.submit(p)
    e.submit(p10)
    for slot in (5, -1, 32):  # no picture, out of range
        with pytest.raises(capi.B200Error):
            e.export(slot, p.params)
    for crop in [(W - 2, 0, 4, 2), (0, H - 2, 2, 4), (0, 0, 0, 2), (0, 0, 2, 0), (1, 0, 2, 2), (0, 1, 2, 2), (0, 0, 3, 2), (0, 0, 2, 3), (-2, 0, 2, 2)]:
        for rgb in (None, "bt709"):
            with pytest.raises(capi.B200Error):
                e.export(0, p.params, crop=crop, rgb=rgb)
    with pytest.raises(ValueError):
        e.export(0, p.params, rgb="srgb")
    buf = torch.zeros(4 * W * H, dtype=torch.uint8, device="cuda")
    base = buf.data_ptr()
    ptrs, pitches = [base, base + 2 * W * H, base + 3 * W * H], [2 * W, 2 * W, 2 * W]
    ok = capi.Export(0, 0, W, H, capi.EXPORT_YUV, 0)
    assert raw_export(e, 0, ok, ptrs, pitches) == 0
    for c in range(3):  # a plane the format needs is missing
        for fmt in (capi.EXPORT_YUV, capi.EXPORT_RGB_BT601):
            assert raw_export(e, 0, capi.Export(0, 0, W, H, fmt, 0), [None if i == c else v for i, v in enumerate(ptrs)], pitches) == INVALID
    for slot, fmt, row in ((0, capi.EXPORT_YUV, [W, W // 2, W // 2]), (1, capi.EXPORT_YUV, [2 * W, W, W]), (0, capi.EXPORT_RGB_BT2020, [W, W, W])):
        for c in range(3):  # a pitch below one row
            assert raw_export(e, slot, capi.Export(0, 0, W, H, fmt, 0), ptrs, [r - 1 if i == c else 2 * W for i, r in enumerate(row)]) == INVALID
        assert raw_export(e, slot, capi.Export(0, 0, W, H, fmt, 0), ptrs, row) == 0
    bad = [capi.Export(0, 0, W, H, 4, 0), capi.Export(0, 0, W, H, 255, 0), capi.Export(0, 0, W, H, capi.EXPORT_RGB_BT709, 0x02),
           capi.Export(0, 0, W, H, capi.EXPORT_YUV, 0x80), capi.Export(0, 0, W, H, capi.EXPORT_YUV, 0, (C.c_uint8 * 2)(1, 0)),
           capi.Export(0, 0, W, H, capi.EXPORT_YUV, 0, (C.c_uint8 * 2)(0, 1))]
    for ex in bad:
        assert raw_export(e, 0, ex, ptrs, pitches) == INVALID
    assert raw_export(e, 0, ok, ptrs, pitches) == 0
    torch.cuda.synchronize()
    # the engine decodes and exports as before
    q = synth.make_picture(W, H, "P", seed=70, dst_slot=2, ref_slots=(0,))
    e.submit(q)
    orc.reconstruct(p)
    orc.reconstruct(q)
    want = orc.read_slot(2, q.params)
    assert_same(e.read_slot(2, q.params), want, "after the rejected exports")
    assert_same([to_np(t) for t in e.export(2, q.params)], want, "export after the rejected exports")
    assert_same(list(to_np(e.export(2, q.params, rgb="bt601"))), list(export_ref.rgb_planes(1, False, 8, 8, want)), "RGB after the rejected exports")
    orc.close()
    e.close()
