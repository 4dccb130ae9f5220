"""Speed of b200_engine_export_slot on one GPU, printed as one JSON line (RESULTS.md records it):

  micro  microseconds per 3840x2160 picture for the YUV export (2-D device copies) and the RGB export (k_export_rgb) at 8 and 10
         bit: CUDA events around `--exports` back-to-back exports on one stream, after warm-up; achieved bytes/s from the bytes the
         export must read and write, against the H100 SXM data sheet's 3.35 TB/s.
  chain  frames/s of bench.py's headline chain (4K 8-bit random access, records resident in HBM, `value`), alternately without
         and with an RGB (BT.709) export of every picture on a stream of its own, right after the picture is issued.

Usage: python tools/export_bench.py [--exports 200] [--steps 10] [--rounds 3]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from libde265_b200 import capi, synth  # noqa: E402
from libde265_b200.engine import Engine  # noqa: E402

W, H = 3840, 2160
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def export_bytes(bd, rgb):
    """Bytes one 4:2:0 export of the whole picture must move: the planes read, the planes written."""
    src = W * H * 3 // 2 * (2 if bd > 8 else 1)
    return src + (3 * W * H if rgb else src)


def micro(n_exports):
    out = {}
    for bd in (8, 10):
        e = Engine(0)
        params = capi.PicParams(width=W, height=H, chroma_format_idc=1, bit_depth_luma=bd, bit_depth_chroma=bd, log2_ctb_size=6)
        e.upload_slot(0, params, synth.random_planes(W, H, bd, 1))
        stream = torch.cuda.Stream()
        for fmt, name in ((capi.EXPORT_YUV, "yuv"), (capi.EXPORT_RGB_BT709, "rgb")):
            bps = 1 if fmt != capi.EXPORT_YUV or bd == 8 else 2
            planes = [torch.empty((H, W) if fmt != capi.EXPORT_YUV or c == 0 else (H // 2, W // 2), dtype=torch.uint8 if bps == 1 else torch.int16,
                                  device="cuda") for c in range(3)]
            ex = capi.Export(0, 0, W, H, fmt, 0)
            ptrs, pitches = capi.PlaneArray(*[p.data_ptr() for p in planes]), capi.StrideArray(*[p.stride(0) * bps for p in planes])
            st = C.c_void_p(stream.cuda_stream)

            def run(n):
                for _ in range(n):
                    capi.check(e.lib.b200_engine_export_slot(e.handle, 0, C.byref(ex), ptrs, pitches, st), "export")

            run(20)
            stream.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            run(n_exports)
            e1.record(stream)
            e1.synchronize()
            us = 1000.0 * e0.elapsed_time(e1) / n_exports
            nbytes = export_bytes(bd, fmt != capi.EXPORT_YUV)
            out[f"{name}{bd}"] = {"us_per_picture": round(us, 2), "bytes": nbytes, "tb_per_s": round(nbytes / us / 1e6, 3),
                                  "share_of_3.35_tb_per_s": round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3)}
        e.sync()
        e.close()
    return out


def chain(steps, rounds):
    """bench.py's `value` loop (run_prepared, 32 pictures per step, two step variants) with and without an export per picture."""
    e = Engine(0)
    seq, key_slot, _ = bench.build_workload(W, H, 8)
    e.upload_slot(key_slot, seq[0].params, synth.random_planes(W, H, 8, 2))
    prepared = [e.prepare(p) for p in seq]
    stream = torch.cuda.ExternalStream(e.stream(), device=torch.device("cuda", 0))
    xs = torch.cuda.Stream()
    ring = [torch.empty((3, H, W), dtype=torch.uint8, device="cuda") for _ in range(8)]
    ex = capi.Export(0, 0, W, H, capi.EXPORT_RGB_BT709, 0)
    xst = C.c_void_p(xs.cuda_stream)
    counter = {"step": 0, "pic": 0}

    def step(export):
        v = counter["step"] % bench.STEP_VARIANTS
        counter["step"] += 1
        for h, p in zip(prepared[32 * v:32 * (v + 1)], seq[32 * v:32 * (v + 1)]):
            e.run_prepared(h)
            if export:
                o = ring[counter["pic"] % len(ring)]
                counter["pic"] += 1
                capi.check(e.lib.b200_engine_export_slot(e.handle, p.params.dst_slot, C.byref(ex), capi.PlaneArray(*[o[c].data_ptr() for c in range(3)]),
                                                         capi.StrideArray(W, W, W), xst), "export")

    def timed(export):
        e.sync()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            step(export)
        e.join()
        stream.wait_stream(xs)  # the exports are part of the step
        e1.record(stream)
        e1.synchronize()
        return 32 * steps / (e0.elapsed_time(e1) / 1000.0)

    for export in (False, True, False, True):  # warm-up: staging, renamed surfaces, the export kernel
        step(export)
    res = {"without_export": [], "with_rgb_export": []}
    for _ in range(rounds):
        res["without_export"].append(round(timed(False), 1))
        res["with_rgb_export"].append(round(timed(True), 1))
    e.sync()
    for h in prepared:
        e.free_prepared(h)
    e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--exports", type=int, default=200)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("export_bench.py measures on a CUDA device; none is available")
    line = {"card": card(), "micro_3840x2160": micro(a.exports), "chain_frames_per_s": chain(a.steps, a.rounds)}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
