#!/usr/bin/env python3
"""CPU-only analysis of the intra dependency DAG the engine's k_intra executes: tasks as the host planner forms them (the
small TUs of one plane inside a 16x16-luma / 8x8-chroma region, or one larger TU), level = 1 + max level of the neighbour
units a task may read (availability masks).  Prints the DAG depth (the number of dependent task latencies an intra picture
costs at least) and the tasks per level (how many warps can work at the same time).
The critical path weights each task with a task latency (defaults: the H100 costs below); it is printed with its makeup
(hops, large-TU hops, TUs per region hop), so the model can be re-run with newly measured costs.
Usage: python tools/dag_depth.py [synthetic | intra4k | intra1080] [--fixed-us F] [--tu-us T] [--large-us L]"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from libde265_b200 import synth  # noqa: E402


# per-task latencies of tools/trace_intra.py on an H100 SXM (400 W limit, 1980 MHz), bench's 4K I picture: producer done -> own
# done of a region task = 2.97 us + 0.296 us per TU, of a large TU (either plane) 3.3 us (hand-off 0.53 + ready..done 2.78)
COSTS = {"fixed_us": 2.97, "tu_us": 0.296, "large_us": 3.3}


def analyse(tus, W, H, name, fixed_us, tu_us, large_us):
    intra = (tus["flags"] & 1) != 0
    idx = np.nonzero(intra)[0]
    cur_key, cur_task, ntask = [None] * 3, [0] * 3, 0
    task_of = np.zeros(len(idx), np.int64)
    for k, i in enumerate(idx):
        t = tus[i]
        c, nT = int(t["cidx"]), 1 << int(t["log2_size"])
        G = 16 >> (1 if c else 0)
        key = ("L", i) if nT >= G else (int(t["y"]) // G, int(t["x"]) // G)
        if key != cur_key[c]:
            cur_key[c], cur_task[c] = key, ntask
            ntask += 1
        task_of[k] = cur_task[c]
    lvl = [np.zeros(((H >> (1 if c else 0)) // 4 + 2, (W >> (1 if c else 0)) // 4 + 2), np.int32) for c in range(3)]
    tl = np.zeros(ntask, np.int32)
    order = np.argsort(task_of, kind="stable")
    bounds = np.searchsorted(task_of[order], np.arange(ntask + 1))
    for t in range(ntask):
        ks = order[bounds[t]:bounds[t + 1]]
        best = 0
        for k in ks:
            tu = tus[idx[k]]
            c, x4, y4, n4, av = int(tu["cidx"]), int(tu["x"]) // 4, int(tu["y"]) // 4, (1 << int(tu["log2_size"])) // 4, int(tu["avail"])
            L = lvl[c]
            for g in range(2 * n4):
                if (av >> g) & 1 and x4 > 0:
                    best = max(best, L[y4 + g, x4 - 1])
                if (av >> (17 + g)) & 1 and y4 > 0:
                    best = max(best, L[y4 - 1, x4 + g])
            if (av >> 16) & 1 and x4 > 0 and y4 > 0:
                best = max(best, L[y4 - 1, x4 - 1])
        tl[t] = best + 1
        for k in ks:
            tu = tus[idx[k]]
            c, x4, y4, n4 = int(tu["cidx"]), int(tu["x"]) // 4, int(tu["y"]) // 4, (1 << int(tu["log2_size"])) // 4
            lvl[c][y4:y4 + n4, x4:x4 + n4] = tl[t]
    # weighted critical path: a task starts when the last producer of the units it may read is done
    fin = [np.zeros_like(lvl[c], dtype=np.float64) for c in range(3)]
    own = [np.full(lvl[c].shape, -1, np.int64) for c in range(3)]
    endt, pred, large = np.zeros(ntask), np.full(ntask, -1, np.int64), np.zeros(ntask, bool)
    for t in range(ntask):
        ks = order[bounds[t]:bounds[t + 1]]
        start = 0.0
        for k in ks:
            tu = tus[idx[k]]
            c, x4, y4, n4, av = int(tu["cidx"]), int(tu["x"]) // 4, int(tu["y"]) // 4, (1 << int(tu["log2_size"])) // 4, int(tu["avail"])
            cells = [(y4 + g, x4 - 1) for g in range(2 * n4) if (av >> g) & 1 and x4 > 0]
            cells += [(y4 - 1, x4 + g) for g in range(2 * n4) if (av >> (17 + g)) & 1 and y4 > 0]
            if (av >> 16) & 1 and x4 > 0 and y4 > 0:
                cells.append((y4 - 1, x4 - 1))
            for yx in cells:
                if fin[c][yx] > start and own[c][yx] != t:
                    start, pred[t] = fin[c][yx], own[c][yx]
        tu0 = tus[idx[ks[0]]]
        large[t] = len(ks) == 1 and (1 << int(tu0["log2_size"])) > 8
        endt[t] = start + (large_us if large[t] else fixed_us + tu_us * len(ks))
        for k in ks:
            tu = tus[idx[k]]
            c, x4, y4, n4 = int(tu["cidx"]), int(tu["x"]) // 4, int(tu["y"]) // 4, (1 << int(tu["log2_size"])) // 4
            fin[c][y4:y4 + n4, x4:x4 + n4] = endt[t]
            own[c][y4:y4 + n4, x4:x4 + n4] = t
    path, t = [], int(np.argmax(endt))
    while t >= 0:
        path.append(t)
        t = int(pred[t])
    path = np.array(path)
    ntu = bounds[path + 1] - bounds[path]
    reg = path[~large[path]]
    widths = np.bincount(tl)[1:]
    print(f"{name}: modelled critical path {endt.max() / 1000:.2f} ms (region task {fixed_us} us + {tu_us} us per TU, large TU {large_us} us)")
    print(f"{name}: critical path {len(path)} hops, {int(large[path].sum())} of them large TUs, region hops {len(reg)} with "
          f"{(bounds[reg + 1] - bounds[reg]).mean() if len(reg) else 0:.2f} TUs each ({int(ntu.sum())} TUs on the path)")
    print(f"{name}: {len(idx)} intra TUs in {ntask} tasks; DAG depth {int(tl.max())} levels; tasks per level mean {widths.mean():.1f}, "
          f"p10 {int(np.percentile(widths, 10))}, p50 {int(np.percentile(widths, 50))}, p90 {int(np.percentile(widths, 90))}, max {int(widths.max())}")


def main():
    args, costs = sys.argv[1:], dict(COSTS)
    for k in COSTS:
        opt = "--" + k.replace("_", "-")
        if opt in args:
            i = args.index(opt)
            costs[k] = float(args[i + 1])
            del args[i:i + 2]
    what = args[0] if args else "synthetic"
    if what == "synthetic":
        p = synth.make_picture(3840, 2160, "I", seed=1000)
        analyse(p.tus, 3840, 2160, "synthetic 4K I picture of bench.py (CTB 64)", **costs)
        return
    import oracle_lib
    from libde265_b200 import de265
    dec = de265.Decoder(oracle_lib.ref_path("libde265_hooked.so"))
    store = []

    def sink(pic, planes, strides):
        store.append((np.ctypeslib.as_array(C.cast(pic.tus, C.POINTER(C.c_uint8)), shape=(pic.n_tu * 24,)).view(synth.TU_DT).copy(), pic.params.width,
                      pic.params.height))
        return 0

    dec.attach(sink)
    dec.decode_stream(open(os.path.join(ROOT, "tests", "golden", what + ".h265"), "rb").read(), lambda img: None)
    dec.close()
    for n, (tus, W, H) in enumerate(store):
        analyse(tus, W, H, f"{what} picture {n}", **costs)


if __name__ == "__main__":
    main()
