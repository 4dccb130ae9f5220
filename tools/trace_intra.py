#!/usr/bin/env python3
"""Debug: per-task trace of k_intra for one synthetic 4K I picture (B200_TRACE_INTRA)."""
import os, sys, struct, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
path = os.path.join(ROOT, "gpurun_out", "intra_trace.bin")
if os.path.exists(path): os.remove(path)
os.environ["B200_TRACE_INTRA"] = path
from libde265_b200 import synth
from libde265_b200.engine import Engine
W, H = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (3840, 2160)
PT = sys.argv[3] if len(sys.argv) > 3 else "I"
p = synth.make_picture(W, H, PT, seed=1000, dst_slot=2, ref_slots=(0, 1)) if PT != "I" else synth.make_picture(W, H, "I", seed=1000)
eng = Engine(0)
if PT != "I":
    for s_ in (0, 1):
        eng.upload_slot(s_, p.params, synth.random_planes(W, H, 8, s_))
eng.enable_timing(True)
for _ in range(2):
    eng.submit(p); eng.sync()
print("stage ms:", eng.last_timing())
raw = open(path, "rb").read()
n = struct.unpack_from("<Q", raw, 0)[0]
# last record
rec = np.frombuffer(raw[-(8 * 4 * n):], dtype=np.uint64).reshape(n, 4)
t0 = rec[:, 0].astype(np.int64); wait = rec[:, 1].astype(np.int64); work = rec[:, 2].astype(np.int64); meta = rec[:, 3]
cnt = (meta & 0xff).astype(int); plane = ((meta >> 8) & 0xff).astype(int); lg = ((meta >> 16) & 0xff).astype(int)
print("claim time percentiles us (rel. to first):", [round(float(x) / 1e3, 1) for x in np.percentile(t0 - t0.min(), [10, 50, 90, 99, 100])])
end = t0 + ((wait + work) / 1.9).astype(np.int64)
print("end time percentiles us:", [round(float(x) / 1e3, 1) for x in np.percentile(end - t0.min(), [10, 50, 90, 99, 100])])
print("tasks", n, "TUs", cnt.sum(), "span ms (claim first..last)", (t0.max() - t0.min()) / 1e6)
clk = 1.9e3  # cycles per us (approx)
print("work us: mean %.2f p50 %.2f p90 %.2f p99 %.2f max %.2f" % (work.mean()/clk, np.percentile(work,50)/clk, np.percentile(work,90)/clk, np.percentile(work,99)/clk, work.max()/clk))
print("wait us: mean %.2f p50 %.2f p90 %.2f max %.2f" % (wait.mean()/clk, np.percentile(wait,50)/clk, np.percentile(wait,90)/clk, wait.max()/clk))
for c in range(3):
    for k in sorted(set(cnt[plane == c])):
        m = (plane == c) & (cnt == k)
        print(f" plane {c} TUs/task {k:2d}: n={m.sum():6d} work mean {work[m].mean()/clk:7.2f} us  (log2 of first TU: {np.bincount(lg[m]).tolist()})")
print("sum of work / 1e3:", work.sum() / clk / 1e3, "ms  => with", 132 * 3 * 8, "warps:", work.sum() / clk / 1e3 / (132 * 3 * 8), "ms")
# ticket-order view (tickets are in DAG-level order): when are the tasks of each slice of the ticket range claimed / finished?
idx = np.arange(n)
base = t0.min()
print("ticket range   claim us (p50,max)   end us (p50,max)   wait us mean   work us mean   TUs")
for a, b in [(i * n // 10, (i + 1) * n // 10) for i in range(10)]:
    sl = slice(a, b)
    print(f" {a:6d}-{b:6d}   {np.percentile(t0[sl]-base,50)/1e3:7.1f} {float((t0[sl]-base).max())/1e3:7.1f}   {np.percentile(end[sl]-base,50)/1e3:7.1f} {float((end[sl]-base).max())/1e3:7.1f}   "
          f"{wait[sl].mean()/clk:7.2f}   {work[sl].mean()/clk:7.2f}   {cnt[sl].sum()}")
late = np.argsort(end)[-12:]
print("last tasks to finish: ticket, claim us, wait us, work us, TUs, plane")
for i in late:
    print(f"  {i:6d} {float(t0[i]-base)/1e3:8.1f} {wait[i]/clk:8.1f} {work[i]/clk:8.1f} {cnt[i]:3d} {plane[i]}")
