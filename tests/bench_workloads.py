"""The pictures bench.py decodes, built by bench.py's own functions with rank 0's seeds exactly as bench.run_config uses them,
and the ORACLE CHAIN: the CPU oracle decoding them in bench order (step s replays the records of variant s % 2), recording the
md5 of every picture and the whole DPB at the end.  Shared by test_cpu_bench_workload_oracle.py (which pins the chain to the
reference) and test_gpu_bench_workload.py (which holds every path bench.py times to it)."""
import hashlib
import os
import sys
from dataclasses import dataclass

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import oracle_lib  # noqa: E402
from libde265_b200 import shard, synth  # noqa: E402

PER_STEP = 32


def md5_planes(planes):
    return hashlib.md5(b"".join(p.tobytes() for p in planes)).hexdigest()


@dataclass
class Workload:
    name: str
    seq: list        # 2 x 32 pictures in decode order (bench's variants)
    key_slot: int    # slot of the POC 0 reference (None: all-intra)
    ref0: list       # planes uploaded to key_slot before the first step (None: all-intra)


def build(name, bench_mod=bench):
    """The workload of bench config `name` for rank 0 (bench_mod: bench reloaded under another DPB policy)."""
    cfg = bench_mod.CONFIGS[name]
    w, h, bd = cfg["width"], cfg["height"], cfg["bd"]
    if cfg["kind"] == "ra":  # the headline config starts at the rank's stream seed, the other random-access leg 7000 later
        seq, key_slot, _ = bench_mod.build_workload(w, h, bd, seed0=shard.stream_seed(0) + (0 if name == "main_ra_4k" else 7000))
        return Workload(name, seq, key_slot, synth.random_planes(w, h, bd, shard.reference_seed(0)))
    seq, _, _ = bench_mod.build_intra_workload(w, h, bd, seed0=shard.stream_seed(0) + 3000)
    return Workload(name, seq, None, None)


def schedule(wl, steps):
    """(step, index in the step, index into wl.seq) in the order bench.step_resident issues the pictures."""
    for s in range(steps):
        v = s % bench.STEP_VARIANTS
        for i in range(PER_STEP):
            yield s, i, PER_STEP * v + i


def describe(wl, steps, n):
    """Step, index, POC, kind and slot of the n-th picture of the schedule (for failure messages)."""
    s, i, j = list(schedule(wl, steps))[n]
    p = wl.seq[j]
    pred = p.pus["flags"] & 3 if len(p.pus) else np.zeros(0, np.uint8)
    kind = "B" if (pred & 2).any() else "P" if pred.any() else "I"
    return f"step {s} index {i} (POC {p.params.poc}, {kind}, slot {p.params.dst_slot})"


class Chain:
    """The oracle decoding `steps` steps of the workload: pic_md5[n] = md5 of the n-th picture right after it was decoded,
    dpb[slot] = md5 of what every slot holds at the end.  `stop` = decode only up to picture n of the schedule.
    The oracle keeps the final state (self.orc) until close()."""

    def __init__(self, wl, steps, stop=None):
        self.wl, self.steps = wl, steps
        self.orc = oracle_lib.Oracle()
        if wl.ref0 is not None:
            self.orc.upload_slot(wl.key_slot, wl.seq[0].params, wl.ref0)
        self.pic_md5, self.last = [], None
        held = {} if wl.key_slot is None else {wl.key_slot: wl.seq[0].params}
        for n, (_, _, j) in enumerate(schedule(wl, steps)):
            p = wl.seq[j]
            self.orc.reconstruct(p)
            self.last = self.orc.read_slot(p.params.dst_slot, p.params)
            self.pic_md5.append(md5_planes(self.last))
            held[p.params.dst_slot] = p.params
            if n == stop:
                break
        self.dpb = {s: md5_planes(self.orc.read_slot(s, prm)) for s, prm in sorted(held.items())}
        self.params_of = held

    def close(self):
        self.orc.close()


def oracle_picture(wl, steps, n):
    """The oracle's planes of the n-th picture of the schedule (re-runs the chain up to it)."""
    c = Chain(wl, steps, stop=n)
    c.close()
    return c.last


def oracle_slot(wl, steps, slot):
    """The oracle's planes of `slot` at the end of `steps` steps."""
    c = Chain(wl, steps)
    out = c.orc.read_slot(slot, c.params_of[slot])
    c.close()
    return out


def records_digest(pics):
    """md5 over everything a picture record carries (parameters and every array), in decode order."""
    md = hashlib.md5()
    for p in pics:
        md.update(bytes(p.params))
        for name in ("pus", "weights", "tus", "coeffs", "slices", "ctbs", "bs_map", "qp_map", "nofilt_map"):
            a = getattr(p, name)
            md.update(name.encode())
            if a is not None:
                md.update(np.ascontiguousarray(a).tobytes())
    return md.hexdigest()
