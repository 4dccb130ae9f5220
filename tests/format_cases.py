"""Sequences that change format mid-stream, as one shared case list: a new picture size, chroma format, bit depth or CTB size
between pictures decoded by one engine, with P / B pictures whose reference lists mix slots of the current format with slots of
every other kind.  test_cpu_format_switch.py pins the oracle to the reference on every case and test_gpu_format_switch.py the
engine to the oracle.

The reference's rule for a reference picture of another format (motion.cc:385-405): a slot whose width, height, chroma format,
luma or chroma bit depth differs from the picture's counts as missing, and the prediction from it is mid-grey.  A slot that
differs only in its CTB size is an ordinary reference.

Every picture writes every one of its samples (its PUs and intra TUs tile the picture; test_cpu_format_switch.py checks it).
That matters here: a name that is rewritten in another format keeps its old samples in the engine when the bytes per sample
stay the same (9 <-> 10 <-> 12 bit), while the reference and the oracle start from a zero-filled picture; only samples that no
record writes could show the difference, and only a malformed stream has such samples.

Every case carries the checks that prove its switches and references are present in the generated records
(test_cpu_format_switch.py::test_every_case_reaches_its_switches)."""
import functools
from collections import namedtuple

import numpy as np

from libde265_b200 import capi, synth

Fmt = namedtuple("Fmt", "W H bd bdc cf ctb")
Case = namedtuple("Case", "id steps checks")


def fmt(W, H, bd=8, bdc=None, cf=1, ctb=6):
    return Fmt(W, H, bd, bd if bdc is None else bdc, cf, ctb)


def bps(bd):
    return 2 if bd > 8 else 1


def ref_kind(cur, ref):
    """How the format of a reference slot relates to the picture's: 'size', 'chroma' (chroma format), 'bytes' (bytes per
    sample of a plane), 'depth' (a bit depth, same bytes per sample) -- each a mismatch, the first that applies -- or 'ctb'
    (only the CTB size differs) and 'same', which are ordinary references."""
    if (cur.W, cur.H) != (ref.W, ref.H):
        return "size"
    if cur.cf != ref.cf:
        return "chroma"
    if (bps(cur.bd), bps(cur.bdc)) != (bps(ref.bd), bps(ref.bdc)):
        return "bytes"
    if (cur.bd, cur.bdc) != (ref.bd, ref.bdc):
        return "depth"
    return "ctb" if cur.ctb != ref.ctb else "same"


MISMATCH = ("size", "chroma", "bytes", "depth")


@functools.lru_cache(maxsize=None)
def make_sequence(case_id):
    """The case's pictures in decode order (cached: the records are only read)."""
    c = BY_ID[case_id]
    seed0 = 800 + 40 * CASE_IDS.index(case_id)
    return [synth.make_picture(f.W, f.H, t, seed=seed0 + i, dst_slot=dst, ref_slots=refs, bit_depth=f.bd, bit_depth_chroma=f.bdc,
                               chroma_format_idc=f.cf, log2_ctb=f.ctb)
            for i, (f, t, dst, refs) in enumerate(c.steps)]


def slot_formats(case):
    """([{slot: Fmt of the picture it holds} just before each step], {slot: Fmt} at the end)."""
    held, out = {}, []
    for f, _, dst, _ in case.steps:
        out.append(dict(held))
        held[dst] = f
    return out, held


def pu_ref_kinds(case, pics):
    """[{kind: number of PU lists that predict from a slot of that kind}] per picture (slots never written are left out)."""
    before, _ = slot_formats(case)
    out = []
    for (f, _, _, _), held, p in zip(case.steps, before, pics):
        cnt = {}
        for pu in p.pus:
            for l in range(2):
                s = int(pu["ref_slot"][l])
                if pu["flags"] & (1 << l) and s in held:
                    k = ref_kind(f, held[s])
                    cnt[k] = cnt.get(k, 0) + 1
        out.append(cnt)
    return out


def mismatched_ref_slots(case, i):
    """The slots picture i references that hold a picture of another format."""
    held = slot_formats(case)[0][i]
    f, _, _, refs = case.steps[i]
    return sorted(s for s in refs if s in held and ref_kind(f, held[s]) in MISMATCH)


# ---- checks: (description, predicate over (case, pictures)) ----
def refs_of(*kinds):
    def f(case, pics):
        seen = {}
        for cnt in pu_ref_kinds(case, pics):
            for k, v in cnt.items():
                seen[k] = seen.get(k, 0) + v
        return all(seen.get(k, 0) > 0 for k in kinds)
    return f"PUs that predict from slots of kind {kinds}", f


def mixed_list(*kinds):
    """One picture whose PUs predict from slots of every listed kind."""
    def f(case, pics):
        return any(all(cnt.get(k, 0) > 0 for k in kinds) for cnt in pu_ref_kinds(case, pics))
    return f"one picture that predicts from slots of every kind {kinds}", f


def switches(*what):
    """Consecutive pictures that change each listed format field (W, H, bd, bdc, cf, ctb, bytes)."""
    def f(case, pics):
        seen = set()
        for (a, *_), (b, *_) in zip(case.steps, case.steps[1:]):
            for k in Fmt._fields:
                if getattr(a, k) != getattr(b, k):
                    seen.add(k)
            if (bps(a.bd), bps(a.bdc)) != (bps(b.bd), bps(b.bdc)):
                seen.add("bytes")
        return set(what) <= seen
    return f"format switches of {what}", f


def same_bytes_only():
    """Every switch keeps the size, chroma format and bytes per sample: the engine neither drains nor reallocates."""
    def f(case, pics):
        return all((a.W, a.H, a.cf, bps(a.bd), bps(a.bdc)) == (b.W, b.H, b.cf, bps(b.bd), bps(b.bdc)) for (a, *_), (b, *_) in zip(case.steps, case.steps[1:]))
    return "no switch changes the size, chroma format or bytes per sample", f


def rewrites_ctb(case):
    """Whether a picture writes a name that holds a picture of the same format but another CTB size."""
    before, _ = slot_formats(case)
    return any(dst in held and ref_kind(f, held[dst]) == "ctb" for (f, _, dst, _), held in zip(case.steps, before))


def sao_kernels():
    """8-bit SAO pictures at CTB 64 / 32 and at CTB 16: the engine runs k_sao8 on the first, k_sao on the second."""
    def f(case, pics):
        kinds = [p.params.log2_ctb_size >= 5 for p in pics if p.params.bit_depth_luma == 8 and p.params.flags & capi.PIC_SAO_ENABLED]
        return True in kinds and False in kinds and any(a != b for a, b in zip(kinds, kinds[1:]))
    return "8-bit SAO pictures that switch between CTB >= 32 and CTB 16", f


def rewrites_name(kind):
    """A picture writes a name that holds a picture of another format of this kind."""
    def f(case, pics):
        before, _ = slot_formats(case)
        return any(dst in held and ref_kind(fm, held[dst]) == kind for (fm, _, dst, _), held in zip(case.steps, before))
    return f"a picture rewrites a name that holds a picture of kind {kind!r}", f


def first_format_survives():
    """The first format comes back after the others, and its pictures reference names that were written before the first switch
    and that still hold those pictures at the end (the tests read every name back at the end)."""
    def f(case, pics):
        first = case.steps[0][0]
        n_first = next(i for i, (fm, *_) in enumerate(case.steps) if fm != first)
        old = {dst for _, _, dst, _ in case.steps[:n_first]} - {dst for _, _, dst, _ in case.steps[n_first:]}
        back = [i for i, (fm, *_) in enumerate(case.steps) if i > n_first and fm == first]
        kinds = pu_ref_kinds(case, pics)
        return bool(back) and any(set(case.steps[i][3]) & old and kinds[i].get("same") for i in back)
    return "names of the first format survive the other formats and are referenced when it comes back", f


# ---- the case list ----
A = fmt(416, 240)
HD = fmt(1920, 1080)
R = fmt(200, 136)
S8, S10 = fmt(320, 192), fmt(320, 192, 10)
D9, D10 = fmt(320, 192, 9), fmt(320, 192, 10)
D10_12, D12_9 = fmt(256, 128, 10, 12), fmt(256, 128, 12, 9)
C420, C400 = fmt(256, 128), fmt(256, 128, cf=0)
T64, T16, T32 = fmt(208, 120, ctb=6), fmt(208, 120, ctb=4), fmt(208, 120, ctb=5)
X10 = fmt(192, 128, 10)
X8 = fmt(192, 128, 8)
UHD8, HD10 = fmt(3840, 2160), fmt(1920, 1080, 10)

CASES = [
    # 416x240 -> 1920x1080 -> 200x136 -> 416x240: the last format writes names 2 and 3 (3 held the 1080p picture) while names 0 and
    # 1 still hold the pictures of the start, which it references
    Case("size", [(A, "I", 0, ()), (A, "P", 1, (0,)), (A, "B", 2, (0, 1)),
                  (HD, "I", 3, ()), (HD, "P", 4, (3, 0, 1)),
                  (R, "I", 5, ()), (R, "B", 6, (5, 3, 1)),
                  (A, "P", 7, (0, 1, 5)), (A, "B", 2, (0, 7, 4, 6)), (A, "B", 3, (0, 1, 2))],
         [switches("W", "H"), refs_of("same", "size"), rewrites_name("size"), first_format_survives()]),
    # 8 -> 10 -> 8 bit at one size: every switch reallocates, the TMA tensor maps go away and come back
    Case("bytes_8_10_8", [(S8, "I", 0, ()), (S8, "P", 1, (0,)),
                          (S10, "I", 2, ()), (S10, "P", 3, (2, 0)), (S10, "B", 0, (2, 3, 1)),
                          (S8, "P", 4, (1, 0, 3)), (S8, "B", 2, (4, 1, 0))],
         [switches("bd", "bytes"), refs_of("same", "bytes"), rewrites_name("bytes"), mixed_list("same", "bytes")]),
    # 9/9 <-> 10/10: no drain and no reallocation, the surfaces are relabelled, and references across the switch predict grey
    Case("depth_9_10", [(D9, "I", 0, ()), (D9, "P", 1, (0,)),
                        (D10, "I", 2, ()), (D10, "B", 3, (2, 0, 1)), (D10, "B", 0, (2, 3, 1)),
                        (D9, "B", 4, (1, 0, 2)), (D9, "B", 2, (4, 1, 3))],
         [same_bytes_only(), switches("bd", "bdc"), refs_of("same", "depth"), rewrites_name("depth"), mixed_list("same", "depth")]),
    # 10/12 <-> 12/9: luma and chroma depths both change, bytes per sample do not
    Case("depth_10_12_to_12_9", [(D10_12, "I", 0, ()), (D10_12, "P", 1, (0,)),
                                 (D12_9, "I", 2, ()), (D12_9, "B", 3, (2, 0, 1)), (D12_9, "P", 0, (3, 1)),
                                 (D10_12, "B", 4, (1, 0, 2)), (D10_12, "B", 2, (4, 1, 3))],
         [same_bytes_only(), switches("bd", "bdc"), refs_of("same", "depth"), rewrites_name("depth"), mixed_list("same", "depth")]),
    # 4:2:0 <-> 4:0:0 at one size
    Case("chroma_420_400", [(C420, "I", 0, ()), (C420, "P", 1, (0,)),
                            (C400, "I", 2, ()), (C400, "B", 3, (2, 0, 1)), (C400, "P", 0, (2, 3)),
                            (C420, "B", 4, (1, 0, 3)), (C420, "B", 2, (4, 1, 0))],
         [switches("cf"), refs_of("same", "chroma"), rewrites_name("chroma"), mixed_list("same", "chroma")]),
    # CTB 64 -> 16 -> 32 at one size: the pool keeps its format (no drain), the per-stream sync buffer grows, SAO switches from
    # k_sao8 to k_sao and back; references across CTB sizes are ordinary references
    Case("ctb_64_16_32", [(T64, "I", 0, ()), (T64, "P", 1, (0,)),
                          (T16, "B", 2, (0, 1)), (T16, "I", 3, ()),
                          (T32, "B", 4, (2, 3, 1)), (T32, "P", 0, (4, 1))],
         [switches("ctb"), refs_of("same", "ctb"), sao_kernels(), mixed_list("same", "ctb")]),
    # one 10-bit B picture predicting from the current format and from a slot of each other kind at once
    Case("mixed_refs10", [(X10, "I", 0, ()), (fmt(256, 128, 10), "I", 1, ()), (X8, "I", 2, ()), (fmt(192, 128, 9), "I", 3, ()),
                          (fmt(192, 128, 10, cf=0), "I", 4, ()), (fmt(192, 128, 10, 12), "I", 5, ()), (fmt(192, 128, 10, ctb=5), "I", 6, ()),
                          (X10, "B", 7, (0, 1, 2, 3, 4, 5, 6)), (X10, "P", 1, (7, 2, 3, 5))],
         [mixed_list("same", "ctb", "size", "bytes", "depth", "chroma"), rewrites_name("size")]),
    # the same for an 8-bit picture (the TMA-staged MC kernel): there is no other depth with one byte per sample
    Case("mixed_refs8", [(X8, "I", 0, ()), (fmt(256, 128), "I", 1, ()), (X10, "I", 2, ()), (fmt(192, 128, cf=0), "I", 3, ()),
                         (fmt(192, 128, ctb=4), "I", 4, ()),
                         (X8, "B", 5, (0, 1, 2, 3, 4)), (X8, "P", 2, (5, 1, 3))],
         [mixed_list("same", "ctb", "size", "bytes", "chroma"), rewrites_name("bytes")]),
    # full size: 3840x2160 8-bit -> 1920x1080 10-bit -> 3840x2160 8-bit
    Case("large", [(UHD8, "I", 0, ()), (HD10, "P", 1, (0,)), (UHD8, "B", 2, (0, 1))],
         [switches("W", "H", "bytes"), refs_of("same", "size")]),
]
CASE_IDS = [c.id for c in CASES]
BY_ID = {c.id: c for c in CASES}


def luma_coverage(pic):
    """Per 4x4 luma block: how many PU or intra-TU records write it."""
    W, H = pic.params.width, pic.params.height
    m = np.zeros(((H + 3) // 4, (W + 3) // 4), np.int32)
    for pu in pic.pus:
        m[pu["y"] // 4:(pu["y"] + pu["h"]) // 4, pu["x"] // 4:(pu["x"] + pu["w"]) // 4] += 1
    t = pic.tus[(pic.tus["cidx"] == 0) & ((pic.tus["flags"] & (capi.TU_INTRA | capi.TU_PCM)) != 0)]
    for tu in t:
        n = 1 << int(tu["log2_size"])
        m[tu["y"] // 4:(tu["y"] + n) // 4, tu["x"] // 4:(tu["x"] + n) // 4] += 1
    return m
