"""ctypes access to the CPU oracle (oracle/libhevc_oracle.so) and, when present, the real reference
(oracle/_ref/*.so).  TEST INFRASTRUCTURE: imported by tests/, __graft_entry__.smoke() and the
cpu_baseline / --impl reference legs of bench.py only."""
import ctypes as C
import os
import subprocess

from libde265_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_SO = os.path.join(ORACLE_DIR, "libhevc_oracle.so")
REF_DIR = os.path.join(ORACLE_DIR, "_ref")

_orc = None


def build_oracle():
    subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "oracle"])


def oracle():
    global _orc
    if _orc is None:
        if not os.path.exists(ORACLE_SO):
            build_oracle()
        lib = C.CDLL(ORACLE_SO)
        vp = C.c_void_p
        lib.orc_create.restype = vp
        lib.orc_destroy.argtypes = [vp]
        lib.orc_destroy.restype = None
        lib.orc_reconstruct.argtypes = [vp, C.POINTER(capi.Picture)]
        lib.orc_fill_slot.argtypes = [vp, C.c_int, C.POINTER(capi.PicParams), C.c_int, C.c_int]
        lib.orc_upload_slot.argtypes = [vp, C.c_int, C.POINTER(capi.PicParams), capi.PlaneArray, capi.StrideArray]
        lib.orc_read_slot.argtypes = [vp, C.c_int, capi.PlaneArray, capi.StrideArray]
        _orc = lib
    return _orc


def ref_path(name):
    p = os.path.join(REF_DIR, name)
    return p if os.path.exists(p) else None


class Oracle:
    """Python wrapper of the CPU restatement's picture replay (orc_*)."""

    def __init__(self):
        self.lib = oracle()
        self.ctx = self.lib.orc_create()

    def close(self):
        if self.ctx:
            self.lib.orc_destroy(self.ctx)
            self.ctx = None

    def reconstruct(self, pic):
        cp = getattr(pic, "c", pic)
        rc = self.lib.orc_reconstruct(self.ctx, C.byref(cp))
        if rc:
            raise RuntimeError(f"orc_reconstruct failed: {rc}")

    def upload_slot(self, slot, params, planes):
        pa = capi.PlaneArray(*[p.ctypes.data for p in planes])
        sa = capi.StrideArray(*[p.strides[0] for p in planes])
        assert self.lib.orc_upload_slot(self.ctx, slot, C.byref(params), pa, sa) == 0

    def fill_slot(self, slot, params, vy, vc):
        assert self.lib.orc_fill_slot(self.ctx, slot, C.byref(params), vy, vc) == 0

    def read_slot(self, slot, params):
        import numpy as np
        dt = np.uint16 if params.bit_depth_luma > 8 else np.uint8
        shapes = [(params.height, params.width)]
        if params.chroma_format_idc:
            shapes += [(params.height // 2, params.width // 2)] * 2
        out = [np.empty(s, dt) for s in shapes]
        ptrs = [o.ctypes.data for o in out] + [None] * (3 - len(out))
        strides = [o.strides[0] for o in out] + [0] * (3 - len(out))
        assert self.lib.orc_read_slot(self.ctx, slot, capi.PlaneArray(*ptrs), capi.StrideArray(*strides)) == 0
        return out


REPLAY_SO = os.path.join(REF_DIR, "libref_replay.so")
_rr = None


def ref_replay_lib():
    """oracle/_ref/libref_replay.so: b200 records replayed through the REFERENCE's own reconstruction functions
    (oracle/ref_replay.cc); None when oracle/_ref was not built / shipped."""
    global _rr
    if _rr is None and os.path.exists(REPLAY_SO):
        lib = C.CDLL(REPLAY_SO)
        vp = C.c_void_p
        lib.rr_create.restype = vp
        lib.rr_create.argtypes = [C.c_int]
        lib.rr_destroy.argtypes = [vp]
        lib.rr_destroy.restype = None
        lib.rr_reconstruct.argtypes = [vp, C.POINTER(capi.Picture)]
        lib.rr_fill_slot.argtypes = [vp, C.c_int, C.POINTER(capi.PicParams), C.c_int, C.c_int]
        lib.rr_upload_slot.argtypes = [vp, C.c_int, C.POINTER(capi.PicParams), capi.PlaneArray, capi.StrideArray]
        lib.rr_read_slot.argtypes = [vp, C.c_int, capi.PlaneArray, capi.StrideArray]
        if hasattr(lib, "rr_set_options"):  # absent from a library built from an older oracle/ref_replay.cc
            lib.rr_set_options.argtypes = [vp, C.c_int, C.c_int]
            lib.rr_avail_mismatch.argtypes = [vp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        _rr = lib
    return _rr


def ref_replay_has_options():
    """True when the replay library takes the constrained_intra / check_avail options (rr_set_options).  A library shipped
    prebuilt from an older oracle/ref_replay.cc lacks them: tests that need them then rely on the stored digests or skip."""
    lib = ref_replay_lib()
    return lib is not None and hasattr(lib, "rr_set_options")


def ref_replay_handles_ctb_change():
    """True when the replay library reallocates a slot's image on a CTB-size change (rr_handles_ctb_change).  A library shipped
    prebuilt from an older oracle/ref_replay.cc corrupts its heap when a name is rewritten with a smaller CTB: tests that
    need it then rely on the stored digests."""
    lib = ref_replay_lib()
    return lib is not None and hasattr(lib, "rr_handles_ctb_change")


class RefReplay(Oracle):
    """Same interface as Oracle, executed by the reference's own code (simd=True: the table de265_acceleration_AUTO selects,
    i.e. SSE4.1 + AVX2 + AVX-512 where the host has them; False: the scalar fallback table).
    constrained_intra: the reference derives intra availability with constrained_intra_pred_flag set, from the records'
    prediction modes.  check_avail: reconstruct() raises AvailMismatch at the first intra TU whose record mask differs from
    the mask the reference derives."""

    def __init__(self, simd=True, constrained_intra=False, check_avail=False):
        lib = ref_replay_lib()
        if lib is None:
            raise RuntimeError("oracle/_ref/libref_replay.so not built (make -C oracle ref; needs /root/reference)")

        class _Shim:  # present the rr_* entry points under the orc_* names the base class calls
            orc_destroy, orc_reconstruct, orc_upload_slot, orc_fill_slot, orc_read_slot = (lib.rr_destroy, lib.rr_reconstruct, lib.rr_upload_slot,
                                                                                           lib.rr_fill_slot, lib.rr_read_slot)
        self.lib, self.rr = _Shim, lib
        self.options = ref_replay_has_options()
        if (constrained_intra or check_avail) and not self.options:
            raise RuntimeError(f"{REPLAY_SO} predates rr_set_options: rebuild it (make -C oracle ref; needs /root/reference)")
        self.ctx = lib.rr_create(1 if simd else 0)
        if self.options:
            assert lib.rr_set_options(self.ctx, int(constrained_intra), int(check_avail)) == 0

    def reconstruct(self, pic):
        cp = getattr(pic, "c", pic)
        rc = self.rr.rr_reconstruct(self.ctx, C.byref(cp))
        i, rec, ref = C.c_uint32(), C.c_uint64(), C.c_uint64()
        if self.options and self.rr.rr_avail_mismatch(self.ctx, C.byref(i), C.byref(rec), C.byref(ref)):
            t = cp.tus[i.value]
            raise AvailMismatch(f"TU {i.value} (x={t.x}, y={t.y}, {1 << t.log2_size}x{1 << t.log2_size}, cidx {t.cidx}): record avail "
                                f"{rec.value:#x} != reference {ref.value:#x}")
        if rc:
            raise RuntimeError(f"rr_reconstruct failed: {rc}")


class AvailMismatch(AssertionError):
    """An intra TU's record availability mask differs from the one the reference derives."""
