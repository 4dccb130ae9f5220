"""ctypes mirror of include/b200hevc.h (the C-ABI drop-in boundary).

The product path is the CUDA library ``libb200hevc.so`` built in-tree by ``__graft_entry__.build()``.
There is no CPU fallback: ``load()`` raises if the library is missing and engine creation raises if
no CUDA device is present.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200hevc.so")

B200_MAX_SLOTS = 32

# --- flags (b200hevc.h) ---
PIC_SAO_ENABLED = 0x0001
PIC_STRONG_INTRA_SMOOTHING = 0x0002
PIC_PCM_LF_DISABLE = 0x0004
PIC_LF_ACROSS_TILES = 0x0008
PIC_INTRA_SMOOTHING_OFF = 0x0010
PIC_SKIP_DEBLOCK = 0x0020
PIC_SKIP_SAO = 0x0040
PIC_SCALING_LIST = 0x0080
PIC_RECORDS_PINNED = 0x0100  # record arrays page-locked and stable until the picture is done: uploaded without the staging copy

STAGE_ALL, STAGE_INTER_PRED, STAGE_RECON, STAGE_DEBLOCK = 0, 1, 2, 3

PU_PRED_L0, PU_PRED_L1, PU_WEIGHTED = 1, 2, 4

TU_INTRA = 0x0001
TU_CBF = 0x0002
TU_TSKIP = 0x0004
TU_BYPASS = 0x0008
TU_RDPCM_H = 0x0010
TU_RDPCM_V = 0x0020
TU_DST = 0x0040
TU_NO_BOUNDARY_FILTER = 0x0080
TU_PCM = 0x0100
TU_ROTATE = 0x0200
TU_SCALING_LIST = 0x0400
TU_INTER_MATRIX = 0x0800

AVAIL_CORNER_BIT = 16
AVAIL_TOP_BIT0 = 17

SLICE_DEBLOCK_DISABLED, SLICE_LF_ACROSS_SLICES, SLICE_SAO_LUMA, SLICE_SAO_CHROMA = 1, 2, 4, 8

SCALING_FACTOR_BYTES = 6 * 16 + 6 * 64 + 6 * 256 + 6 * 1024


class PicParams(C.Structure):
    _fields_ = [
        ("width", C.c_uint16), ("height", C.c_uint16),
        ("chroma_format_idc", C.c_uint8), ("bit_depth_luma", C.c_uint8), ("bit_depth_chroma", C.c_uint8),
        ("log2_ctb_size", C.c_uint8), ("flags", C.c_uint16),
        ("pps_cb_qp_offset", C.c_int8), ("pps_cr_qp_offset", C.c_int8),
        ("dst_slot", C.c_uint8), ("stop_after_stage", C.c_uint8), ("reserved", C.c_uint8 * 2),
        ("poc", C.c_int32),
    ]


class PU(C.Structure):
    _fields_ = [
        ("x", C.c_uint16), ("y", C.c_uint16), ("w", C.c_uint8), ("h", C.c_uint8),
        ("flags", C.c_uint8), ("reserved", C.c_uint8), ("ref_slot", C.c_int8 * 2), ("wt_idx", C.c_uint16),
        ("mv", (C.c_int16 * 2) * 2), ("pad", C.c_uint32),
    ]


class WeightEntry(C.Structure):
    _fields_ = [("w", (C.c_int16 * 3) * 2), ("o", (C.c_int16 * 3) * 2), ("log2wd_luma", C.c_uint8),
                ("log2wd_chroma", C.c_uint8), ("pad", C.c_uint8 * 2)]


class TU(C.Structure):
    _fields_ = [
        ("x", C.c_uint16), ("y", C.c_uint16), ("log2_size", C.c_uint8), ("cidx", C.c_uint8), ("flags", C.c_uint16),
        ("intra_mode", C.c_uint8), ("qp", C.c_uint8), ("n_coeff", C.c_uint16), ("coeff_off", C.c_uint32),
        ("avail", C.c_uint64),
    ]


class Coeff(C.Structure):
    _fields_ = [("pos", C.c_uint16), ("level", C.c_int16)]


class SliceInfo(C.Structure):
    _fields_ = [("slice_addr_rs", C.c_uint32), ("beta_offset", C.c_int8), ("tc_offset", C.c_int8),
                ("flags", C.c_uint8), ("pad", C.c_uint8)]


class CtbInfo(C.Structure):
    _fields_ = [("slice_idx", C.c_uint16), ("tile_id", C.c_uint16), ("sao_type", C.c_uint8), ("sao_eo_class", C.c_uint8),
                ("sao_band_pos", C.c_uint8 * 3), ("sao_offset", (C.c_int8 * 4) * 3), ("pad", C.c_uint8 * 3)]


EXPORT_YUV, EXPORT_RGB_BT601, EXPORT_RGB_BT709, EXPORT_RGB_BT2020 = 0, 1, 2, 3
EXPORT_FULL_RANGE = 0x01


class Export(C.Structure):
    """b200_export: crop window in luma samples, B200_EXPORT_* format, flags."""
    _fields_ = [("x", C.c_uint16), ("y", C.c_uint16), ("width", C.c_uint16), ("height", C.c_uint16),
                ("format", C.c_uint8), ("flags", C.c_uint8), ("reserved", C.c_uint8 * 2)]


class Picture(C.Structure):
    _fields_ = [
        ("params", PicParams),
        ("n_pu", C.c_uint32), ("n_weights", C.c_uint32), ("n_tu", C.c_uint32), ("n_coeff", C.c_uint32), ("n_slices", C.c_uint32),
        ("pus", C.POINTER(PU)), ("weights", C.POINTER(WeightEntry)), ("tus", C.POINTER(TU)), ("coeffs", C.POINTER(Coeff)),
        ("slices", C.POINTER(SliceInfo)), ("ctbs", C.POINTER(CtbInfo)),
        ("bs_map", C.POINTER(C.c_uint8)), ("qp_map", C.POINTER(C.c_int8)), ("nofilt_map", C.POINTER(C.c_uint8)),
        ("scaling_factors", C.POINTER(C.c_uint8)),
    ]


assert C.sizeof(PicParams) == 20 and C.sizeof(PU) == 24 and C.sizeof(WeightEntry) == 28
assert C.sizeof(TU) == 24 and C.sizeof(Coeff) == 4 and C.sizeof(SliceInfo) == 8 and C.sizeof(CtbInfo) == 24
assert C.sizeof(Export) == 12

PlaneArray = C.c_void_p * 3
StrideArray = C.c_size_t * 3

# every symbol include/b200hevc.h declares (tests check that the built library exports them all)
EXPORTS = [
    "b200_engine_create", "b200_engine_destroy", "b200_engine_submit_picture", "b200_engine_fill_slot",
    "b200_engine_upload_slot", "b200_engine_read_slot", "b200_engine_read_slot_async", "b200_engine_sync",
    "b200_engine_slot_device_planes", "b200_engine_enable_timing", "b200_engine_last_timing",
    "b200_engine_launch_count", "b200_engine_stream", "b200_engine_prepare_picture", "b200_engine_run_prepared",
    "b200_engine_free_prepared", "b200_engine_timing_sum", "b200_engine_set_streams", "b200_engine_join", "b200_plan_picture_host", "b200_last_error",
    "b200_engine_wait_slot", "b200_host_alloc", "b200_host_free", "b200_engine_submit_picture_async", "b200_engine_flush", "b200_engine_last_ticket", "b200_engine_wait_ticket",
    "b200_engine_export_slot",
    "b200_abi_version",
    "b200_rec_create", "b200_rec_destroy", "b200_rec_begin_picture", "b200_rec_add_slice", "b200_rec_add_weights",
    "b200_rec_add_pu", "b200_rec_add_tu", "b200_rec_set_ctb", "b200_rec_bs_map", "b200_rec_qp_map",
    "b200_rec_nofilt_map", "b200_rec_set_scaling_factors", "b200_rec_end_picture",
    "b200_picture_serialized_size", "b200_picture_serialize", "b200_picture_deserialize",
    # include/b200hevc_dsp.h (boundary B1)
    "b200_dsp_create", "b200_dsp_destroy", "b200_dsp_run_batch",
]

(DSP_QPEL, DSP_EPEL, DSP_PRED_UNI, DSP_PRED_AVG, DSP_PRED_WEIGHTED, DSP_PRED_WEIGHTED_BI, DSP_TRANSFORM_ADD, DSP_DST_ADD, DSP_INTRA_DC,
 DSP_INTRA_PLANAR, DSP_INTRA_ANGULAR, DSP_DEBLOCK_LUMA, DSP_DEBLOCK_CHROMA) = range(1, 14)


class DspCmd(C.Structure):
    """b200_dsp_cmd (include/b200hevc_dsp.h)."""
    _fields_ = [("op", C.c_int32), ("bit_depth", C.c_int32), ("dst", C.c_void_p), ("dststride", C.c_ssize_t), ("src", C.c_void_p),
                ("src2", C.c_void_p), ("srcstride", C.c_ssize_t), ("w", C.c_int32), ("h", C.c_int32), ("a", C.c_int32 * 8)]


_lib = None


# The engine pipelines pictures over up to 12 CUDA streams.  With the default of 8 hardware connections, streams share a
# connection and a stream that waits for an event (a B picture waiting for its reference) holds up an unrelated stream behind
# it (measured: the next intra picture started only when the previous one had finished).  Must be set before CUDA initialises.
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")


def load(path=None):
    """Load libb200hevc.so and declare prototypes.  Raises OSError when it has not been built."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or os.environ.get("B200_LIB") or LIB_PATH  # B200_LIB: an experiment build of the same sources (build.py)
    if not os.path.exists(p):
        raise OSError(f"{p} not found: run `python -c 'import __graft_entry__ as g; g.build()'` first "
                      "(there is no CPU fallback for the reconstruction engine)")
    lib = C.CDLL(p)
    vp = C.c_void_p
    lib.b200_engine_create.argtypes = [C.POINTER(vp), C.c_int]
    lib.b200_engine_destroy.argtypes = [vp]
    lib.b200_engine_destroy.restype = None
    lib.b200_engine_submit_picture.argtypes = [vp, C.POINTER(Picture)]
    lib.b200_engine_fill_slot.argtypes = [vp, C.c_int, C.POINTER(PicParams), C.c_int, C.c_int]
    lib.b200_engine_upload_slot.argtypes = [vp, C.c_int, C.POINTER(PicParams), PlaneArray, StrideArray]
    lib.b200_engine_read_slot.argtypes = [vp, C.c_int, PlaneArray, StrideArray]
    lib.b200_engine_read_slot_async.argtypes = [vp, C.c_int, PlaneArray, StrideArray]
    lib.b200_engine_sync.argtypes = [vp]
    lib.b200_engine_submit_picture_async.argtypes = [vp, C.POINTER(Picture)]
    lib.b200_engine_flush.argtypes = [vp]
    lib.b200_engine_last_ticket.argtypes = [vp]
    lib.b200_engine_last_ticket.restype = C.c_ulonglong
    lib.b200_engine_wait_ticket.argtypes = [vp, C.c_ulonglong]
    lib.b200_engine_wait_slot.argtypes = [vp, C.c_int]
    lib.b200_host_alloc.argtypes = [C.c_size_t]
    lib.b200_host_alloc.restype = vp
    lib.b200_host_free.argtypes = [vp]
    lib.b200_host_free.restype = None
    lib.b200_engine_slot_device_planes.argtypes = [vp, C.c_int, PlaneArray, StrideArray]
    lib.b200_engine_export_slot.argtypes = [vp, C.c_int, C.POINTER(Export), PlaneArray, StrideArray, vp]
    lib.b200_engine_enable_timing.argtypes = [vp, C.c_int]
    lib.b200_engine_last_timing.argtypes = [vp, C.POINTER(C.c_float * 6)]
    lib.b200_engine_prepare_picture.argtypes = [vp, C.POINTER(Picture), C.POINTER(vp)]
    lib.b200_engine_run_prepared.argtypes = [vp, vp]
    lib.b200_engine_free_prepared.argtypes = [vp, vp]
    lib.b200_engine_free_prepared.restype = None
    lib.b200_engine_timing_sum.argtypes = [vp, C.POINTER(C.c_float * 6), C.POINTER(C.c_int), C.c_int]
    lib.b200_engine_launch_count.argtypes = [vp]
    lib.b200_engine_launch_count.restype = C.c_uint64
    lib.b200_engine_stream.argtypes = [vp]
    lib.b200_plan_picture_host.argtypes = [C.POINTER(Picture), C.POINTER(C.c_uint32 * 8)] + [C.POINTER(C.c_uint32), C.c_size_t] * 4
    lib.b200_dsp_create.argtypes = [C.POINTER(vp), C.c_int]
    lib.b200_dsp_destroy.argtypes = [vp]
    lib.b200_dsp_destroy.restype = None
    lib.b200_dsp_run_batch.argtypes = [vp, C.POINTER(DspCmd), C.c_int]
    lib.b200_engine_set_streams.argtypes = [vp, C.c_int]
    lib.b200_engine_join.argtypes = [vp]
    lib.b200_engine_stream.restype = vp
    lib.b200_last_error.restype = C.c_char_p
    lib.b200_rec_create.argtypes = [C.POINTER(vp)]
    lib.b200_rec_destroy.argtypes = [vp]
    lib.b200_rec_destroy.restype = None
    lib.b200_rec_begin_picture.argtypes = [vp, C.POINTER(PicParams)]
    lib.b200_rec_add_slice.argtypes = [vp, C.POINTER(SliceInfo)]
    lib.b200_rec_add_weights.argtypes = [vp, C.POINTER(WeightEntry)]
    lib.b200_rec_add_pu.argtypes = [vp, C.POINTER(PU)]
    lib.b200_rec_add_tu.argtypes = [vp, C.POINTER(TU), C.POINTER(C.c_int16), C.POINTER(C.c_int16), C.c_int]
    lib.b200_rec_set_ctb.argtypes = [vp, C.c_int, C.c_int, C.POINTER(CtbInfo)]
    lib.b200_rec_bs_map.argtypes = [vp]
    lib.b200_rec_bs_map.restype = C.POINTER(C.c_uint8)
    lib.b200_rec_qp_map.argtypes = [vp]
    lib.b200_rec_qp_map.restype = C.POINTER(C.c_int8)
    lib.b200_rec_nofilt_map.argtypes = [vp]
    lib.b200_rec_nofilt_map.restype = C.POINTER(C.c_uint8)
    lib.b200_rec_set_scaling_factors.argtypes = [vp, C.POINTER(C.c_uint8)]
    lib.b200_rec_end_picture.argtypes = [vp, C.POINTER(Picture)]
    lib.b200_picture_serialized_size.argtypes = [C.POINTER(Picture)]
    lib.b200_picture_serialized_size.restype = C.c_size_t
    lib.b200_picture_serialize.argtypes = [C.POINTER(Picture), vp, C.c_size_t]
    lib.b200_picture_serialize.restype = C.c_size_t
    lib.b200_picture_deserialize.argtypes = [vp, C.c_size_t, C.POINTER(Picture)]
    lib.b200_picture_deserialize.restype = C.c_size_t
    if path is None:
        _lib = lib
    return lib


class B200Error(RuntimeError):
    pass


def check(rc, what=""):
    if rc < 0:
        msg = load().b200_last_error()
        raise B200Error(f"{what} failed with {rc}: {msg.decode() if msg else ''}")
    return rc
