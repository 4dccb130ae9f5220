"""Thin Python wrapper over b200_engine_* (include/b200hevc.h part 2).  CUDA only — no CPU fallback."""
import ctypes as C

import numpy as np

from . import capi


class Engine:
    def __init__(self, device=0):
        self.lib = capi.load()
        self.device = device
        self._h = C.c_void_p()
        capi.check(self.lib.b200_engine_create(C.byref(self._h), device), "b200_engine_create")

    def close(self):
        if self._h:
            self.lib.b200_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def submit(self, pic):
        """pic: capi.Picture (or an object with a ``.c`` capi.Picture, e.g. synth.SynthPicture)."""
        cp = getattr(pic, "c", pic)
        capi.check(self.lib.b200_engine_submit_picture(self._h, C.byref(cp)), "b200_engine_submit_picture")

    def submit_async(self, pic):
        """Queues the picture (planned by the engine's planner threads, issued in submission order).  The picture's record arrays
        must stay alive until flush() / sync() / read_slot() returns."""
        cp = getattr(pic, "c", pic)
        capi.check(self.lib.b200_engine_submit_picture_async(self._h, C.byref(cp)), "b200_engine_submit_picture_async")

    def flush(self):
        capi.check(self.lib.b200_engine_flush(self._h), "b200_engine_flush")

    def sync(self):
        capi.check(self.lib.b200_engine_sync(self._h), "b200_engine_sync")

    def fill_slot(self, slot, params, vy, vc):
        capi.check(self.lib.b200_engine_fill_slot(self._h, slot, C.byref(params), vy, vc), "b200_engine_fill_slot")

    def upload_slot(self, slot, params, planes):
        """planes: 3 C-contiguous numpy arrays (uint8 or uint16)."""
        pa = capi.PlaneArray(*[p.ctypes.data for p in planes])
        sa = capi.StrideArray(*[p.strides[0] for p in planes])
        capi.check(self.lib.b200_engine_upload_slot(self._h, slot, C.byref(params), pa, sa), "b200_engine_upload_slot")

    def read_slot(self, slot, params):
        """Returns [Y, Cb, Cr] numpy arrays (uint8 for 8-bit, uint16 otherwise)."""
        dt = np.uint16 if params.bit_depth_luma > 8 else np.uint8
        shapes = [(params.height, params.width)]
        if params.chroma_format_idc:
            shapes += [(params.height // 2, params.width // 2)] * 2
        out = [np.empty(s, dt) for s in shapes]
        ptrs = [o.ctypes.data for o in out] + [None] * (3 - len(out))
        strides = [o.strides[0] for o in out] + [0] * (3 - len(out))
        capi.check(self.lib.b200_engine_read_slot(self._h, slot, capi.PlaneArray(*ptrs), capi.StrideArray(*strides)), "b200_engine_read_slot")
        return out

    _RGB = {"bt601": capi.EXPORT_RGB_BT601, "bt709": capi.EXPORT_RGB_BT709, "bt2020": capi.EXPORT_RGB_BT2020}

    def export(self, slot, params, crop=None, rgb=None, full_range=False, stream=None):
        """The picture in `slot` as CUDA tensors on the engine's device, enqueued on `stream` (a torch.cuda.Stream; default: the
        device's current stream), which also allocates the outputs.  Work enqueued on `stream` afterwards sees the picture, and
        pictures or fill_slot / upload_slot that later write the slot wait for the copy.  ``params`` gives the picture's format (as
        for read_slot); ``crop`` = (x, y, width, height) in luma samples, even for 4:2:0 (default: the whole picture).
        Returns [Y, Cb, Cr] (uint8 up to 8 bit, uint16 above; [Y] for 4:0:0), or with ``rgb`` = "bt601" / "bt709" / "bt2020"
        one (3, height, width) uint8 tensor of planar R, G, B (``full_range``: the samples use the full range, not video range).
        With submit_async the call blocks until the slot's picture has been issued to the GPU."""
        import torch
        if rgb is not None and rgb not in self._RGB:
            raise ValueError(f"rgb must be one of {sorted(self._RGB)} or None, not {rgb!r}")
        dev = torch.device("cuda", self.device)
        if stream is None:
            stream = torch.cuda.current_stream(dev)
        x, y, w, h = crop if crop is not None else (0, 0, params.width, params.height)
        if min(x, y, w, h) < 0 or max(x, y, w, h) > 0xFFFF:
            raise capi.B200Error(f"export window {crop} outside the 16-bit range of b200_export")
        with torch.cuda.stream(stream):
            if rgb is not None:
                out = torch.empty((3, h, w), dtype=torch.uint8, device=dev)
                planes = [out[0], out[1], out[2]]
            else:
                dt = [torch.uint16 if params.bit_depth_luma > 8 else torch.uint8, torch.uint16 if params.bit_depth_chroma > 8 else torch.uint8]
                planes = [torch.empty((h, w), dtype=dt[0], device=dev)]
                if params.chroma_format_idc:
                    planes += [torch.empty((h // 2, w // 2), dtype=dt[1], device=dev) for _ in range(2)]
                out = planes
        ex = capi.Export(x, y, w, h, self._RGB[rgb] if rgb is not None else capi.EXPORT_YUV, capi.EXPORT_FULL_RANGE if full_range else 0)
        ptrs = [p.data_ptr() for p in planes] + [None] * (3 - len(planes))
        pitches = [p.stride(0) * p.element_size() for p in planes] + [0] * (3 - len(planes))
        capi.check(self.lib.b200_engine_export_slot(self._h, slot, C.byref(ex), capi.PlaneArray(*ptrs), capi.StrideArray(*pitches),
                                                    C.c_void_p(stream.cuda_stream)), "b200_engine_export_slot")
        return out

    def wait_slot(self, slot):
        """Blocks until the picture in `slot` and every read-back and export of it have finished."""
        capi.check(self.lib.b200_engine_wait_slot(self._h, slot), "b200_engine_wait_slot")

    def read_slot_into(self, slot, planes_ptrs, strides):
        capi.check(self.lib.b200_engine_read_slot(self._h, slot, capi.PlaneArray(*planes_ptrs), capi.StrideArray(*strides)), "b200_engine_read_slot")

    def enable_timing(self, on=True):
        capi.check(self.lib.b200_engine_enable_timing(self._h, int(on)), "b200_engine_enable_timing")

    def last_timing(self):
        ms = (C.c_float * 6)()
        capi.check(self.lib.b200_engine_last_timing(self._h, C.byref(ms)), "b200_engine_last_timing")
        return dict(zip(("h2d", "inter_pred", "recon", "deblock", "sao", "total"), list(ms)))

    def timing_sum(self, reset=True):
        ms = (C.c_float * 6)()
        n = C.c_int(0)
        capi.check(self.lib.b200_engine_timing_sum(self._h, C.byref(ms), C.byref(n), int(reset)), "b200_engine_timing_sum")
        return dict(zip(("h2d", "inter_pred", "recon", "deblock", "sao", "total"), list(ms))), n.value

    def prepare(self, pic):
        cp = getattr(pic, "c", pic)
        h = C.c_void_p()
        capi.check(self.lib.b200_engine_prepare_picture(self._h, C.byref(cp), C.byref(h)), "b200_engine_prepare_picture")
        return h

    def run_prepared(self, h):
        capi.check(self.lib.b200_engine_run_prepared(self._h, h), "b200_engine_run_prepared")

    def free_prepared(self, h):
        self.lib.b200_engine_free_prepared(self._h, h)

    def launch_count(self):
        return int(self.lib.b200_engine_launch_count(self._h))

    def stream(self):
        return self.lib.b200_engine_stream(self._h)

    def set_streams(self, n):
        """Number of CUDA streams pictures are pipelined over (results do not depend on it)."""
        capi.check(self.lib.b200_engine_set_streams(self._h, n), "b200_engine_set_streams")

    def join(self):
        """Stream 0 waits for everything issued so far on the other streams."""
        capi.check(self.lib.b200_engine_join(self._h), "b200_engine_join")
