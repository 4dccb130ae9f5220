"""libde265_b200 — H100 (sm_90a) HEVC reconstruction engine behind libde265's API.

capi   : ctypes mirror of include/b200hevc.h (engine + recorder, the C-ABI boundary)
de265  : host-side mirror of libde265's de265.h decoder API
engine : Python convenience wrapper around b200_engine_*
"""
