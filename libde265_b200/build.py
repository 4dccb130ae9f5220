"""In-tree build of the CUDA library (sm_90a, H100, only).  Used by __graft_entry__.build()."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libb200hevc.so")
SOURCES = ["engine.cu", "recorder.cc"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC,-fvisibility=hidden",
              "-shared", "-I" + os.path.join(ROOT, "include"), "-I" + CSRC]


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", f) for f in os.listdir(os.path.join(ROOT, "include"))]
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False, defines=(), out=None):
    """defines / out: experiment builds (e.g. defines=("MCT_TLS=16",), out=".../libb200hevc_tls16.so"; select with B200_LIB)."""
    out = out or OUT
    if not force and out == OUT and not needs_build():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else []) + [os.path.join(CSRC, s) for s in SOURCES] + ["-o", out]
    subprocess.check_call(cmd)
    return out


if __name__ == "__main__":
    import sys
    build_library(force=True, verbose="-v" in sys.argv)
    print(OUT)
