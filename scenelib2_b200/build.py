"""In-tree build of libsl2b200.so (sm_90a only).  nvcc cross-compiles without a GPU."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = ["csrc/api.cu", "csrc/search.cu", "csrc/ekf.cu", "csrc/consensus.cu", "csrc/reloc.cu", "csrc/update.cu",
           "csrc/detect.cu", "csrc/particles.cu", "csrc/smoe.cu", "csrc/snapshot.cu", "csrc/records.cu", "csrc/ingest.cu"]
HEADERS = ["csrc/sl2_common.cuh", "csrc/sl2_model.cuh", "csrc/sl2_ptx.cuh", "csrc/sl2_score.cuh", "../include/sl2b200.h",
           "host/scenelib2_b200.cpp", "host/scenelib2_b200.h", "host/sl2_compat.h", "host/sl2_headless.cpp",
           "host/png_decode.h", "host/jpeg_decode.h", "host/bmp_decode.h"]
LIB = os.path.join(HERE, "libsl2b200.so")


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(HERE, f)) > t for f in SOURCES + HEADERS)


def build(force=False, verbose=False):
    """Compile every CUDA source for sm_90a into scenelib2_b200/libsl2b200.so."""
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
           "-Xcompiler", "-fPIC", "-shared", "-cudart", "static", "-o", LIB] + SOURCES
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
    if os.environ.get("SL2_EXTRA_NVCC"):  # experiments only
        cmd[1:1] = os.environ["SL2_EXTRA_NVCC"].split()
    subprocess.check_call(cmd, cwd=HERE)
    build_host()
    return LIB


def build_host():
    """C++ host shim (MonoSLAM / Kalman / Feature surface) + headless driver, linked to the C ABI."""
    cxx = os.environ.get("CXX", "g++")
    host = os.path.join(HERE, "host")
    so = os.path.join(host, "libscenelib2_b200_host.so")
    exe = os.path.join(host, "sl2_headless")
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", so,
                           os.path.join(host, "scenelib2_b200.cpp"), "-L" + HERE, "-lsl2b200",
                           "-Wl,-rpath,$ORIGIN/.."])
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-pthread", "-o", exe, os.path.join(host, "sl2_headless.cpp"),
                           "-L" + host, "-lscenelib2_b200_host", "-L" + HERE, "-lsl2b200",
                           "-Wl,-rpath,$ORIGIN:$ORIGIN/.."])
    return exe


if __name__ == "__main__":
    print(build(force=True, verbose=True))
