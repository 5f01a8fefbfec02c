"""Builds libygg_b200.so in-tree with nvcc for sm_90a (H100; no JIT cache: the .so travels with the repo)."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# YGG_B200_LIB selects an alternative prebuilt library (kernel-variant experiments only).
LIB = os.environ.get("YGG_B200_LIB") or os.path.join(HERE, "libygg_b200.so")
EXTRA_FLAGS = os.environ.get("YGG_B200_NVCC_FLAGS", "").split()
SOURCES = ["ygg_engine.cu", "ygg_dataspec.cc", "ygg_model_io.cc", "ygg_comm.cc", "ygg_binning.cu"]
HEADERS = ["ygg_device.cuh", "ygg_kernels.cuh", "../../include/ygg_b200.h",
           "../../include/ygg_b200_dataspec.h", "../../include/ygg_b200_model.h", "ygg_hist.cuh", "ygg_hist_seg.cuh", "ygg_wide.cuh", "ygg_presort.cuh",
           "../../include/ygg_b200_comm.h", "ygg_internal.h"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "-ldl",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.sep not in cand or os.path.exists(cand)):
            return cand
    return "nvcc"


def stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    for f in SOURCES + HEADERS:
        p = os.path.join(CSRC, f)
        if os.path.exists(p) and os.path.getmtime(p) > t:
            return True
    return False


def build(force=False, verbose=False):
    if os.environ.get("YGG_B200_LIB") and os.path.exists(LIB) and not force:
        return LIB
    if not force and not stale():
        return LIB
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    # torchrun ranks may all find the library stale at once: one builds (to a temporary name, renamed atomically),
    # the others wait on the lock and then find it fresh
    import fcntl
    with open(LIB + ".lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not stale():
                return LIB
            tmp = "%s.%d.tmp" % (LIB, os.getpid())
            cmd = [_nvcc()] + NVCC_FLAGS + EXTRA_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + srcs
            subprocess.check_call(cmd)
            os.replace(tmp, LIB)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
