"""Builds voicefixer_b200/libvfx_b200.so in-tree with nvcc for sm_90a (no JIT cache), and the
host-only audio file codec voicefixer_b200/libvfx_hostio.so with gcc."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libvfx_b200.so")
SOURCES = ["engine.cu", "conv_gemm_simt.cu", "conv_gemm_tc.cu", "resstack_pair.cu", "elementwise.cu", "frontend.cu",
           "gru.cu", "hf_cut.cu", "oracle_fe.cu", "resample.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


HOSTIO_SRC = os.path.join(HERE, "hostio", "flac_codec.c")
HOSTIO_LIB = os.path.join(HERE, "libvfx_hostio.so")


def build_hostio(force=False):
    """gcc -> libvfx_hostio.so (include/vfx_hostio.h: FLAC reader / writer for the file API)."""
    hdr = os.path.join(HERE, "..", "include", "vfx_hostio.h")
    if (not force and os.path.exists(HOSTIO_LIB) and os.path.getmtime(HOSTIO_LIB) >= os.path.getmtime(HOSTIO_SRC)
            and os.path.getmtime(HOSTIO_LIB) >= os.path.getmtime(hdr)):
        return HOSTIO_LIB
    cmd = [os.environ.get("CC", "gcc"), "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", HOSTIO_LIB, HOSTIO_SRC]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("gcc failed on flac_codec.c:\n" + r.stdout)
    return HOSTIO_LIB


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [
        os.path.join(HERE, "..", "include", "vfx_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    build_hostio(force)
    if not force and not needs_build():
        return LIB
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")] + [
        os.path.join(HERE, "..", "include", "vfx_b200.h")]
    for s in SOURCES:
        obj = os.path.join(objdir, s.replace(".cu", ".o"))
        src = os.path.join(CSRC, s)
        if (not force and os.path.exists(obj)
                and all(os.path.getmtime(obj) > os.path.getmtime(d) for d in [src] + headers)):
            continue
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {s}:\n{out}")
        if verbose or out.strip():
            print(out)
    objs = [os.path.join(objdir, s.replace(".cu", ".o")) for s in SOURCES]
    cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-lcudart", "-lcuda"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
