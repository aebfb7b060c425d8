"""Build libspartan_b200.so in-tree: nvcc (sm_90a, H100) for the kernels, g++ for the host prover, nvcc to link."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
OUT = os.path.join(HERE, "libspartan_b200.so")
NVCC = os.environ.get("SP_NVCC", "/usr/local/cuda/bin/nvcc")
CXX = "/usr/bin/g++"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CU = ["kernels.cu", "kernels_sc.cu", "kernels_pip.cu", "kernels_inst.cu", "comm.cu"]
CPP = ["prover.cpp", "product.cpp", "snark.cpp", "verifier.cpp", "capi.cpp", "deflate.cpp"]
HDR = ["field.cuh", "mul_ptx.cuh", "curve.cuh", "kcommon.cuh", "quad.cuh","dev.hpp", "host.hpp", "host_fe51.hpp", "engine.hpp", "prover.hpp", "snark.hpp", "wire.hpp", os.path.join("..", "..", "include", "spartan_b200.h")]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(BUILD, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HDR]
    objs = []
    procs = []
    for f in CU:
        o = os.path.join(BUILD, f + ".o")
        objs.append(o)
        if force or _stale(o, [os.path.join(CSRC, f)] + hdrs):
            cmd = [NVCC, "-ccbin", CXX] + ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-c", os.path.join(CSRC, f), "-o", o]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            procs.append((cmd, subprocess.Popen(cmd)))
    for f in CPP:
        o = os.path.join(BUILD, f + ".o")
        objs.append(o)
        if force or _stale(o, [os.path.join(CSRC, f)] + hdrs):
            cmd = [CXX, "-O3", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-Wno-unknown-pragmas", "-I/usr/local/cuda/include", "-c", os.path.join(CSRC, f), "-o", o]
            procs.append((cmd, subprocess.Popen(cmd)))
    for cmd, p in procs:
        if p.wait() != 0:
            raise RuntimeError("build failed: " + " ".join(cmd))
    if force or procs or _stale(OUT, objs):
        # link next to the target and rename: a copy of the tree taken meanwhile never sees a half-written library
        cmd = [NVCC, "-ccbin", CXX] + ARCH + ["-shared", "-cudart", "static", "-o", OUT + ".tmp"] + objs
        subprocess.check_call(cmd)
        os.replace(OUT + ".tmp", OUT)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
