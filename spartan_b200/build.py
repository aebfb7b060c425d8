"""Build libspartan_b200.so in-tree: nvcc (sm_90a, H100) for the kernels, g++ for the host prover, nvcc to link."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
TAG = os.environ.get("SP_BUILD_TAG", "")
# defaults: out-of-line F_q multiplications keep the fused sumcheck kernels inside the instruction
# cache (the F_p multiplication of the curve kernels stays inline: the out-of-line call would add register shuffles to every product),
# 2 CTAs of 256 threads per SM for the sumcheck kernels, <= 128 registers for the MSM kernel
DEFAULT_FLAGS = "-DSP_NI_FQ -DSP_SC_LB=2 -DSP_MSM_LB=4"
EXTRA = os.environ.get("SP_BUILD_FLAGS", DEFAULT_FLAGS).split()
OUT = os.path.join(HERE, "libspartan_b200%s.so" % TAG)
NVCC = os.environ.get("SP_NVCC", "/usr/local/cuda/bin/nvcc")
CXX = "/usr/bin/g++"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CU = ["kernels.cu", "kernels_sc.cu", "kernels_pip.cu", "kernels_inst.cu", "comm.cu"]
CPP = ["prover.cpp", "snark.cpp", "verifier.cpp", "capi.cpp", "deflate.cpp"]
HDR = ["field.cuh", "mul_ptx.cuh", "curve.cuh", "kcommon.cuh", "quad.cuh","dev.hpp", "host.hpp", "host_fe51.hpp", "engine.hpp", "prover.hpp", "snark.hpp", "wire.hpp", os.path.join("..", "..", "include", "spartan_b200.h")]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(os.path.join(HERE, "build" + TAG), exist_ok=True)
    stamp = os.path.join(HERE, "build" + TAG, "flags.txt")
    flags = " ".join(EXTRA)
    if not os.path.exists(stamp) or open(stamp).read() != flags:   # objects built with other -D flags are stale too
        force = True
    hdrs = [os.path.join(CSRC, h) for h in HDR]
    objs = []
    procs = []
    for f in CU:
        o = os.path.join(HERE, "build" + TAG, f + ".o")
        objs.append(o)
        if force or _stale(o, [os.path.join(CSRC, f)] + hdrs):
            cmd = [NVCC, "-ccbin", CXX] + ARCH + EXTRA + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-c", os.path.join(CSRC, f), "-o", o]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            procs.append((cmd, subprocess.Popen(cmd)))
    for f in CPP:
        o = os.path.join(HERE, "build" + TAG, f + ".o")
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
    with open(stamp, "w") as f:
        f.write(flags)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
