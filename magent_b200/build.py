"""Build the engine library in-tree: magent_b200/lib/libmagent.so (sm_90a only).

    python -m magent_b200.build [--force] [--verbose]

nvcc cross-compiles without a GPU.  The CUDA runtime is linked statically so the .so travels to the
GPU machine as-is.  ``-lineinfo`` maps kernel SASS back to source lines for profilers.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib", "libmagent.so")
SOURCES = ["engine.cc", "shim.cc", "host_expand.cc", "backend_cuda.cu"]
HEADERS = ["hd.h", "dev_types.h", "step_phases.h", "obs_phases.h", "mask_phases.h", "nbr_phases.h", "backend.h",
           "engine.h", "host_expand.h",
           os.path.join("..", "..", "include", "magent_runtime_api.h"),
           os.path.join("..", "..", "include", "magent_b200_ext.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-ccbin", "/usr/bin/g++",
         "-Xcompiler", "-fPIC,-fvisibility=hidden,-Wall,-Wno-unused-function",
         "--expt-relaxed-constexpr", "-Xptxas", "-v"]
# host-only sources (.cc) go through g++ directly: no CUDA in them, and host_expand.cc uses per-function ISA targets
CXX = "/usr/bin/g++"                     # the same host compiler nvcc uses (-ccbin)
CXXFLAGS = ["-O3", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-Wall", "-Wno-unused-function", "-pthread"]


def up_to_date():
    if not os.path.exists(LIB):
        return False
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return all(os.path.getmtime(d) <= t for d in deps)


def build(force=False, verbose=False):
    if not force and up_to_date():
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    objs = []
    for src in SOURCES:
        obj = os.path.join(HERE, "lib", src.replace(".", "_") + ".o")
        if src.endswith(".cu"):
            cmd = [NVCC] + FLAGS + ["-x", "cu", "-c", os.path.join(CSRC, src), "-o", obj]
        else:
            cmd = [CXX] + CXXFLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or res.returncode != 0:
            sys.stderr.write(" ".join(cmd) + "\n" + res.stdout + res.stderr)
        if res.returncode != 0:
            raise RuntimeError("nvcc failed on " + src)
        with open(obj + ".ptxas.log", "w") as f:
            # compile times differ from run to run; everything else in the log is deterministic
            f.write("".join(l for l in res.stderr.splitlines(True) if "Compile time" not in l))
        objs.append(obj)
    cmd = [NVCC, "-shared", "-ccbin", "/usr/bin/g++", "-gencode", "arch=compute_90a,code=sm_90a",
           "-Xlinker", "-Bsymbolic", "-Xcompiler", "-pthread", "-o", LIB] + objs
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
