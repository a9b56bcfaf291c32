"""In-tree build of the sm_90a (H100) shared library (nvcc, no torch headers involved).

The library is a plain C-ABI .so (include/v2e_b200.h); it links only the CUDA runtime and driver.
nvcc cross-compiles without a GPU, so this also runs on the CPU-only build container.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libv2e_b200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "--expt-extended-lambda", "-Xcompiler", "-fPIC",
          "-I", os.path.join(os.path.dirname(HERE), "include")]

# translation unit -> extra flags. emu.cu needs -fmad=false: the reference evaluates each tensor
# op separately, so no multiply-add may be contracted (DESIGN.md "bit-exact arithmetic").
UNITS = {
    "emu.cu": ["-fmad=false"],
    "slomo.cu": [],
    "conv_tc.cu": [],
    "sinks.cu": [],
    "prep.cu": [],
    "render.cu": [],
    "mjpeg.cu": [],
}


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def sources():
    return [u for u in UNITS if os.path.exists(os.path.join(CSRC, u))]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(os.path.dirname(HERE), "include", "v2e_b200.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    nvcc = _nvcc()
    objs = []
    procs = []
    for u in sources():
        obj = os.path.join(LIBDIR, u.replace(".cu", ".o"))
        cmd = [nvcc] + ARCH + COMMON + UNITS[u] + ["-c", os.path.join(CSRC, u), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd), file=sys.stderr)
        procs.append((u, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for u, p in procs:
        out, _ = p.communicate()
        if verbose and out:
            sys.stderr.write(out.decode())
        if p.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (u, out.decode()))
    cmd = [nvcc] + ARCH + ["-shared", "-o", LIB] + objs
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
