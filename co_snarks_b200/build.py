"""nvcc build of libcosnarks_gpu.so for sm_90a (H100), in-tree next to the package."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libcosnarks_gpu.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = GENCODE + ["-lineinfo", "-O3", "-std=c++17",
         "--expt-relaxed-constexpr", "-DCS_ENABLE_BLS12_381", "-Xcompiler", "-fPIC", "-Xcompiler", "-O2", "-shared", "-cudart", "static"]


def sources():
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith(".cu")]


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(os.path.dirname(HERE), "include", "cosnarks_gpu.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, extra=()):
    if not force and not needs_build():
        return OUT
    objs = []
    os.makedirs(os.path.join(HERE, "_obj"), exist_ok=True)
    procs = []
    for s in sources():
        o = os.path.join(HERE, "_obj", os.path.basename(s) + ".o")
        cmd = [NVCC] + [f for f in FLAGS if f != "-shared"] + list(extra) + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(o)
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stdout.write(out)
        if p.returncode:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    subprocess.check_call([NVCC, "-shared", "-cudart", "static"] + GENCODE + ["-o", OUT] + objs)
    return OUT


if __name__ == "__main__":
    print(build(force="-f" in sys.argv, verbose="-v" in sys.argv))
