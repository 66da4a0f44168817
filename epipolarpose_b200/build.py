"""Builds libepb.so (sm_90a only) in-tree with nvcc.  No JIT cache: the .so
sits next to this file so it travels with a repo snapshot."""
import concurrent.futures
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "..", "build", "obj")
LIB = os.path.join(HERE, "libepb.so")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo",
              "-std=c++17", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"]
PER_FILE = {"geometry.cu": ["--fmad=false"], "input.cu": ["--fmad=false"],    # double rounding as on the CPU
            "pss.cu": ["--fmad=false"]}


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(HERE, "..", "include", "epb.h"))
    nvcc = _nvcc()
    jobs = []
    for s in sources():
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s[:-3] + ".o")
        if force or _stale(obj, [src] + headers):
            jobs.append([nvcc] + NVCC_FLAGS + PER_FILE.get(s, []) + ["-c", src, "-o", obj])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        if verbose and r.stderr:
            sys.stderr.write(r.stderr)

    with concurrent.futures.ThreadPoolExecutor(max_workers=8) as ex:
        list(ex.map(run, jobs))
    objs = [os.path.join(OBJ, s[:-3] + ".o") for s in sources()]
    if force or jobs or _stale(LIB, objs):
        run([nvcc, "-shared", "-o", LIB] + objs + ["-lcudart", "-lcuda"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
