"""Build the C-ABI shared library (elliot_b200/csrc/libelliot_b200.so) with nvcc for sm_90a.

In-tree, no torch dependency: the library exposes plain `extern "C"` entry points
(include/elliot_b200.h) and is loaded with ctypes.  `python -m elliot_b200.build` rebuilds.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(CSRC, "libelliot_b200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
         "-Xptxas", "-v", "-Wno-deprecated-gpu-targets"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(HERE, "..", "include", "elliot_b200.h"))
    objs = []
    logs = []
    todo = []
    for src in sources():
        obj = src[:-3] + ".o"
        objs.append(obj)
        if force or _stale(obj, [src] + hdrs):
            todo.append((src, obj))

    def compile_one(job):
        src, obj = job
        return src, subprocess.run([nvcc] + ARCH + FLAGS + ["-c", src, "-o", obj], capture_output=True, text=True)

    # translation units are independent: compile the stale ones side by side (a from-scratch build is dominated by the two
    # tensor-core files, ~1.5 min each on one core)
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=max(1, min(8, os.cpu_count() or 1))) as pool:
        for src, r in pool.map(compile_one, todo):
            logs.append((os.path.basename(src), r.stderr))
            if r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
                raise RuntimeError(f"nvcc failed on {src}")
            if verbose:
                sys.stderr.write(r.stderr)
    if force or _stale(LIB, objs):
        cmd = [nvcc] + ARCH + ["-shared", "-o", LIB] + objs + ["-lcudart_static", "-lpthread", "-ldl", "-lrt"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return LIB, logs


if __name__ == "__main__":
    lib, logs = build(force="--force" in sys.argv, verbose=True)
    print(lib)
