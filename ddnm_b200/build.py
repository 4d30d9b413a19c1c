"""Build libddnm_b200.so (sm_90a only) with nvcc; sources in ddnm_b200/csrc, objects in build/, the shared
library lands IN-TREE next to this file so it travels with the repo snapshot to the GPU box."""
import concurrent.futures as cf
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(ROOT, "build", "obj")
LIB = os.path.join(HERE, "libddnm_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O3", "-lineinfo", "-Xcompiler", "-fPIC",
         "-DDDNM_BUILD"]


def _newer(src, dst, deps):
    if not os.path.exists(dst):
        return True
    t = os.path.getmtime(dst)
    return any(os.path.getmtime(p) > t for p in [src] + deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    srcs = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(ROOT, "include", "ddnm_b200.h"))
    hdrs.append(os.path.abspath(__file__))   # FLAGS (the target architecture) live here: objects older than them are rebuilt
    jobs = []
    for s in srcs:
        src, obj = os.path.join(CSRC, s), os.path.join(OBJ, s[:-3] + ".o")
        if force or _newer(src, obj, hdrs):
            jobs.append((src, obj))

    def cc(job):
        src, obj = job
        cmd = [NVCC] + FLAGS + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose and (r.stdout or r.stderr):
            print(r.stdout, r.stderr)
        return obj

    with cf.ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(cc, jobs))
    objs = [os.path.join(OBJ, s[:-3] + ".o") for s in srcs]
    if jobs or _newer(os.path.abspath(__file__), LIB, []):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
