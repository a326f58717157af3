"""In-tree build of libcnmf_b200.so (nvcc, sm_90a: H100).

    python -m cnmf_b200.build [--force]

nvcc cross-compiles without a GPU.  Objects go to build/ (git-ignored), the shared library to
cnmf_b200/libcnmf_b200.so (git-ignored).
"""
import concurrent.futures
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ_DIR = os.path.join(ROOT, "build", "obj")
LIB_PATH = os.path.join(HERE, "libcnmf_b200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + [ "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-ffp-contract=off", "--expt-relaxed-constexpr",
]


def sources():
    out = []
    for f in sorted(os.listdir(CSRC)):
        if f.endswith(".cu") or f.endswith(".cpp"):
            out.append(os.path.join(CSRC, f))
    return out


def headers_mtime():
    m = 0.0
    for d in (CSRC, os.path.join(ROOT, "include")):
        for f in os.listdir(d):
            if f.endswith((".h", ".cuh")):
                m = max(m, os.path.getmtime(os.path.join(d, f)))
    return m


def _compile(src, obj):
    cmd = [NVCC] + NVCC_FLAGS + ["-x", "cu", "-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    return src, r.returncode, r.stdout + r.stderr


def build(force=False, verbose=True):
    os.makedirs(OBJ_DIR, exist_ok=True)
    hm = headers_mtime()
    jobs, objs = [], []
    for src in sources():
        obj = os.path.join(OBJ_DIR, os.path.basename(src) + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hm):
            jobs.append((src, obj))
    if jobs:
        with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for src, rc, out in ex.map(lambda a: _compile(*a), jobs):
                if verbose and out.strip():
                    print(out)
                if rc != 0:
                    raise RuntimeError("nvcc failed on %s\n%s" % (src, out))
                if verbose:
                    print("compiled", os.path.relpath(src, ROOT))
    if jobs or not os.path.exists(LIB_PATH):
        cmd = [NVCC, "-shared", "-o", LIB_PATH] + objs + ARCH + ["-Xcompiler", "-fPIC", "-lpthread", "-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed\n" + r.stdout + r.stderr)
        if verbose:
            print("linked", os.path.relpath(LIB_PATH, ROOT))
    return LIB_PATH


if __name__ == "__main__":
    build(force="--force" in sys.argv)
