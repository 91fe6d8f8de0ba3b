"""Build libsatb200.so (sm_90a) in-tree with nvcc.

    python friendly-stable-audio-tools_b200/build.py [--force] [--verbose]

Objects go to ``csrc/build/`` and the shared library to
``friendly-stable-audio-tools_b200/libsatb200.so`` (both git-ignored).
Cross-compiles without a GPU.  Only files whose sources (or headers) changed are rebuilt.
"""
import concurrent.futures
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(CSRC, "build")
LIB = os.path.join(HERE, "libsatb200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
         "-Xptxas", "-v"]


def _headers_digest():
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for f in sorted(os.listdir(root)):
            if f.endswith((".cuh", ".h")):
                h.update(open(os.path.join(root, f), "rb").read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(src, obj, stamp, digest, verbose):
    cmd = [NVCC] + FLAGS + ["-c", src, "-o", obj]
    p = subprocess.run(cmd, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{p.stdout}\n{p.stderr}")
    with open(stamp, "w") as f:
        f.write(digest)
    log = p.stderr
    with open(obj + ".ptxas.log", "w") as f:
        f.write(log)
    if verbose:
        print(log)
    return src


def build(force=False, verbose=False):
    os.makedirs(BUILD, exist_ok=True)
    hd = _headers_digest()
    srcs = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    jobs = []
    objs = []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(BUILD, s[:-3] + ".o")
        stamp = obj + ".stamp"
        digest = hashlib.sha256(open(src, "rb").read()).hexdigest() + hd
        objs.append(obj)
        fresh = (not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == digest)
        if not fresh:
            jobs.append((src, obj, stamp, digest))
    if jobs:
        with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            futs = [ex.submit(_compile, *j, verbose) for j in jobs]
            for f in futs:
                print("compiled", os.path.basename(f.result()), flush=True)
    if jobs or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-cudart", "static", "-Xlinker", "--no-undefined",
                                                     "-lpthread", "-ldl", "-lrt"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError(f"link failed:\n{p.stdout}\n{p.stderr}")
        print("linked", LIB, flush=True)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
