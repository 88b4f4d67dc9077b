"""Build the zeekstd_b200 native library IN-TREE.

  python -m zeekstd_b200.build            -> zeekstd_b200/libzeekstd_b200.so   (nvcc, sm_90a; the product)
  python -m zeekstd_b200.build --emul     -> tests/emul/_build/libzeekstd_b200_emul.so  (g++, TEST ONLY:
                                             device code interpreted by tests/emul/cuda_emul.h)
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["zk_decode.cu", "zk_encode.cu", "zk_api.cu", "zk_host.cpp"]
PRODUCT_SO = os.path.join(HERE, "libzeekstd_b200.so")
EMUL_DIR = os.path.join(ROOT, "tests", "emul", "_build")
EMUL_SO = os.path.join(EMUL_DIR, "libzeekstd_b200_emul.so")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _newer(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(d) <= t for d in deps)


def _deps() -> list[str]:
    d = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    d.append(os.path.join(ROOT, "include", "zeekstd_b200.h"))
    return d


def build_product(force: bool = False, verbose: bool = False) -> str:
    if not force and _newer(PRODUCT_SO, _deps()):
        return PRODUCT_SO
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src + ".o")
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-x", "cu", "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            raise RuntimeError(f"nvcc failed on {src}")
    cmd = [nvcc, "-shared", "-o", PRODUCT_SO] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
    subprocess.run(cmd, check=True)
    return PRODUCT_SO


def build_emul(force: bool = False, sanitize: bool = False) -> str:
    so = EMUL_SO.replace(".so", "_asan.so") if sanitize else EMUL_SO
    deps = _deps() + [os.path.join(ROOT, "tests", "emul", "cuda_emul.h")]
    if not force and _newer(so, deps):
        return so
    os.makedirs(EMUL_DIR, exist_ok=True)
    cxx = os.environ.get("CXX", "g++")
    flags = ["-std=c++17", "-O1" if sanitize else "-O2", "-g", "-fPIC", "-shared", "-DZK_EMUL", "-Wall", "-Wno-unused-function",
             "-Wno-unknown-pragmas", "-Wno-unused-variable", "-include", os.path.join(ROOT, "tests", "emul", "cuda_emul.h")]
    if sanitize:
        flags += ["-fsanitize=address,undefined", "-fno-omit-frame-pointer"]
    cmd = [cxx] + flags + sum([["-x", "c++", os.path.join(CSRC, s)] for s in SOURCES], []) + ["-o", so]
    subprocess.run(cmd, check=True)
    return so


if __name__ == "__main__":
    if "--emul" in sys.argv:
        print(build_emul(force="--force" in sys.argv, sanitize="--asan" in sys.argv))
    else:
        print(build_product(force="--force" in sys.argv, verbose="-v" in sys.argv))
