"""Build libbsc_b200/libbsc_b200.so (sm_90a, H100) with nvcc.  In-tree, incremental per source."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libbsc_b200.so")
CLI = os.path.join(HERE, "bsc_b200")          # file-level front end (cli/bsc_b200.cpp), bsc1 container + multi-GPU block scheduler
SOURCES = ["api.cu", "adler32.cu", "bwt_encode.cu", "bwt_encode_batched.cu", "bwt_decode.cu", "st_encode.cu", "st_encode_batched.cu", "st_decode.cu", "qlfc.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC,-O2,-Wall,-Wno-unused-function", "-ccbin", "/usr/bin/g++",
         "-Xptxas", "-v"] + os.environ.get("BSCB200_NVCC_EXTRA", "").split()      # e.g. -DQE_DIAG (diagnostic builds only)


def _deps():
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".inc", ".h"))] + \
           [os.path.join(os.path.dirname(HERE), "include", "libbsc_b200.h")]


def _stale(target, srcs):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in srcs)


def _compile(src):
    obj = os.path.join(OBJ, src.replace(".cu", ".o"))
    path = os.path.join(CSRC, src)
    if not _stale(obj, [path] + _deps()):
        return obj, ""
    p = subprocess.run([NVCC] + FLAGS + ["-c", path, "-o", obj], capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, p.stdout, p.stderr))
    return obj, p.stderr


def build(verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    with ThreadPoolExecutor(max_workers=6) as ex:
        results = list(ex.map(_compile, SOURCES))
    objs = [o for o, _ in results]
    if verbose:
        for _, log in results:
            if log:
                sys.stderr.write(log)
    if _stale(LIB, objs):
        p = subprocess.run([NVCC, "-shared", "-o", LIB] + objs + ["-Xlinker", "-Bsymbolic", "-lcudart", "-ccbin", "/usr/bin/g++"],
                           capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (p.stdout, p.stderr))
    cli_src = os.path.join(HERE, "cli", "bsc_b200.cpp")
    if _stale(CLI, [cli_src, LIB, os.path.join(os.path.dirname(HERE), "include", "libbsc_b200.h")]):
        p = subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-pthread", cli_src, "-o", CLI, "-L" + HERE, "-lbsc_b200", "-Wl,-rpath,$ORIGIN"],
                           capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError("CLI build failed:\n%s\n%s" % (p.stdout, p.stderr))
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv))
