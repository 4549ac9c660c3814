"""In-tree build of the sm_90a extension ``baton_b200/_C.so``.

``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo`` per ``.cu`` (the
kernels include no PyTorch header, so each file compiles in seconds), ``g++`` for
``bindings.cpp`` against the PyTorch headers, one shared object linked in-tree
so it travels to the GPU box with the repo snapshot.  Incremental: a file is
recompiled only when it (or a header) is newer than its object; everything is rebuilt when the compiler, the
flags or the PyTorch version differ from those recorded next to the objects.

    python -m baton_b200.build_ext [--force] [--verbose]
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import sysconfig
import time
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "csrc", "build")
TRACE = os.environ.get("BATON_BUILD_TRACE") == "1"      # kernel-timeline build: own objects, own shared object
if TRACE:
    BUILD = os.path.join(HERE, "csrc", "build_trace")
TARGET = os.path.join(HERE, "_C_trace.so" if TRACE else "_C.so")

CU_SOURCES = ["gemm_wgmma.cu", "gemm_fp8.cu", "quant.cu", "attention.cu", "im2col_tma.cu", "gemm_simt.cu", "fedavg.cu", "elementwise.cu", "conv.cu", "norm.cu", "loss.cu", "conv_halo.cu", "compress.cu", "dropout.cu", "lora.cu",
              "vit.cu"]
HEADERS = ["ptx.cuh", "launch.h", "pdl.cuh", "mx.cuh", "sgd.cuh", "dp.cuh", "epilogue.cuh", "secagg.cuh", "rows.cuh", "dropout.cuh"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--use_fast_math", "-Xptxas", "-v"]
if os.environ.get("BATON_BUILD_PHASE_TIMING") == "1":     # in-kernel %globaltimer stamps in the FedAvg collective
    NVCC_FLAGS.append("-DB200_FEDAVG_PHASE_TIMING")
if TRACE:
    NVCC_FLAGS += ["-DB200_TRACE", "-DB200_FEDAVG_PHASE_TIMING"]    # kernel timeline + in-kernel phase stamps of the collective


def _nvcc() -> str:
    for cand in (os.environ.get("CUDA_HOME", "") + "/bin/nvcc", "/usr/local/cuda/bin/nvcc", shutil.which("nvcc") or ""):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _newer(src_paths, out_path) -> bool:
    if not os.path.exists(out_path):
        return True
    t = os.path.getmtime(out_path)
    return any(os.path.getmtime(p) > t for p in src_paths)


def _run(cmd, verbose, log_path=None):
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if log_path:
        with open(log_path, "w") as f:
            f.write(" ".join(cmd) + "\n" + proc.stdout)
    if proc.returncode != 0:
        sys.stderr.write(proc.stdout)
        raise RuntimeError("build step failed: {}".format(" ".join(cmd[:3])))
    if verbose:
        sys.stdout.write(proc.stdout)


def build(force: bool = False, verbose: bool = False) -> str:
    import torch
    from torch.utils import cpp_extension

    os.makedirs(BUILD, exist_ok=True)
    nvcc = _nvcc()
    # objects record the compiler and flags they were built with: a tree built for another architecture (or with
    # other defines) is rebuilt from scratch instead of being relinked because its sources look older
    stamp = os.path.join(BUILD, "flags.txt")
    want = "\n".join([nvcc] + NVCC_FLAGS + [torch.__version__]) + "\n"
    if not force and (not os.path.exists(stamp) or open(stamp).read() != want):
        force = True
    headers = [os.path.join(CSRC, h) for h in HEADERS]
    t0 = time.time()
    jobs = []
    objs = []
    for cu in CU_SOURCES:
        src = os.path.join(CSRC, cu)
        obj = os.path.join(BUILD, cu.replace(".cu", ".o"))
        objs.append(obj)
        if force or _newer([src] + headers, obj):
            jobs.append(([nvcc] + NVCC_FLAGS + ["-I", CSRC, "-c", src, "-o", obj], obj + ".log"))
    bind_src = os.path.join(CSRC, "bindings.cpp")
    bind_obj = os.path.join(BUILD, "bindings.o")
    objs.append(bind_obj)
    if force or _newer([bind_src] + headers, bind_obj):
        inc = []
        for p in cpp_extension.include_paths("cuda") if hasattr(cpp_extension, "include_paths") else []:
            inc += ["-isystem", p]
        inc += ["-isystem", sysconfig.get_paths()["include"]]
        abi = int(getattr(torch._C, "_GLIBCXX_USE_CXX11_ABI", True))
        jobs.append((["g++", "-O2", "-std=c++17", "-fPIC", "-DTORCH_EXTENSION_NAME=_C",
                      "-DTORCH_API_INCLUDE_EXTENSION_H", "-D_GLIBCXX_USE_CXX11_ABI={}".format(abi),
                      "-I", CSRC] + inc + ["-c", bind_src, "-o", bind_obj], bind_obj + ".log"))
    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as pool:
            list(pool.map(lambda j: _run(j[0], verbose, j[1]), jobs))
    if jobs or force or not os.path.exists(TARGET):
        torch_lib = os.path.join(os.path.dirname(torch.__file__), "lib")
        cuda_lib = os.path.join(os.path.dirname(os.path.dirname(nvcc)), "lib64")
        link = ["g++", "-shared", "-o", TARGET] + objs + [
            "-L" + torch_lib, "-L" + cuda_lib, "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch",
            "-ltorch_python", "-lcudart", "-Wl,-rpath," + torch_lib, "-Wl,--no-as-needed"]
        _run(link, verbose)
    with open(stamp, "w") as fh:
        fh.write(want)
    if verbose:
        print("built {} in {:.1f}s ({} compile steps)".format(TARGET, time.time() - t0, len(jobs)))
    return TARGET


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="--verbose" in sys.argv or "-v" in sys.argv)
    print(TARGET)
