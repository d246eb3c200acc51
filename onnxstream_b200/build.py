"""In-tree build of libonnxstream_b200.so (hand-written sm_90a CUDA + C++ host) with nvcc/g++ -- no cmake, no JIT cache.

The built library lives next to the sources (git-ignored).
`python -m onnxstream_b200.build` rebuilds what changed; `--force` rebuilds everything.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# Build variants for A/B experiments: OSB_BUILD_VARIANT=name OSB_NVCC_EXTRA="-DFOO" builds
# csrc/libonnxstream_b200_<name>.so from csrc/build_<name>/ (the product library is the unnamed variant).
VARIANT = os.environ.get("OSB_BUILD_VARIANT", "")
OBJ = os.path.join(CSRC, "build" + ("_" + VARIANT if VARIANT else ""))
LIB = os.path.join(CSRC, "libonnxstream_b200" + ("_" + VARIANT if VARIANT else "") + ".so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CXX = os.environ.get("OSB_CXX", "/usr/bin/g++")

CU_SOURCES = ["kernels_basic.cu", "kernels_gemm.cu", "gemm_wgmma.cu", "attention_wgmma.cu"]
CPP_SOURCES = ["engine.cpp", "engine_run.cpp", "plan.cpp", "capi.cpp", "comm.cpp", "workspace.cpp"]
HEADERS = ["common.cuh", "tc_ptx.cuh", "gemm_i8.cuh", "engine.h", "engine_impl.h", "plan.h", "workspace.h", "../../include/onnxstream_b200_kernels.h", "../../include/onnxstream_b200.h"]

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
              "-Xcompiler", "-fPIC", "-ccbin", CXX] + os.environ.get("OSB_NVCC_EXTRA", "").split()
CXX_FLAGS = ["-std=c++17", "-O2", "-fPIC", "-I/usr/local/cuda/include", "-Wall", "-Wno-sign-compare", "-Wno-unused-function"]


# where a read-only checkout of the reference (github.com/vitoplantamura/OnnxStream) is looked for: next to this repository, or at
# /root/reference; ONNXSTREAM_REF_SRC (its src/ directory) overrides both
REFERENCE_SRC_CANDIDATES = (os.path.join(os.path.dirname(os.path.dirname(HERE)), "reference", "src"), "/root/reference/src")


def reference_src():
    """The reference's src/ directory, or None: only the oracle, its YOLOv8n fixture and the C++ link test need it."""
    env = os.environ.get("ONNXSTREAM_REF_SRC", "")
    for ref in ((env,) if env else REFERENCE_SRC_CANDIDATES):
        if os.path.isfile(os.path.join(ref, "onnxstream.cpp")):
            return ref
    return None


def _newer(src_paths, target):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(p) > t for p in src_paths if os.path.exists(p))


def _run(cmd):
    r = subprocess.run(cmd, cwd=CSRC, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed: " + " ".join(cmd) + "\n" + r.stdout)
    return r.stdout


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    jobs = []
    objs = []
    for src in CU_SOURCES + CPP_SOURCES:
        obj = os.path.join(OBJ, src.rsplit(".", 1)[0] + ".o")
        objs.append(obj)
        if force or _newer([os.path.join(CSRC, src)] + hdrs, obj):
            if src.endswith(".cu"):
                jobs.append([NVCC] + NVCC_FLAGS + ["-c", src, "-o", obj])
            else:
                jobs.append([CXX] + CXX_FLAGS + ["-c", src, "-o", obj])
    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for out in ex.map(_run, jobs):
                if verbose and out.strip():
                    print(out)
    if jobs or force or not os.path.exists(LIB):
        _run([NVCC, "-shared", "-o", LIB] + objs + ["-cudart", "static", "-ccbin", CXX, "-Xlinker", "--no-undefined", "-ldl", "-lpthread"])
    # keep the C++ drop-in link test (reference apps + compat_onnxstream.cpp) in step with the engine ABI
    link_script = os.path.join(os.path.dirname(HERE), "scripts", "link_reference_apps.sh")
    compat_obj = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "link_test", "compat.o")
    if not VARIANT and reference_src() and os.path.exists(link_script) and _newer(hdrs + [os.path.join(CSRC, "compat_onnxstream.cpp"), LIB], compat_obj):
        r = subprocess.run(["bash", link_script], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=dict(os.environ, REF=reference_src()))
        if r.returncode != 0:
            raise RuntimeError("link test (reference apps against the engine) failed:\n" + r.stdout[-3000:])
    return LIB


if __name__ == "__main__":
    lib = build(force="--force" in sys.argv, verbose=True)
    print(lib)
