"""In-tree build of libdkb200.so (nvcc, sm_90a only).  `python -m diffusionkit_b200.build`."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdkb200.so")
SOURCES = ["api.cu", "gemm.cu", "conv_fused.cu", "attention.cu", "elementwise.cu", "text.cu", "canny.cu", "depth.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]
# ptxas performance advisory: "wgmma.mma_async instructions are serialized due to ..."
SERIALISED_WGMMA = "C7510"


def _stale(obj, src):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    deps = [src] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    deps.append(os.path.join(HERE, "..", "include", "dkb200.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        if not os.path.exists(src):
            continue
        obj = os.path.join(CSRC, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, src):
            cmd = [nvcc, *NVCC_FLAGS, "-c", src, "-o", obj]
            procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = []
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed.append(s)
            sys.stderr.write(f"[build] {s} FAILED\n{out}\n")
        elif SERIALISED_WGMMA in out:
            # ptxas serialised a kernel's wgmma instructions (a function call in a wgmma kernel): the code would run,
            # only much slower, so it is refused here instead of surfacing as a silent slowdown
            failed.append(s)
            os.remove(os.path.join(CSRC, s.replace(".cu", ".o")))
            sys.stderr.write(f"[build] {s} FAILED: ptxas serialised wgmma instructions ({SERIALISED_WGMMA})\n{out}\n")
        elif verbose:
            sys.stderr.write(f"[build] {s}\n{out}\n")
    if failed:
        raise RuntimeError(f"nvcc failed: {', '.join(failed)}")
    if procs or not os.path.exists(LIB):
        cmd = [nvcc, "-shared", "-Wno-deprecated-gpu-targets", "-o", LIB, *objs, "-lcudart", "-ldl"]
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
