"""Build `libstarvector_b200.so` in-tree with nvcc for sm_90a (no torch extension, no JIT cache).

    python -m starvector_b200.build            # incremental
    python -m starvector_b200.build --force
    python -m starvector_b200.build --variant timeline # second library with the dataflow kernel's timeline records, see VARIANTS

The library has a plain C ABI (include/starvector_b200.h) and links only the static CUDA
runtime, so it travels to the GPU box with the repo snapshot and loads through ctypes.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libstarvector_b200.so")
SOURCES = ["sv_kernels_basic.cu", "sv_gemm_rowgroup.cu", "sv_gemm_wgmma.cu", "sv_attention.cu", "sv_decode_fused.cu", "sv_decode_mega.cu", "sv_decode_flow.cu", "sv_beam.cu", "sv_beam_session.cu", "sv_spec_session.cu", "sv_preprocess.cu", "sv_score.cu", "sv_engine.cu"]
HEADERS = ["sv_common.cuh", "sv_kernels.h", "sv_ring.cuh", "sv_select.cuh", "sv_sample.cuh", "sv_beam_core.h", "sv_beam_body.cuh", "sv_preprocess_core.h", "sv_spec_core.h", os.path.join("..", "..", "include", "starvector_b200.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr", "-Xcompiler", "-ffp-contract=off",
]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found: cannot build libstarvector_b200.so")


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


# Instrumented builds of the same sources (run-time selection: SV_LIB_PATH=<that .so>); never loaded by default.
VARIANTS = {
    "timeline": ["-DSV_FLOW_TIMELINE=1"],     # dataflow decode kernel with its device timeline records compiled in (scripts/flow_timeline.py)
}


def build(force: bool = False, verbose: bool = False, variant: str = "") -> str:
    global OBJ, LIB
    extra = []
    if variant:
        extra = VARIANTS[variant]
        OBJ = os.path.join(HERE, f"build_{variant}")
        LIB = os.path.join(HERE, f"libstarvector_b200_{variant}.so")
    os.makedirs(OBJ, exist_ok=True)
    nvcc = _nvcc()
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    jobs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        if force or _stale(o, [s] + hdrs):
            jobs.append([nvcc, *NVCC_FLAGS, *extra, "-c", s, "-o", o])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed:\n{' '.join(cmd)}\n{r.stdout}\n{r.stderr}")

    with ThreadPoolExecutor(max_workers=min(4, max(1, len(jobs)))) as ex:
        list(ex.map(run, jobs))
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _stale(LIB, objs):
        run([nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB, *objs])
    return LIB


if __name__ == "__main__":
    _variant = sys.argv[sys.argv.index("--variant") + 1] if "--variant" in sys.argv else ""
    print(build(force="--force" in sys.argv, verbose=True, variant=_variant))
