"""Builds libpfnav.so (hand-written sm_90a CUDA + the C ABI of include/pfnav.h) in-tree with nvcc.

The extension is NOT optional: callers fail loudly when it is missing (no CPU fallback)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libpfnav.so")
SOURCES = ["pfnav_fields.cu", "pfnav_agents.cu", "pfnav_plan.cu", "pfnav_route.cu", "pfnav_blockers.cu", "pfnav_region.cu", "pfnav_pfmap.cu", "pfnav_mgpu.cu", "pfnav_query.cu", "pfnav_pool.cu", "pfnav_commands.cu", "pfnav_events.cu", "pfnav_inputs.cu", "pfnav_checkpoint.cu", "pfnav_digest.cu"]
# H100 only: the kernels use Hopper's arch-specific features (TMA, mbarrier), so sm_90a code is built and nothing else
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = GENCODE + [
    "-O3", "-lineinfo", "-std=c++17",
    # bit-parity with the reference's x86-64 SSE float arithmetic: no FMA contraction
    "-fmad=false",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=default", "-cudart", "static",
]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "pfnav.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    def compile_one(src):
        obj = os.path.join(CSRC, src.replace(".cu", ".o"))
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(
                os.path.getmtime(os.path.join(CSRC, src)), *[os.path.getmtime(h) for h in HEADERS]):
            return obj
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose:
            sys.stderr.write(r.stderr)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, r.stderr))
        return obj

    HEADERS = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))] + \
              [os.path.join(HERE, "..", "include", "pfnav.h")]
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:      # one nvcc per translation unit
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [nvcc, "-shared", "-cudart", "static"] + GENCODE + ["-o", LIB] + objs + ["-ldl", "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
