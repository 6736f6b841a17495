"""In-tree build of libgut_b200.so (sm_90a only).  Called by __graft_entry__.build() and lazily by the loader.

One nvcc compile per translation unit so the projection kernels can be built with -fmad=false (integer
parity of tile counts / sort keys, see csrc/gut_project.cu) while the compositing kernels keep FMA contraction.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libgut_b200.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-ffp-contract=off"]
UNITS = {
    "gut_project.cu": ["-fmad=false"],
    "gut_sort.cu": [],
    "gut_binning.cu": [],
    # compositing kernels: same numerics mode as the reference build (-use_fast_math, setup_3dgut.py:108-109):
    # flush-to-zero, approximate div/sqrt/exp; parity is tolerance-based for these (DESIGN.md section 5)
    "gut_render.cu": ["--use_fast_math"],
    "gut_render_nht.cu": ["--use_fast_math"],
    "gut_render_kbuffer.cu": ["--use_fast_math", "--extended-lambda"],
    "gut_api.cu": ["-fmad=false"],
    "grt.cu": ["--use_fast_math"],
    # optimizer step: plain IEEE arithmetic (the reference plugin is built without fast-math, setup_optimizers.py)
    "gut_optim.cu": [],
    "gut_loss.cu": [],
    # evaluation metrics: no contraction, so that the composite rounds as its torch expression does (the PNG bytes and the LPIPS input
    # agree); IEEE division for the colour correction
    "gut_metrics.cu": ["-fmad=false"],
    "gut_debug.cu": [],
    # NHT feature decoder: fp16 tensor-core MLP, IEEE fp32 encoding and epilogues
    "nht_decoder.cu": [],
    # 3DGRUT hybrid: mirror rays and the composite, no contraction so that they match hybrid.py's torch expressions bit for bit
    "hybrid.cu": ["-fmad=false"],
    # playground mesh LBVH build and closest-hit queries (the triangle test itself is written with round-to-nearest intrinsics)
    "playground.cu": [],
    # exact k-nearest neighbours: the box bound and the distance must round the same way (DESIGN.md section 19)
    "gut_knn.cu": ["-fmad=false"],
}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build the sm_90a extension")


def sources():
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "gut_b200.h"), os.path.join(HERE, "..", "include", "grt_b200.h"),
                                                                os.path.join(HERE, "..", "include", "nht_b200.h"), os.path.abspath(__file__)]
    return deps


def needs_build() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(p) > t for p in sources())


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile into a private temp directory under an exclusive file lock and publish the library with one atomic rename: with one
    process per GPU under torchrun every rank may call this at once, and none may ever dlopen a half-written file."""
    import fcntl
    import tempfile

    if not force and not needs_build():
        return OUT
    nvcc = _nvcc()
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    with open(os.path.join(objdir, ".lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not needs_build():  # another rank built it while we waited
                return OUT
            with tempfile.TemporaryDirectory(dir=objdir, prefix="tmp_") as tmp:
                procs, objs = [], []
                for unit, extra in UNITS.items():
                    obj = os.path.join(tmp, unit.replace(".cu", ".o"))
                    cmd = [nvcc, *ARCH, *COMMON, *extra, "-Xptxas", "-v" if verbose else "-warn-spills", "-c", os.path.join(CSRC, unit), "-o", obj]
                    if verbose:
                        print(" ".join(cmd), file=sys.stderr)
                    procs.append((cmd, subprocess.Popen(cmd)))  # translation units compile in parallel
                    objs.append(obj)
                for cmd, pr in procs:
                    if pr.wait() != 0:
                        raise subprocess.CalledProcessError(pr.returncode, cmd)
                staged = os.path.join(tmp, "libgut_b200.so")
                subprocess.check_call([nvcc, *ARCH, "-shared", "-o", staged, *objs])
                os.replace(staged, OUT)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return OUT


if __name__ == "__main__":
    print(build(force=True, verbose="-v" in sys.argv))
