"""In-tree build of the CUDA library (and, for tests, the C oracle)."""
from __future__ import annotations

import os
import subprocess
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent
CSRC = PKG / "csrc"
LIB = PKG / "libwheeledlab_b200.so"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "-fmad=false",                    # bit-exact parity with the oracle (DESIGN.md "Determinism")
    "-Xcompiler", "-fPIC", "-shared",
]


def _stale(target: Path, sources) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(s).stat().st_mtime > t for s in sources)


def build_native(force: bool = False, verbose: bool = False) -> Path:
    srcs = [CSRC / "wl_api.cu"]
    deps = srcs + list(CSRC.glob("*.cuh")) + [ROOT / "include" / "wheeledlab_b200.h"]
    if force or _stale(LIB, deps):
        extra = [f"-DWL_STEP_MIN_BLOCKS={os.environ['WL_STEP_MIN_BLOCKS']}"] if os.environ.get("WL_STEP_MIN_BLOCKS") else []
        cmd = [NVCC, *NVCC_FLAGS, *extra, *(["-Xptxas", "-v"] if verbose else []), "-o", str(LIB), *map(str, srcs)]
        subprocess.run(cmd, check=True, cwd=str(ROOT))
    return LIB


TORCH_OPS = PKG / "_wl_torch_ops.so"


def build_torch_ops(force: bool = False) -> Path:
    """The PyTorch-extension front (csrc/wl_torch_ops.cpp, `torch.ops.wheeledlab_b200.*`): plain g++ against torch's headers,
    linked to the CUDA library next to it (rpath $ORIGIN).  No kernels in it; ~10 s to compile."""
    import torch
    from torch.utils import cpp_extension as ce
    build_native()
    src = CSRC / "wl_torch_ops.cpp"
    if force or _stale(TORCH_OPS, [src, ROOT / "include" / "wheeledlab_b200.h"]):
        tlib = ce.library_paths()[0]
        cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}",
               *[f"-I{p}" for p in ce.include_paths()], "-I/usr/local/cuda/include", str(src), "-o", str(TORCH_OPS),
               f"-L{tlib}", "-ltorch", "-ltorch_cpu", "-ltorch_cuda", "-lc10", "-lc10_cuda", f"-L{PKG}", f"-l:{LIB.name}",
               "-Wl,-rpath,$ORIGIN", f"-Wl,-rpath,{tlib}"]
        subprocess.run(cmd, check=True, cwd=str(ROOT))
    return TORCH_OPS


def build_oracle(force: bool = False, native: bool = False) -> Path:
    odir = ROOT / "oracle"
    targets = ["libwl_oracle.so", "libwl_oracle_f64.so"] + (["libwl_oracle_native.so"] if native else [])
    if force:
        subprocess.run(["make", "-C", str(odir), "clean"], check=True)
    subprocess.run(["make", "-C", str(odir), *targets], check=True, stdout=subprocess.DEVNULL)
    return odir / "libwl_oracle.so"


if __name__ == "__main__":
    print(build_native(force=True, verbose=True))
    print(build_torch_ops(force=True))
    print(build_oracle())
