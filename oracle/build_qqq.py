"""Recipe: compile the REFERENCE's own QQQ kernel (gptqmodel_ext/qqq: qqq.cpp, qqq_gemm.cu; a Marlin derivative on
mma.sync) for sm_90a from a GPTQModel source checkout, into oracle/_ref/ (git-ignored build output).  The checkout is
$GPTQMODEL_SRC, by default /root/reference.

  [GPTQMODEL_SRC=/path/to/GPTQModel] python oracle/build_qqq.py

Nothing is copied into the repository.  Loading oracle/_ref/gptqmodel_qqq.so with torch.ops.load_library registers
torch.ops.gptqmodel_qqq.qqq_gemm.  Used by tests/test_gpu_qqq.py (cross-check) and tools/qqq_bench.py (competitor).
"""
import os
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
SRC = os.environ.get("GPTQMODEL_SRC") or "/root/reference"
REF = Path(SRC) / "gptqmodel_ext" / "qqq"
OUT = ROOT / "oracle" / "_ref"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
SO = OUT / "gptqmodel_qqq.so"


def main():
    if not REF.exists():
        print(f"{REF} not present: using the prebuilt oracle/_ref if any")
        return 0
    import torch
    from torch.utils import cpp_extension as ce

    OUT.mkdir(parents=True, exist_ok=True)
    inc = [f"-I{REF}"] + [f"-I{p}" for p in ce.include_paths("cuda")]
    import sysconfig
    inc.append(f"-I{sysconfig.get_paths()['include']}")
    abi = f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}"
    common = ["-O3", "-std=c++17", abi, "-DTORCH_API_INCLUDE_EXTENSION_H"]
    cuflags = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-Xcompiler", "-fPIC",
               "--expt-relaxed-constexpr", "--expt-extended-lambda", "-U__CUDA_NO_HALF_OPERATORS__",
               "-U__CUDA_NO_HALF_CONVERSIONS__", "-U__CUDA_NO_HALF2_OPERATORS__", "-diag-suppress=177,174,2361"]
    t0 = time.time()
    objs = []
    for src in (REF / "qqq_gemm.cu", REF / "qqq.cpp"):
        obj = OUT / ("qqq_" + src.stem + ".o")
        if not (obj.exists() and obj.stat().st_mtime > src.stat().st_mtime):
            if src.suffix == ".cu":
                cmd = [NVCC, *common, *cuflags, *inc, "-c", str(src), "-o", str(obj)]
            else:
                cmd = ["g++", *common, "-fPIC", *inc, "-c", str(src), "-o", str(obj)]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                print(" ".join(cmd))
                print(r.stderr[-4000:])
                raise SystemExit(f"compile failed: {src.name}")
        objs.append(obj)
    libdir = os.path.join(os.path.dirname(torch.__file__), "lib")
    cmd = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(SO), *map(str, objs), f"-L{libdir}",
           "-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_cuda", "-lc10_cuda", "-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        print(r.stderr[-4000:])
        raise SystemExit("link failed")
    print(f"built {SO} ({SO.stat().st_size / 1e6:.1f} MB) in {time.time() - t0:.0f}s")
    return 0


if __name__ == "__main__":
    sys.exit(main())
