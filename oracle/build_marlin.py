"""Recipe: compile the REFERENCE's own Marlin kernel (gptqmodel_ext/marlin, fp16 op) for sm_90a from a GPTQModel source
checkout, into oracle/_ref/ (git-ignored build output).  The checkout is $GPTQMODEL_SRC, by default /root/reference.

  [GPTQMODEL_SRC=/path/to/GPTQModel] python oracle/build_marlin.py [--jobs 8]

Nothing is copied into the repository: the only files written are the generated template instantiations
(generate_kernels.py's own output, rendered into oracle/_ref/marlin_gen/ so the checkout may be read-only) and the
objects / .so.  Flags follow gptqmodel/utils/marlin.py:153-208 (default_jit_cuda_cflags: -O3, --use_fast_math is NOT
set there, bf16 enabled, -static-global-template-stub=false, lineinfo) with the arch fixed to sm_90a.
Used by tools/competitors.py and bench.py's `competitors` block as the "marlin_ref" arm.
"""
import argparse
import importlib.util
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
SRC = os.environ.get("GPTQMODEL_SRC") or "/root/reference"
REF = Path(SRC) / "gptqmodel_ext" / "marlin"
OUT = ROOT / "oracle" / "_ref"
GEN = OUT / "marlin_gen"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", type=int, default=os.cpu_count() or 4)
    ap.add_argument("--dtype", default="fp16")
    args = ap.parse_args()
    if not REF.exists():
        print(f"{REF} not present: using the prebuilt oracle/_ref if any")
        return 0
    import torch
    from torch.utils import cpp_extension as ce

    GEN.mkdir(parents=True, exist_ok=True)
    spec = importlib.util.spec_from_file_location("_marlin_gen", REF / "generate_kernels.py")
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    expected = gen.build_expected_kernels(GEN)
    srcs = []
    for path, text in expected.items():
        if f"kernel_{args.dtype}_" not in path.name:
            continue
        if not path.exists() or path.read_text() != text:
            path.write_text(text)
        srcs.append(path)
    srcs += [REF / f"gptq_marlin_{args.dtype}.cu", REF / "gptq_marlin_repack.cu", REF / "awq_marlin_repack.cu",
             REF / f"marlin_torch_{args.dtype}.cpp"]
    inc = [f"-I{REF}"] + [f"-I{p}" for p in ce.include_paths("cuda")]
    abi = f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}"
    common = ["-O3", "-std=c++17", abi, "-DTORCH_API_INCLUDE_EXTENSION_H", "-DPy_LIMITED_API=0x03090000"]
    cuflags = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-Xcompiler", "-fPIC",
               "--expt-relaxed-constexpr", "--expt-extended-lambda", "-static-global-template-stub=false",
               "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__", "-U__CUDA_NO_BFLOAT16_CONVERSIONS__",
               "-U__CUDA_NO_HALF2_OPERATORS__", "-diag-suppress=177,174,2361", "-Xfatbin", "-compress-all"]

    def compile_one(src):
        obj = OUT / (src.stem + ".o")
        if obj.exists() and obj.stat().st_mtime > src.stat().st_mtime:
            return obj, 0.0
        t0 = time.time()
        if src.suffix == ".cu":
            cmd = [NVCC, *common, *cuflags, *inc, "-c", str(src), "-o", str(obj)]
        else:
            cmd = ["g++", *common, "-fPIC", *inc, "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            print(" ".join(cmd))
            print(r.stderr[-4000:])
            raise SystemExit(f"compile failed: {src.name}")
        return obj, time.time() - t0

    t0 = time.time()
    with ThreadPoolExecutor(args.jobs) as ex:
        objs = []
        for obj, dt in ex.map(compile_one, srcs):
            print(f"  {obj.name}: {dt:.0f}s", flush=True)
            objs.append(obj)
    so = OUT / f"gptqmodel_marlin_{args.dtype}.so"
    libdir = os.path.join(os.path.dirname(torch.__file__), "lib")
    cmd = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(so), *map(str, objs), f"-L{libdir}",
           "-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_cuda", "-lc10_cuda", "-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        print(r.stderr[-4000:])
        raise SystemExit("link failed")
    print(f"built {so} ({so.stat().st_size / 1e6:.1f} MB) in {time.time() - t0:.0f}s")
    return 0


if __name__ == "__main__":
    sys.exit(main())
