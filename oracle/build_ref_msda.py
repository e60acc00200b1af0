#!/usr/bin/env python
"""Build the REFERENCE's own MSDeformAttn CUDA op for sm_90a (H100) into the git-ignored oracle/_ref/ (no reference
source is copied into this repository).

    PSALM_REFERENCE_ROOT=<reference checkout> python oracle/build_ref_msda.py

Recipe: copy ops/src to a temporary directory (the reference tree is treated as read-only), apply the two-line
`value.type()` -> `value.scalar_type()` fix inside the AT_DISPATCH macros (ms_deform_attn_cuda.cu:69,139; torch >= 2
removed the deprecated overload), compile with torch.utils.cpp_extension for compute capability 9.0a.
oracle/gen_golden_msda_cuda.py runs the built op once on a GPU to store the fixture tests/golden/msda_ref_cuda.npz, and
tools/bench_msda.py times it beside our kernels when it is present.
"""
import glob
import os
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS = "psalm/model/mask_decoder/Mask2Former_Simplify/modeling/pixel_decoder/ops/src"
OUT = os.path.join(ROOT, "oracle", "_ref")


def main():
    ref_root = os.environ.get("PSALM_REFERENCE_ROOT")
    ref_ops = os.path.join(ref_root, OPS) if ref_root else None
    if not ref_ops or not os.path.isdir(ref_ops):
        print("reference sources not found (set PSALM_REFERENCE_ROOT): nothing to build")
        return 1
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "8")
    scratch = os.path.join(tempfile.mkdtemp(prefix="psalm_ref_msda_"), "src")
    shutil.copytree(ref_ops, scratch)
    cu = os.path.join(scratch, "cuda", "ms_deform_attn_cuda.cu")
    src = open(cu).read()
    n = src.count("HALF(value.type(),")
    src = src.replace("HALF(value.type(),", "HALF(value.scalar_type(),")   # lines 69 and 139 only
    open(cu, "w").write(src)
    print("patched %d dispatch sites" % n)
    from torch.utils.cpp_extension import load
    os.makedirs(OUT, exist_ok=True)
    sources = [os.path.join(scratch, "vision.cpp")] + glob.glob(os.path.join(scratch, "cpu", "*.cpp")) + \
        glob.glob(os.path.join(scratch, "cuda", "*.cu"))
    load(name="MultiScaleDeformableAttention", sources=sources, extra_include_paths=[scratch],
         extra_cflags=["-DWITH_CUDA"], extra_cuda_cflags=["-DWITH_CUDA", "-DCUDA_HAS_FP16=1", "-D__CUDA_NO_HALF_OPERATORS__",
                                                          "-D__CUDA_NO_HALF_CONVERSIONS__", "-D__CUDA_NO_HALF2_OPERATORS__"],
         build_directory=OUT, is_python_module=False, verbose=True)
    print("built:", glob.glob(os.path.join(OUT, "*.so")))
    return 0


if __name__ == "__main__":
    sys.exit(main())
