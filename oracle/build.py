"""Build recipes for the checker side (TEST INFRASTRUCTURE, never imported by detectron2_b200/).

build_oracle()  gcc -> oracle/_build/libd2oracle.so   (the C restatement, oracle/d2_oracle.c)
build_ref()     g++ -> oracle/_ref/d2_ref_cpu.so      (the reference's own CPU csrc, compiled from
                where the reference source tree lies (REF_SRC); sources are never copied.  The
                tests compare against reference outputs stored under tests/golden/, not against this .so.)

Reference build recipe follows SURVEY.md Appendix B.1: vision.cpp + */*_cpu.cpp + cocoeval.cpp,
loaded with torch.ops.load_library (TORCH_LIBRARY ops only; never imported as a python module).
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(HERE, "_build", "libd2oracle.so")
REF_DIR = os.path.join(HERE, "_ref")
REF_SO = os.path.join(REF_DIR, "d2_ref_cpu.so")
REF_CUDA_SO = os.path.join(REF_DIR, "d2_ref_cuda.so")
REF_SRC = "/root/reference/detectron2/layers/csrc"


def _newer(target, sources):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def build_oracle(force=False):
    src = os.path.join(HERE, "d2_oracle.c")
    if not force and _newer(ORACLE_SO, [src]):
        return ORACLE_SO
    os.makedirs(os.path.dirname(ORACLE_SO), exist_ok=True)
    cmd = ["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-fvisibility=hidden",
           "-Wall", "-Wextra", "-o", ORACLE_SO, src, "-lm"]
    subprocess.check_call(cmd)
    return ORACLE_SO


def build_ref(force=False):
    """Compile the reference CPU csrc in place. Returns the .so path, or None when the reference
    tree is absent and no .so was built before."""
    if os.path.exists(REF_SO) and not force:
        return REF_SO
    if not os.path.isdir(REF_SRC):
        return REF_SO if os.path.exists(REF_SO) else None
    from torch.utils.cpp_extension import load

    os.makedirs(REF_DIR, exist_ok=True)
    sources = [os.path.join(REF_SRC, "vision.cpp")] + sorted(glob.glob(os.path.join(REF_SRC, "**", "*.cpp")))
    load(name="d2_ref_cpu", sources=sources, extra_include_paths=[REF_SRC], build_directory=REF_DIR,
         is_python_module=False, verbose=False)
    # keep only the library; drop object files / ninja logs so the snapshot stays small
    for f in os.listdir(REF_DIR):
        if not f.endswith(".so"):
            try:
                os.remove(os.path.join(REF_DIR, f))
            except OSError:
                pass
    return REF_SO


def build_ref_cuda(force=False):
    """The reference's full csrc (CPU + CUDA kernels) compiled for sm_90a: the GPU kernel-to-beat of the rotated ops and
    of deformable convolution (SURVEY.md Appendix B.2, flags of the reference's setup.py:74-80).  A python extension
    module (`import d2_ref_cuda` after putting oracle/_ref on sys.path) because the five deform-conv functions are
    pybind-only (csrc/vision.cpp:86-102).  Compiles here without a GPU; only tools/ and tests/ ever load it."""
    if os.path.exists(REF_CUDA_SO) and not force:
        return REF_CUDA_SO
    if not os.path.isdir(REF_SRC):
        return REF_CUDA_SO if os.path.exists(REF_CUDA_SO) else None
    from torch.utils.cpp_extension import load

    bdir = os.path.join(REF_DIR, "_cuda_build")
    os.makedirs(bdir, exist_ok=True)
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    sources = ([os.path.join(REF_SRC, "vision.cpp")] + sorted(glob.glob(os.path.join(REF_SRC, "**", "*.cpp")))
               + sorted(glob.glob(os.path.join(REF_SRC, "**", "*.cu"))) + sorted(glob.glob(os.path.join(REF_SRC, "*.cu"))))
    load(name="d2_ref_cuda", sources=sources, extra_include_paths=[REF_SRC], build_directory=bdir, with_cuda=True,
         extra_cflags=["-DWITH_CUDA"],
         extra_cuda_cflags=["-DWITH_CUDA", "-O3", "-DCUDA_HAS_FP16=1", "-D__CUDA_NO_HALF_OPERATORS__",
                            "-D__CUDA_NO_HALF_CONVERSIONS__", "-D__CUDA_NO_HALF2_OPERATORS__"],
         is_python_module=False, verbose=False)
    os.replace(os.path.join(bdir, "d2_ref_cuda.so"), REF_CUDA_SO)
    import shutil

    shutil.rmtree(bdir, ignore_errors=True)
    return REF_CUDA_SO


if __name__ == "__main__":
    print(build_oracle(force="--force" in sys.argv))
    print(build_ref(force="--force" in sys.argv))
    if "--cuda" in sys.argv:
        print(build_ref_cuda(force="--force" in sys.argv))
